"""The compact wire format (pt_compact_ops: 8-byte ins/del and 16-byte mark records, include/peritext_b200.h): the host
converter is elementwise and lossless for representable logs — checked on CPU by expanding in numpy exactly like the device
kernels do — and refuses logs it cannot represent."""
import ctypes

import numpy as np
import pytest

from peritext_b200 import workload
from peritext_b200.engine import INSDEL_C8_DT, MARK_C16_DT, EngineError, _check, _packed_ops, load_library
from peritext_b200.packing import DESC_DT, INSDEL_DT, MARK_DT, TOKEN_POOLED, PackedBatch


def convert(batch, threads=3):
    L = load_library()
    desc = np.ascontiguousarray(batch.desc); ins = np.ascontiguousarray(batch.insdel); mk = np.ascontiguousarray(batch.marks)
    ci = np.zeros(max(1, len(ins)), INSDEL_C8_DT); cm = np.zeros(max(1, len(mk)), MARK_C16_DT)
    ops = _packed_ops(desc, ins, len(ins), mk, len(mk))
    _check(L.pt_compact_ops(ctypes.byref(ops), ci.ctypes.data, cm.ctypes.data, threads), "pt_compact_ops")
    return ci[: len(ins)], cm[: len(mk)]


def expand(ci, cm):
    ins = np.zeros(len(ci), INSDEL_DT); mk = np.zeros(len(cm), MARK_DT)
    w = ci["w"]; tok = w >> 10
    ins["ctr"], ins["ref_ctr"], ins["actor"], ins["ref_actor"] = ci["ctr"], ci["ref_ctr"], w & 0xF, (w >> 4) & 0xF
    ins["payload"] = (((w >> 8) & 3) << 30) | np.where(tok & 0x200000, 0x20000000, 0) | (tok & 0x1FFFFF)
    w = cm["w"]
    mk["ctr"], mk["start_ctr"], mk["end_ctr"], mk["arrival"], mk["attr"] = cm["ctr"], cm["start_ctr"], cm["end_ctr"], cm["arrival"], cm["attr"]
    mk["actor"], mk["start_actor"], mk["end_actor"], mk["kind"], mk["bounds"] = w & 0xF, (w >> 4) & 0xF, (w >> 8) & 0xF, (w >> 12) & 7, (w >> 15) & 0xF
    return ins, mk


@pytest.mark.parametrize("cfg,n_docs,ops", [("c4", 40, 1000), ("c3", 4, 4000), ("c2", 4, 4000)])
def test_round_trip(cfg, n_docs, ops):
    b = workload.generate(cfg, n_docs=n_docs, ops_per_doc=ops)
    ins, mk = expand(*convert(b))
    assert ins.tobytes() == b.insdel.tobytes()
    assert mk.tobytes() == b.marks.tobytes()


def test_pooled_values_and_unicode_tokens():
    from oracle.oracle import Micromerge
    from peritext_b200.packing import pack_logs
    from tests.harness import generateDocs
    docs, _, init = generateDocs(Micromerge, "ab", 1)
    c1 = docs[0].change([{"path": ["text"], "action": "insert", "index": 1, "values": [" is great!", "é", "\\U0001F600", "中"]}])["change"]
    b = pack_logs([[init, c1]])
    ins, mk = expand(*convert(b))
    assert ins.tobytes() == b.insdel.tobytes()


def test_unrepresentable_logs_are_refused():
    b = workload.generate("c2", n_docs=1, ops_per_doc=2000)
    b.desc["max_ctr"][0] = 70000
    with pytest.raises(EngineError):
        convert(b)


def edge_batch():
    """One log with every record field at the widest value the compact form holds: counters, arrival 65535, actor rank 15
    in every actor field, pooled value 0x1FFFFF, code point U+10FFFF, mark kind 7 and bounds 15."""
    desc = np.zeros(1, DESC_DT)
    desc[0] = (0, 0, 3, 1, 16, 65535)
    ins = np.zeros(3, INSDEL_DT)
    ins[0] = (65534, 0, 15, 0, 0x10FFFF)
    ins[1] = (65535, 65534, 15, 15, TOKEN_POOLED | 0x1FFFFF)
    ins[2] = (65533, 65535, 15, 15, 1 << 30)
    mk = np.zeros(1, MARK_DT)
    mk[0] = (65535, 15, 7, 15, 65535, 65535, 15, 15, 7, 65535, 0)
    return PackedBatch(desc, ins, mk)


def test_the_exact_edge_round_trips():
    b = edge_batch()
    ins, mk = expand(*convert(b))
    assert ins.tobytes() == b.insdel.tobytes()
    assert mk.tobytes() == b.marks.tobytes()


# (array, record, field, value one past its width, the field's name in the error)
ONE_PAST = [("insdel", 1, "ctr", 65536, "insert/delete ctr"), ("insdel", 2, "ref_ctr", 65536, "insert/delete ref_ctr"),
            ("insdel", 0, "actor", 16, "insert/delete actor"), ("insdel", 1, "ref_actor", 16, "insert/delete ref_actor"),
            ("insdel", 1, "payload", TOKEN_POOLED | 0x200000, "value token"),
            ("marks", 0, "ctr", 65536, "mark ctr"), ("marks", 0, "start_ctr", 65536, "mark start_ctr"),
            ("marks", 0, "end_ctr", 65536, "mark end_ctr"), ("marks", 0, "arrival", 65536, "mark arrival"),
            ("marks", 0, "actor", 16, "mark actor"), ("marks", 0, "start_actor", 16, "mark start_actor"),
            ("marks", 0, "end_actor", 16, "mark end_actor"), ("marks", 0, "kind", 8, "mark kind"), ("marks", 0, "bounds", 16, "mark bounds")]


@pytest.mark.parametrize("arr,k,field,value,name", ONE_PAST, ids=[f"{a}-{f}" for a, _, f, _, _ in ONE_PAST])
def test_each_field_one_past_its_width_is_refused(arr, k, field, value, name):
    """A record field the compact form would truncate (a faulty log's out-of-range reference or actor) is refused, whatever
    the descriptor says: truncated, it would name another element and merge where the plain form reports the fault."""
    b = edge_batch()
    getattr(b, arr)[k][field] = value
    with pytest.raises(EngineError, match=name):
        convert(b, threads=2)


def test_out_of_width_records_of_a_real_log_are_refused():
    """c4 logs (max_ctr well below 65536, 3 actors): a delete whose ref_ctr is a real counter + 65536, an insert whose actor
    rank is 16 + a real rank, a mark whose start_ctr is a real counter + 65536.  Each is refused alone, every thread count."""
    b = workload.generate("c4", n_docs=4, ops_per_doc=1000)
    assert int(b.desc["max_ctr"].max()) < 65536 and int(b.desc["n_actors"].max()) <= 16
    dels = np.nonzero((b.insdel["payload"] >> 30) == 1)[0]
    inss = np.nonzero((b.insdel["payload"] >> 30) == 0)[0]
    for arr, k, field, add, name in [("insdel", dels[len(dels) // 2], "ref_ctr", 65536, "ref_ctr"),
                                     ("insdel", inss[-1], "actor", 16, "insert/delete actor"),
                                     ("marks", len(b.marks) - 1, "start_ctr", 65536, "mark start_ctr")]:
        bad = PackedBatch(b.desc, b.insdel.copy(), b.marks.copy())
        a = getattr(bad, arr)
        a[k][field] = int(a[k][field]) + add
        for threads in (1, 3, 8):
            with pytest.raises(EngineError, match=name):
                convert(bad, threads=threads)
    convert(b)
