"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every symbol that
include/peritext_b200.h declares; without a GPU it fails loudly instead of falling back."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "peritext_b200.h")).read()
    return sorted(set(re.findall(r"\b(pt_[a-z_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import engine
    lib = engine.load_library()
    syms = declared_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(lib, s), s
    assert sorted(engine.EXPORTS) == syms
    assert b"sm_90a" in lib.pt_version()


# every layout the binding mirrors -> its header type (the mirrors' field names are the header's)
HEADER_TYPES = {
    "_PackedOps": ("pt_packed_ops", "pt_packed_compact"), "_PackedRuns": ("pt_packed_runs",), "_ChangeTable": ("pt_change_table",),
    "_AppendRemap": ("pt_append_remap",), "_ChangeInput": ("pt_change_input",), "_ChangeView": ("pt_change_view",),
    "_ExchangeInput": ("pt_exchange_input",), "_ExchangeView": ("pt_exchange_view",), "_ActorTables": ("pt_actor_tables",),
    "_ActorInput": ("pt_actor_input",), "_ActorView": ("pt_actor_view",), "_SyncView": ("pt_sync_view",), "_SpansView": ("pt_spans_view",),
    "_Limits": ("pt_limits",), "_PatchView": ("pt_patch_view",), "_JsonPools": ("pt_json_pools",), "_JsonView": ("pt_json_view",),
    "_ChangesJsonInput": ("pt_changes_json_input",), "_ChangesJsonView": ("pt_changes_json_view",),
    "INSDEL_DT": ("pt_insdel_rec",), "MARK_DT": ("pt_mark_rec",), "DESC_DT": ("pt_log_desc",), "RESULT_DT": ("pt_log_result",),
    "SPAN_DT": ("pt_span",), "CHANGE_DT": ("pt_change_rec",), "DEP_DT": ("pt_dep_rec",), "CDESC_DT": ("pt_change_desc",),
    "ELEM_REF_DT": ("pt_elem_ref",), "ELEM_POS_DT": ("pt_elem_pos",), "INPUT_OP_DT": ("pt_input_op",), "CHANGE_STATUS_DT": ("pt_change_status",),
    "EXTRA_DT": ("pt_change_extra",), "CHANGES_REQUEST_DT": ("pt_changes_request",), "CLOCK_DT": ("pt_clock_entry",),
    "INSDEL_C8_DT": ("pt_insdel_c8",), "MARK_C16_DT": ("pt_mark_c16",), "RUN_DT": ("pt_run_rec",), "PAIR_DT": ("pt_exchange_pair",),
    "QUERY_DT": ("pt_elem_query",), "PATCH_REC_DT": ("pt_patch_rec",), "PATCH_ITEM_DT": ("pt_patch_item",),
}


def mirrored_layouts():
    """name -> (size, [(field, offset, size)]) of every ctypes Structure defined in peritext_b200.engine and every *_DT dtype of
    peritext_b200.packing and peritext_b200.engine."""
    import numpy as np
    from peritext_b200 import engine, packing
    out = {}
    for name, c in vars(engine).items():
        if isinstance(c, type) and issubclass(c, ctypes.Structure) and c.__module__ == engine.__name__:
            out[name] = (ctypes.sizeof(c), [(f, getattr(c, f).offset, getattr(c, f).size) for f, *_ in c._fields_])
    for mod in (packing, engine):
        for name, dt in vars(mod).items():
            if name.endswith("_DT") and isinstance(dt, np.dtype):
                out[name] = (dt.itemsize, [(f, dt.fields[f][1], dt.fields[f][0].itemsize) for f in dt.names])
    return out


def test_struct_layouts_match_header(tmp_path):
    """Every mirrored struct has the header's size, and every field its offset and size, checked by the C compiler."""
    layouts = mirrored_layouts()
    assert sorted(layouts) == sorted(HEADER_TYPES), "mirrors without a header type, or header types without a mirror"
    lines = ['#include "peritext_b200.h"']
    for name, (size, fields) in sorted(layouts.items()):
        for t in HEADER_TYPES[name]:
            lines.append(f'_Static_assert(sizeof({t}) == {size}, "{name}: sizeof({t}) is not {size}");')
            for f, off, fsize in fields:
                lines.append(f'_Static_assert(offsetof({t}, {f}) == {off}, "{name}.{f}: offsetof({t}, {f}) is not {off}");')
                lines.append(f'_Static_assert(sizeof((({t}*)0)->{f}) == {fsize}, "{name}.{f}: sizeof({t}.{f}) is not {fsize}");')
    src = tmp_path / "layouts.c"
    src.write_text("\n".join(lines) + "\n")
    r = subprocess.run(["gcc", "-std=c11", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from peritext_b200.engine import BatchEngine, EngineError
    with pytest.raises(EngineError, match="no CPU fallback"):
        BatchEngine(0)


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under peritext_b200/ may reference it."""
    pkg = os.path.join(ROOT, "peritext_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, f), encoding="utf-8").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M), f
                assert "oracle/" not in txt.replace("tests/", ""), f


def test_run_compression_is_lossless():
    """pt_compress_runs (host code of the C-ABI library): expanding the runs gives back the records bit for bit."""
    import numpy as np
    from peritext_b200 import workload
    from peritext_b200.engine import compress_runs
    for cfg in ("c2", "c3", "c4"):
        b = workload.generate(cfg, n_docs=6, ops_per_doc=1500)
        r = compress_runs(b)
        out = np.zeros(len(b.insdel), b.insdel.dtype)
        for li in range(b.n_logs):
            o, t, k = int(b.desc[li]["insdel_off"]), int(r.tok_off[li]), 0
            for q in r.runs[int(r.run_off[li]): int(r.run_off[li + 1])]:
                cnt, kind = int(q["kind_count"]) & 0x3FFFFFFF, int(q["kind_count"]) >> 30
                for j in range(cnt):
                    if kind == 0:
                        out[o + k] = (int(q["ctr0"]) + j, int(q["ref_ctr"]) if j == 0 else int(q["ctr0"]) + j - 1, int(q["actor"]),
                                      int(q["ref_actor"]) if j == 0 else int(q["actor"]), int(r.tokens[t])); t += 1
                    else:
                        out[o + k] = (int(q["ctr0"]) + j, int(q["ref_ctr"]) + j, int(q["actor"]), int(q["ref_actor"]), 1 << 30)
                    k += 1
            assert k == int(b.desc[li]["n_insdel"])
        assert out.tobytes() == b.insdel.tobytes()
        assert r.nbytes < b.insdel.nbytes + b.marks.nbytes + b.desc.nbytes * 2
