import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, ctypes
from peritext_b200 import workload
from peritext_b200.engine import PipelinedEngine, INSDEL_C8_DT, MARK_C16_DT, _packed_ops, load_library
from peritext_b200.packing import INSDEL_DT, MARK_DT, PackedBatch
b = workload.generate("c4", n_docs=int(sys.argv[1]) if len(sys.argv) > 1 else 30000)
def pinned(a): return torch.from_numpy(a.view(np.uint8).reshape(-1)).pin_memory()
p_ins, p_mk = pinned(b.insdel), pinned(b.marks)
pb = PackedBatch(b.desc, p_ins.numpy()[: b.insdel.nbytes].view(INSDEL_DT), p_mk.numpy()[: b.marks.nbytes].view(MARK_DT), meta=b.meta)
L = load_library()
ci = torch.empty(len(b.insdel) * 8, dtype=torch.uint8).pin_memory(); cm = torch.empty(len(b.marks) * 16, dtype=torch.uint8).pin_memory()
desc = np.ascontiguousarray(b.desc)
ops = _packed_ops(desc, pb.insdel, len(pb.insdel), pb.marks, len(pb.marks))
for T in (16, 32, 64, 128):
    L.pt_compact_ops(ctypes.byref(ops), ci.data_ptr(), cm.data_ptr(), T)
    t0 = time.perf_counter(); L.pt_compact_ops(ctypes.byref(ops), ci.data_ptr(), cm.data_ptr(), T); dt = time.perf_counter() - t0
    print("convert threads", T, "ms", round(dt * 1e3, 2), "GB/s in", round((b.insdel.nbytes + b.marks.nbytes) / dt / 1e9, 1))
pipe = PipelinedEngine(0, chunks=4)
for compact in (False, True):
    for T in ((0,) if not compact else (32, 64, 128)):
        for _ in range(2): pipe.run(pb, compact=compact, threads=T)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for _ in range(5): pipe.run(pb, compact=compact, threads=T)
        torch.cuda.synchronize(); print("pipe compact", compact, "threads", T, "ms", round((time.perf_counter() - t0) / 5 * 1e3, 2))
