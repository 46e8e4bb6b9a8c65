"""Developer tool: K2 hash variant on uniform strings (BASELINE config 5 shape), timing + launches for a profiler run."""
import sys, os
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np, torch
from polyfuzz_b200 import engine, synth
n_to = int(sys.argv[1]); n_from = int(sys.argv[2]); reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
to = synth.uniform_strings(n_to, seed=0); frm = synth.uniform_strings(n_from, seed=1)
v = engine.NgramTfidf((3, 3), True, True)
rows_to, rows_from = v.fit_rows([to, frm]); csr_to, csr_from = v.emit(rows_to), v.emit(rows_from)
ix = engine.SparseIndex(csr_to, variant="hash")
print("slots", engine._hash_slots(ix), "tiles", ix.n_tiles, "V", v.n_vocab)
ts = []
for _ in range(reps):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); oi, ov = engine.spcos_topk(csr_from, ix, 10, 0.0); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
print(f"hash K2 {n_from} x {n_to}: {min(ts):.2f} ms  err={int(ix._hash_err.item())}")
