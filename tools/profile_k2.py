"""Developer tool: set up the 100k company-names workload (real fixture when present) and launch K2 a few times (for a profiler run)."""
import sys, os
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch
from polyfuzz_b200 import datasets, engine
n = int(sys.argv[1]); tile = int(sys.argv[2]); variant = sys.argv[3]; reps = int(sys.argv[4]) if len(sys.argv) > 4 else 3
names, _ = datasets.load_company_names(n)
v = engine.NgramTfidf((3, 3), True, True)
(rows,) = v.fit_rows([names]); csr = v.emit(rows)
ix = engine.SparseIndex(csr, tile=tile, variant=variant)
for _ in range(reps):
    engine.spcos_topk(csr, ix, 10, 0.0, self_match=True, n_splits=1, variant=variant)
torch.cuda.synchronize()
print("done")
