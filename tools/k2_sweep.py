"""Developer tool: time K1 stages and K2 over tile sizes on the company-names workload (real fixture when present).

    python tools/k2_sweep.py [N] [TILES] [VARIANTS] [--rows 8,16] [--rounds R] [--lib PATH] [--json FILE]

--rows sets the block kernel's rows per CTA (PFZ_BLOCK_ROWS) per configuration; --rounds R times every (variant, tile, rows)
configuration once per round, the configurations alternating, so slow drift of the clock falls on all of them alike.
--lib loads another build of libpfz.so (e.g. one built with PFZ_NVCC_EXTRA='-DPFZ_B3_MIN_CTAS(BF)=(24/(BF))'), and
--json appends one record per configuration to FILE.
"""
import argparse
import json
import os
import sys
import time
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("n", nargs="?", type=int, default=100_000)
ap.add_argument("tiles", nargs="?", default="512,1024,1536,2048,2560,2816")
ap.add_argument("variants", nargs="?", default="dense32,dense,list")
ap.add_argument("--rows", default=None, help="block kernel rows per CTA, comma list (default: PFZ_BLOCK_ROWS)")
ap.add_argument("--rounds", type=int, default=1)
ap.add_argument("--lib", default=None)
ap.add_argument("--json", default=None)
args = ap.parse_args()

from polyfuzz_b200 import _lib
if args.lib:
    _lib._LIB_PATH = os.path.abspath(args.lib)
import torch
from polyfuzz_b200 import datasets, engine

n = args.n
tiles = [int(t) for t in args.tiles.split(",")]
variants = args.variants.split(",")
rows_list = [int(r) for r in args.rows.split(",")] if args.rows else [engine.BLOCK_ROWS]
names, _kind = datasets.load_company_names(n)
torch.cuda.init()


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        out = fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); out = fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return out, float(np.median(ts)), float(np.min(ts))


t0 = time.time(); v = engine.NgramTfidf((3, 3), True, True)
(rows,), t_fit, _ = timed(lambda: v.fit_rows([names]), 3, 1)
csr, t_emit, _ = timed(lambda: v.emit(rows), 3, 1)
torch.cuda.synchronize()
ip = csr.indptr.cpu().numpy(); nnz = int(ip[-1])
df = np.bincount(csr.indices[:nnz].cpu().numpy(), minlength=v.n_vocab).astype(np.float64)
P = float((df * df).sum())
print(f"n={n} V={v.n_vocab} nnz={nnz} P={P:.4g} fit(stageA+vocab incl. H2D, host idf)={t_fit:.2f} ms emit={t_emit:.2f} ms wall={time.time()-t0:.2f}s")
ref = None
configs = [(variant, tile, br) for variant in variants for tile in tiles for br in (rows_list if variant == "block" else [None])]
indexes = {}
for rnd in range(args.rounds):
    for variant, tile, br in configs:
        if br is not None:
            engine.BLOCK_ROWS = br
        if (variant, tile) not in indexes:
            indexes[(variant, tile)] = timed(lambda: engine.SparseIndex(csr, tile=tile, variant=variant), 3, 1)
        idx_obj, t_ix, _ = indexes[(variant, tile)]
        (oi, ov), t_k2, t_min = timed(lambda: engine.spcos_topk(csr, idx_obj, 10, 0.0, self_match=True, n_splits=1, variant=variant), 5, 2)
        if ref is None:
            ref = (oi.clone(), ov.clone())
        same = bool(torch.equal(oi, ref[0]) and torch.equal(ov, ref[1]))
        pairs = float(n) * n - n
        print(f"round {rnd} {variant:5s} rows={br} same={same} tile={tile:5d} n_tiles={idx_obj.n_tiles:4d} index_build={t_ix:7.2f} ms  "
              f"K2 median={t_k2:8.2f} ms min={t_min:8.2f} ms  pairs/s={pairs / (t_k2 * 1e-3):.3e}  postings/s={P / (t_k2 * 1e-3):.3e}  "
              f"B_alg GB/s={(P * 12 + nnz * 12 + n * 120) / (t_k2 * 1e-3) / 1e9:.1f}", flush=True)
        if args.json:
            with open(args.json, "a") as f:
                f.write(json.dumps({"lib": args.lib or "package", "round": rnd, "variant": variant, "tile": tile, "rows": br, "same": same,
                                    "k2_median_ms": t_k2, "k2_min_ms": t_min}) + "\n")
