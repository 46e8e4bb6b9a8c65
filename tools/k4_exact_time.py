"""Developer tool: time K4's exact mode (Embeddings(precision="fp64")) against the bf16 path on C4-shaped inputs.

    python tools/k4_exact_time.py [--n 100000] [--d 768] [--k 10] [--rounds 12] [--warmup 3] [--kcand 0,16] [--data c4,clustered]

Per data set, in one process: the bf16 `dense_topk` and the exact pipeline alternate, each between CUDA events after the
warm-up; the exact pipeline is split into its stages (prep of both sides, fp16 filter, fp64 re-score + certificate,
fallback).  Medians of `--rounds` calls.  c4 = the C4 inputs (torch seeds 0 / 1, Gaussian rows); clustered = 400 centres plus
Gaussian noise of the same scale.  The card's name, power limit and SM clocks are read with nvidia-smi in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np
import torch

from polyfuzz_b200 import dense


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def make(kind, n, d, dev):
    if kind == "c4":
        torch.manual_seed(0); X = torch.randn(n, d, device=dev)
        torch.manual_seed(1); Y = torch.randn(n, d, device=dev)
        return X, Y
    g = torch.Generator(device=dev).manual_seed(7)
    C = torch.randn(400, d, device=dev, generator=g)
    X = C[torch.randint(0, 400, (n,), device=dev, generator=g)] + torch.randn(n, d, device=dev, generator=g)
    Y = C[torch.randint(0, 400, (n,), device=dev, generator=g)] + torch.randn(n, d, device=dev, generator=g)
    return X, Y


def timed(fn):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); out = fn(); e1.record()
    return e0, e1, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kcand", default="0", help="comma list of filter candidates per row; 0 = the default for k")
    ap.add_argument("--data", default="c4,clustered")
    a = ap.parse_args()
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for kind in a.data.split(","):
        X, Y = make(kind, a.n, a.d, dev)
        xb, _ = dense.to_bf16_rows(X, True); yb, _ = dense.to_bf16_rows(Y, True)
        for kc in [int(v) for v in a.kcand.split(",")]:
            kc = kc or dense.k_cand_for(a.k)
            rec = {"bf16": [], "prep": [], "filter": [], "rescore": [], "fallback": [], "exact": []}
            fb_rows = None
            for r in range(a.warmup + a.rounds):
                b = timed(lambda: dense.dense_topk(xb, yb, a.k, 0.0))
                p = timed(lambda: (dense.stage_exact(X), dense.stage_exact(Y)))
                xs, ys = p[2]
                f = timed(lambda: dense.candidates_f16(xs, ys, kc, 0.0))
                ci, cv = f[2]
                s = timed(lambda: dense.exact_rescore(xs, ys, ci, cv, a.k, 0.0))
                idx, val, rows, cnt = s[2]
                fbk = timed(lambda: dense.exact_fallback(xs, ys, idx, val, rows, cnt, 0.0))
                torch.cuda.synchronize()
                if r >= a.warmup:
                    rec["bf16"].append(b[0].elapsed_time(b[1]))
                    rec["prep"].append(p[0].elapsed_time(p[1])); rec["filter"].append(f[0].elapsed_time(f[1]))
                    rec["rescore"].append(s[0].elapsed_time(s[1])); rec["fallback"].append(fbk[0].elapsed_time(fbk[1]))
                    rec["exact"].append(p[0].elapsed_time(fbk[1]))
                fb_rows = int(cnt.item())
                del xs, ys, ci, cv, idx, val, rows, cnt
            out = {"data": kind, "n_from": a.n, "n_to": a.n, "d": a.d, "k": a.k, "k_cand": kc, "fallback_rows": fb_rows,
                   "rounds": a.rounds, "median_ms": {key: round(float(np.median(v)), 3) for key, v in rec.items()},
                   "min_ms": {key: round(float(np.min(v)), 3) for key, v in rec.items()},
                   "max_ms": {key: round(float(np.max(v)), 3) for key, v in rec.items()}}
            print(json.dumps(out), flush=True)
        del X, Y, xb, yb
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
