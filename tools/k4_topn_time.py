"""Developer tool: time K4 at top_n above 32 (DESIGN.md 4.7) in both precisions.

    python tools/k4_topn_time.py [--n 100000] [--d 768] [--k 10,32,33,64,100,256,1024] [--rounds 7] [--warmup 2] [--data c4,sorted]

Per data set and k, in one process, the bf16 and the exact (fp64) call alternate, each between CUDA events after the warm-up;
medians of `--rounds` calls (min-max alongside).  k <= 32 runs today's path (`dense_topk`, `dense_topk_exact`); k > 32 the bounded
path, split into its stages: bound pass, threshold pass, (exact: re-score +) select, overflow re-run (including its one
device-to-host read).  `--both-paths 16,32` also times those k on the bounded path.  c4 = the C4 inputs (torch seeds 0 / 1);
sorted = 400 Gaussian centres plus noise of the same scale, the to-list sorted by centre.  The exact mode's staging
(stage_exact) is done once outside the timed region.  The card's name, power limit and SM clocks are read with nvidia-smi in
the same run."""
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
    cy = torch.sort(torch.randint(0, 400, (n,), device=dev, generator=g)).values
    Y = C[cy] + torch.randn(n, d, device=dev, generator=g)
    return X, Y


def run_once(fn, bounded):
    """(total ms, {stage: ms}, overflow rows, candidates per row) of one call."""
    ev = []
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn(ev if bounded else None)
    e1.record()
    torch.cuda.synchronize()
    stages = {}
    for (name, a), (_, b) in zip(ev, ev[1:]):
        stages[name] = stages.get(name, 0.0) + a.elapsed_time(b)
    return e0.elapsed_time(e1), stages, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--k", default="10,32,33,64,100,256,1024")
    ap.add_argument("--both-paths", default="16,32")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--data", default="c4,sorted")
    a = ap.parse_args()
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    ks = [int(v) for v in a.k.split(",") if v]
    both = [int(v) for v in a.both_paths.split(",") if v]
    for kind in a.data.split(","):
        X, Y = make(kind, a.n, a.d, dev)
        xb, _ = dense.to_bf16_rows(X, True); yb, _ = dense.to_bf16_rows(Y, True)
        xs, ys = dense.stage_exact(X), dense.stage_exact(Y)
        cases = [(k, k > 32) for k in ks] + [(k, True) for k in both if k <= 32]
        for k, bounded in cases:
            calls = {}
            if bounded:
                calls["bf16"] = lambda ev, k=k: dense.dense_topn_bounded(xb, yb, k, 0.0, events=ev)[2]
                calls["fp64"] = lambda ev, k=k: dense.dense_topn_bounded(xs, ys, k, 0.0, events=ev)[2]
            else:
                calls["bf16"] = lambda ev, k=k: (dense.dense_topk(xb, yb, k, 0.0), 0)[1]
                calls["fp64"] = lambda ev, k=k: int(dense.dense_topk_exact(xs, ys, k, 0.0)[2].item())
            rec = {p: {"total": [], "stages": {}} for p in calls}
            extra = {p: None for p in calls}
            for r in range(a.warmup + a.rounds):
                for p, fn in calls.items():                      # alternate the precisions round by round
                    t, stages, out = run_once(fn, bounded)
                    if r >= a.warmup:
                        rec[p]["total"].append(t)
                        for s, v in stages.items():
                            rec[p]["stages"].setdefault(s, []).append(v)
                    extra[p] = out
            for p in calls:
                res = {"data": kind, "k": k, "precision": p, "path": "bounded" if bounded else "top-k kernel", "rounds": a.rounds,
                       "median_ms": round(float(np.median(rec[p]["total"])), 3),
                       "min_ms": round(float(np.min(rec[p]["total"])), 3), "max_ms": round(float(np.max(rec[p]["total"])), 3),
                       "stages_median_ms": {s: round(float(np.median(v)), 3) for s, v in rec[p]["stages"].items()}}
                res["overflow_rows" if bounded else ("fallback_rows" if p == "fp64" else "none")] = extra[p]
                if bounded:
                    res["candidates_per_row"] = candidates_per_row(xb, yb, xs, ys, k, p)
                res.pop("none", None)
                print(json.dumps(res), flush=True)
        del X, Y, xb, yb, xs, ys
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


def candidates_per_row(xb, yb, xs, ys, k, precision):
    """Mean and max threshold-pass count per row (an untimed call with an unbounded capacity on the first 4 096 rows)."""
    from polyfuzz_b200 import _lib
    from polyfuzz_b200.engine import _p, _stream
    exact = precision == "fp64"
    x = xs if exact else xb
    xo = (xs.f16 if exact else xb)[:4096]
    yo = ys.f16 if exact else yb
    m, n_to, d = xo.shape[0], yo.shape[0], xo.shape[1]
    n_tiles = (n_to + 127) // 128
    s = max(1, min(n_tiles, -(-2 * k // 16)))              # as dense_topn_bounded on chunks of >= 33k rows
    li = torch.empty((s, m, 16), dtype=torch.int32, device=xo.device); lv = torch.empty((s, m, 16), dtype=torch.float64, device=xo.device)
    _lib.call("pfz_dense_cos_topk_f16" if exact else "pfz_dense_cos_topk", _p(xo), _p(yo), m, n_to, d, 16, 0.0, 0, 0, 0, s, _p(li), _p(lv), _stream())
    thr = torch.empty(m, dtype=torch.float32, device=xo.device)
    _lib.call("pfz_dense_topn_bound", _p(li), _p(lv), s, m, 16, k, int(exact), _p(x.norm16[:m] if exact else None),
              _p(x.err16[:m] if exact else None), _p(ys.maxima if exact else None), d, 0.0, _p(thr), _stream())
    ci = torch.empty((m, 1), dtype=torch.int32, device=xo.device); cv = torch.empty((m, 1), dtype=torch.float64, device=xo.device)
    cnt = torch.empty(m, dtype=torch.int32, device=xo.device)
    _lib.call("pfz_dense_cos_cand_f16" if exact else "pfz_dense_cos_cand", _p(xo), _p(yo), m, n_to, d, 0.0, _p(thr), 0, s, 1, _p(ci), _p(cv),
              _p(cnt), _stream())
    c = cnt.double()
    return {"mean": round(float(c.mean()), 1), "max": int(cnt.max())}


if __name__ == "__main__":
    main()
