"""Developer tool: time K4's bf16 row staging (pfz_rows_to_bf16, l2 normalisation + bf16 rounding) on C4-shaped inputs.

    python tools/k4_stage_time.py [--n 100000] [--d 768] [--rounds 7] [--reps 20] [--warmup 5] [--baseline path/to/libpfz.so]

Inputs: the C4 from-side (torch seed 0, N(0, 1) rows, fp32) and the same rows widened to fp64.  Each round times `--reps`
back-to-back launches between two CUDA events; the figure is the median time per launch over `--rounds` rounds.  With
`--baseline`, a second build of the library (for example the parent commit's) is loaded next to this tree's and the two
alternate round by round on the same inputs; the tool also reports how many staged bf16 elements differ between them.  The
card's name, power limit and SM clocks are read with nvidia-smi in the same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np
import torch

from polyfuzz_b200 import _lib


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def stage_fn(lib):
    fn = lib.pfz_rows_to_bf16
    fn.argtypes = _lib._PROTOS["pfz_rows_to_bf16"]
    fn.restype = ctypes.c_int

    def run(x, out):
        n, d = x.shape
        rc = fn(x.data_ptr(), int(x.dtype == torch.float64), x.stride(0), n, d, out.shape[1], 1, out.data_ptr(),
                torch.cuda.current_stream().cuda_stream)
        if rc:
            raise RuntimeError("pfz_rows_to_bf16 failed")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--baseline", default=None, help="another build of libpfz.so to alternate with")
    a = ap.parse_args()
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    libs = {"tree": stage_fn(_lib.load())}
    if a.baseline:
        libs["baseline"] = stage_fn(ctypes.CDLL(os.path.abspath(a.baseline)))
    torch.manual_seed(0)
    X32 = torch.randn(a.n, a.d, device=dev)
    d_pad = max(8, (a.d + 7) // 8 * 8)
    for x in (X32, X32.double()):
        outs = {name: torch.empty((a.n, d_pad), dtype=torch.bfloat16, device=dev) for name in libs}
        for name, run in libs.items():
            for _ in range(a.warmup):
                run(x, outs[name])
        rec = {name: [] for name in libs}
        for _ in range(a.rounds):
            for name, run in libs.items():
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    run(x, outs[name])
                e1.record()
                torch.cuda.synchronize()
                rec[name].append(e0.elapsed_time(e1) / a.reps)
        res = {"dtype": str(x.dtype).replace("torch.", ""), "n": a.n, "d": a.d, "rounds": a.rounds, "reps": a.reps,
               "median_ms": {k: round(float(np.median(v)), 4) for k, v in rec.items()},
               "min_ms": {k: round(float(np.min(v)), 4) for k, v in rec.items()},
               "max_ms": {k: round(float(np.max(v)), 4) for k, v in rec.items()},
               "bytes_read_written": int(x.numel() * x.element_size() + a.n * d_pad * 2)}
        if "baseline" in outs:
            res["elements_differing_from_baseline"] = int((outs["tree"].view(torch.int16) != outs["baseline"].view(torch.int16)).sum())
        print(json.dumps(res), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
