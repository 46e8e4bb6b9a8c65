"""Developer tool: time single linkage on the device (K7) against the reference's single_linkage.

    python tools/linkage_time.py [--rounds 20] [--warmup 3] [--thr 0.75] [--out FILE]

Workloads, each at threshold --thr:
  - company_100k: the TF-IDF (3-gram) self-match top-1 of the 100 000 company names;
  - company_1m: the same for 1 000 000 synthetic company names (polyfuzz_b200.synth);
  - uniform_100k / uniform_1m: unique From strings, To drawn at random from them, Similarity uniform in [0, 1).
For each, in one process:
  - the K7 launches alone (pfz_linkage on key ids already on the device) between CUDA events, median of --rounds after --warmup;
  - polyfuzz_b200.single_linkage end to end (filter, factorize, H2D, K7, D2H, the three dicts), host clock, median;
  - the reference's single_linkage (oracle/_ref) once, host clock, and whether its three dicts equal the device's in content
    and order;
  - the rounds the parallel rule needs (tests/linkage_model.py); above 12 the finish kernel decides the rest.
The card's name, power limit and SM clocks are read with nvidia-smi in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import pandas as pd
import torch

import linkage_model as lm
from polyfuzz_b200 import TFIDF, _lib, single_linkage, synth
from polyfuzz_b200.datasets import load_company_names
from polyfuzz_b200.engine import _p, _stream, _to_dev, _ws


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def uniform_frame(n, seed):
    rng = np.random.default_rng(seed)
    names = np.array([f"name {i:07d}" for i in range(n)], dtype=object)
    return pd.DataFrame({"From": names, "To": names[rng.integers(0, n, n)], "Similarity": rng.random(n)})


def kernel_ms(frame, thr, rounds, warmup):
    kept = frame.loc[frame.Similarity > thr, :]
    n = len(kept)
    codes, uniques = pd.factorize(pd.concat([kept["From"], kept["To"]], ignore_index=True))
    K = len(uniques)
    dF, dT = _to_dev(codes[:n].astype(np.int32)), _to_dev(codes[n:].astype(np.int32))
    out = torch.empty((4, K), dtype=torch.int32, device="cuda")
    nw = torch.empty(1, dtype=torch.int32, device="cuda")
    ws_bytes = int(_lib.load().pfz_linkage_ws_bytes(n, K))
    ws = _ws(ws_bytes)

    def run():
        _lib.call("pfz_linkage", _p(dF), _p(dT), n, _p(None), 0.0, K, _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]), _p(nw),
                  _p(ws), ws_bytes, _stream())
    for _ in range(warmup):
        run()
    ts = []
    for _ in range(rounds):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); run(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    launches0 = _lib.launch_count(); run(); torch.cuda.synchronize()
    return float(np.median(ts)), n, K, _lib.launch_count() - launches0, ws_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--thr", type=float, default=0.75)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.init()
    res = {"gpu_before": gpu_info(), "threshold": a.thr, "workloads": {}}
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    ref_shim.install()
    from polyfuzz.linkage import single_linkage as ref_linkage

    names, src = load_company_names()
    work = {}
    tf = TFIDF(n_gram_range=(3, 3), min_similarity=0)
    work["company_100k"] = tf.match(names)
    work["company_1m"] = tf.match(synth.company_names(1_000_000, seed=1))
    work["uniform_100k"] = uniform_frame(100_000, 2)
    work["uniform_1m"] = uniform_frame(1_000_000, 3)
    for name, frame in work.items():
        kms, n, K, launches, ws_bytes = kernel_ms(frame, a.thr, a.rounds, a.warmup)
        single_linkage(frame, a.thr)
        ts = []
        for _ in range(max(3, a.rounds // 4)):
            torch.cuda.synchronize(); t0 = time.perf_counter(); dev = single_linkage(frame, a.thr); ts.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); want = ref_linkage(frame, a.thr); tref = time.perf_counter() - t0
        r = dict(rows=len(frame), kept_rows=n, keys=K, clusters=len(want[0]), kernel_ms=kms, launches=launches, ws_mb=ws_bytes / 2**20,
                 device_single_linkage_ms=float(np.median(ts)) * 1e3, reference_single_linkage_ms=tref * 1e3,
                 equal_to_reference=lm.as_lists(dev) == lm.as_lists(want), rounds=lm.rounds_of(frame, a.thr))
        res["workloads"][name] = r
        print(name, json.dumps(r), flush=True)
    res["company_names_source"] = src
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
