"""Developer tool: time K6 with a FastText model (pfz_wv_lookup + pfz_ft_pool) on the GPU, and the reference's _embed on the
CPU.

    python tools/fasttext_time.py [--keys 1000000] [--d 300] [--bucket 2000000] [--unknown 0,0.3,1] [--rounds 12] [--warmup 3]
                                  [--ref-sample 5000] [--check-sample 2000] [--out FILE]

Workload: the 100 000 company names; a seeded stand-in vocabulary the shape of a FastText model (--keys x --d float32) built
so that a set fraction of the names' distinct space-split tokens is unknown (each --unknown value in turn), padded with
filler keys; a seeded --bucket x --d float32 n-gram table at (min_n, max_n) = (3, 6).  For each fraction, in one process:
  - lookup + pool launches between CUDA events (strings already on the device), median of --rounds after --warmup;
  - algorithmic bytes: known token rows x d x 4 + (sum over unknown tokens of their n-grams) x d x 4 gathered, n x d x 8
    written, over that time against 3.35 TB/s;
  - the device rows of the first --check-sample names against the restatement (tests/fasttext_oracle.py), bit for bit;
  - the reference's _embed (oracle/_ref, gensim stubbed, the FastText stand-in whose get_vector is gensim 4's) on
    --ref-sample names, one thread, extrapolated to 100 000 names.
The card's name, power limit and SM clocks are read with nvidia-smi in the same run."""
import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ[_v] = "1"
import argparse
import json
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from polyfuzz_b200 import _lib, wordvec
from polyfuzz_b200.datasets import load_company_names
from polyfuzz_b200.engine import _p, _stream, _to_dev, _ws
from polyfuzz_b200.strings import pack_strings
import fasttext_oracle as fo
import gensim_oracle as go

HBM_BPS = 3.35e12
MIN_N, MAX_N = 3, 6


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def event_ms(fn, rounds, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(rounds):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def n_ngrams(length, min_n, max_n):
    """How many n-grams gensim takes from a word of `length` characters (fasttext_oracle.ngrams, counted)."""
    lc = length + 2
    c = sum(max(0, lc - n + 1) for n in range(max(min_n, 1), max_n + 1))
    return c - (2 if min_n <= 1 <= max_n else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=300)
    ap.add_argument("--bucket", type=int, default=2_000_000)
    ap.add_argument("--unknown", default="0,0.3,1")
    ap.add_argument("--rounds", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-sample", type=int, default=5000)
    ap.add_argument("--check-sample", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info()}
    names, src = load_company_names()
    n = len(names)
    tokens = list(dict.fromkeys(t for s in names for t in s.split(" ")))
    rng = np.random.default_rng(0)
    V = rng.standard_normal((a.keys, a.d), dtype=np.float32)
    NG = rng.standard_normal((a.bucket, a.d), dtype=np.float32)
    order = rng.permutation(len(tokens))
    res["workload"] = dict(names=n, source=src, distinct_tokens=len(tokens), keys=a.keys, d=a.d, bucket=a.bucket, min_n=MIN_N,
                           max_n=MAX_N)
    torch.cuda.init(); torch.zeros(1, device="cuda")

    blob, off, _ = pack_strings(names)
    d_blob = _to_dev(blob).to(torch.int32) if blob.dtype == np.uint8 else _to_dev(blob.view(np.int32), torch.int32)
    d_off = _to_dev(off)
    tok_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    tok_row = torch.empty(int(off[-1]) + n, dtype=torch.int32, device="cuda")
    ws_bytes = int(_lib.load().pfz_wv_lookup_ws_bytes(n)); ws = _ws(ws_bytes)
    out = torch.empty((n, a.d), dtype=torch.float64, device="cuda")

    ref = os.path.join(ROOT, "oracle", "_ref")
    RefGensim = None
    if a.ref_sample and os.path.isdir(os.path.join(ref, "polyfuzz")):
        go.install_gensim(ref)
        from polyfuzz.models._gensim import GensimEmbeddings as RefGensim

    runs = []
    for frac in [float(f) for f in a.unknown.split(",")]:
        held = {tokens[i] for i in order[:int(round(frac * len(tokens)))]}
        keys = [t for t in tokens if t not in held][:a.keys]
        keys += [f"\x00filler{i}" for i in range(a.keys - len(keys))]
        k2i = {k: i for i, k in enumerate(keys)}
        wv = wordvec.WordVectors(k2i, V, vectors_ngrams=NG, min_n=MIN_N, max_n=MAX_N, bucket=a.bucket)

        def step():
            _lib.call("pfz_wv_lookup", _p(d_blob), _p(d_off), n, _p(wv.key_blob), _p(wv.key_off), _p(wv.key_row), _p(wv.table),
                      wv.cap, _p(tok_off), _p(tok_row), _p(ws), ws_bytes, _stream())
            _lib.call("pfz_ft_pool", _p(d_blob), _p(d_off), n, _p(tok_off), _p(tok_row), _p(wv.vectors), _p(wv.vectors_ngrams), a.d,
                      a.bucket, MIN_N, MAX_N, _p(out), a.d, _stream())
        med, lo, hi = event_ms(step, a.rounds, a.warmup)
        occ = [t for s in names for t in s.split(" ")]
        unknown = [t for t in occ if t not in k2i]
        grams = sum(n_ngrams(len(t), MIN_N, MAX_N) for t in unknown)
        nbytes = (len(occ) - len(unknown)) * a.d * 4 + grams * a.d * 4 + n * a.d * 8
        r = dict(unknown_fraction_of_distinct=frac, tokens=len(occ), tokens_unknown=len(unknown), ngrams_gathered=grams,
                 lookup_pool_ms_median=med, lookup_pool_ms_min=lo, lookup_pool_ms_max=hi, algorithmic_bytes=nbytes,
                 bytes_per_s=nbytes / (med * 1e-3), share_of_hbm=nbytes / (med * 1e-3) / HBM_BPS)
        assert int(tok_off[-1]) == len(occ)
        E = out.cpu().numpy()
        ft = fo.FastTextKeyedVectors(keys, V, NG, MIN_N, MAX_N, a.bucket, k2i)
        cs = names[:a.check_sample]
        r["check_sample"] = len(cs)
        r["bit_equal_to_restatement"] = bool(np.array_equal(go.bits(E[:len(cs)]), go.bits(fo.embed(ft, cs))))
        if RefGensim is not None:
            sample = names[:a.ref_sample]
            t0 = time.perf_counter(); R = np.asarray(RefGensim(ft)._embed(sample), np.float64); t = time.perf_counter() - t0
            r["reference_embed"] = dict(sample=len(sample), seconds=t, extrapolated_s_per_100k=t * 100_000 / len(sample),
                                        bit_equal_to_device=bool(np.array_equal(go.bits(R), go.bits(E[:len(sample)]))))
        runs.append(r)
        print(json.dumps(r), flush=True)
        del wv
        torch.cuda.empty_cache()
    res["runs"] = runs
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
