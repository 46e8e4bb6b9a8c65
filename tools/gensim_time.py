"""Developer tool: time GensimEmbeddings on the GPU (K6 pooling, then K4) against Embeddings on the same pooled arrays, and the
reference's _embed on the CPU.

    python tools/gensim_time.py [--keys 1000000] [--d 300] [--rounds 12] [--warmup 3] [--ref-sample 20000] [--out FILE]

Workload: the 100 000 company names and a stand-in vocabulary the shape of fasttext-wiki-news-subwords-300 (1M keys x 300
float32): the names' distinct space-split tokens, less a seeded 10 % held out so that rows take both pooling paths, plus
seeded filler keys.  In one process:
  - the one-off vocabulary staging (pack of the keys, H2D of the vectors, table build), host clock around a synchronise;
  - the lookup (count + scan + lookup) and pool launches between CUDA events, medians of --rounds after --warmup, with the
    pool's algorithmic bytes (sum of tokens x d x 4 gathered + n x d x 8 written) over its time against 3.35 TB/s;
  - GensimEmbeddings.match self-match top-10 end to end in bf16 and fp64, alternating with Embeddings.match on the pooled
    matrix (embeddings_from = embeddings_to), host clock around a synchronise;
  - the reference's _embed (oracle/_ref, gensim stubbed by tests/gensim_oracle.py) on --ref-sample names, one thread,
    extrapolated to 100 000 names, and its output compared with the device rows bit for bit.
The card's name, power limit and SM clocks are read with nvidia-smi in the same run."""
import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ[_v] = "1"
import argparse
import json
import subprocess
import sys
import time
import types

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from polyfuzz_b200 import Embeddings, GensimEmbeddings, _lib, wordvec
from polyfuzz_b200.datasets import load_company_names
from polyfuzz_b200.engine import _p, _stream, _to_dev, _ws
from polyfuzz_b200.strings import pack_strings

HBM_BPS = 3.35e12


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def vocabulary(names, n_keys, d, seed=0):
    rng = np.random.default_rng(seed)
    tokens = list(dict.fromkeys(t for s in names for t in s.split(" ")))
    held = set(rng.choice(len(tokens), size=len(tokens) // 10, replace=False).tolist())
    keys = [t for i, t in enumerate(tokens) if i not in held]
    keys += [f"\x00filler{i}" for i in range(max(0, n_keys - len(keys)))]
    V = rng.standard_normal((len(keys), d), dtype=np.float32)
    return {k: i for i, k in enumerate(keys)}, V, len(tokens) - len(held), len(held)


def event_ms(fn, rounds, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(rounds):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def wall_ms(fn):
    torch.cuda.synchronize(); t0 = time.perf_counter(); out = fn(); torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-sample", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info()}
    names, src = load_company_names()
    k2i, V, n_found_tokens, n_held = vocabulary(names, a.keys, a.d)
    res["workload"] = dict(names=len(names), source=src, keys=len(k2i), d=a.d, name_tokens_in_vocab=n_found_tokens, held_out=n_held)
    torch.cuda.init(); torch.zeros(1, device="cuda")

    # one-off staging
    stage_ms, wv = wall_ms(lambda: wordvec.WordVectors(k2i, V))
    table_ms = event_ms(lambda: _lib.call("pfz_wv_table_build", _p(wv.key_blob), _p(wv.key_off), wv.n_keys, _p(wv.table), wv.cap,
                                          _stream()), a.rounds, 1)
    res["staging"] = dict(total_ms=stage_ms, table_build_ms=table_ms, cap=wv.cap, device_bytes=int(V.nbytes + wv.table.numel() * 4 +
                          wv.key_blob.numel() * 4 + wv.key_off.numel() * 8 + wv.key_row.numel() * 4))

    # lookup and pool launches on strings already on the device
    blob, off, _ = pack_strings(names)
    d_blob = _to_dev(blob).to(torch.int32) if blob.dtype == np.uint8 else _to_dev(blob.view(np.int32), torch.int32)
    d_off = _to_dev(off)
    n = len(names)
    tok_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    tok_row = torch.empty(int(off[-1]) + n, dtype=torch.int32, device="cuda")
    ws_bytes = int(_lib.load().pfz_wv_lookup_ws_bytes(n)); ws = _ws(ws_bytes)
    out = torch.empty((n, a.d), dtype=torch.float64, device="cuda")

    def lookup():
        _lib.call("pfz_wv_lookup", _p(d_blob), _p(d_off), n, _p(wv.key_blob), _p(wv.key_off), _p(wv.key_row), _p(wv.table), wv.cap,
                  _p(tok_off), _p(tok_row), _p(ws), ws_bytes, _stream())

    def pool():
        _lib.call("pfz_wv_pool", _p(wv.vectors), 0, a.d, _p(tok_off), _p(tok_row), n, _p(out), a.d, _stream())
    lookup_ms = event_ms(lookup, a.rounds, a.warmup)
    pool_ms = event_ms(pool, a.rounds, a.warmup)
    n_tok = int(tok_off[-1])
    rows = tok_row[:n_tok]
    miss_rows = int((torch.zeros(n, dtype=torch.int32, device="cuda").index_add_(
        0, torch.repeat_interleave(torch.arange(n, device="cuda"), tok_off.diff()), (rows < 0).int()) > 0).sum())
    pool_bytes = n_tok * a.d * 4 + n * a.d * 8
    res["kernels"] = dict(tokens=n_tok, tokens_missing=int((rows < 0).sum()), rows_fp64_path=miss_rows, lookup_ms=lookup_ms, pool_ms=pool_ms,
                          pool_bytes=pool_bytes, pool_bytes_per_s=pool_bytes / (pool_ms * 1e-3),
                          pool_share_of_hbm=pool_bytes / (pool_ms * 1e-3) / HBM_BPS,
                          pool_call_ms=wall_ms(lambda: wv.pool(names))[0])
    print(json.dumps(res), flush=True)

    # end to end, alternating with Embeddings.match on the same pooled matrix
    kv = types.SimpleNamespace(key_to_index=k2i, index_to_key=list(k2i), vectors=V)
    E = wv.pool(names).cpu().numpy()
    e2e = {}
    for prec in ("bf16", "fp64"):
        g = GensimEmbeddings(kv, min_similarity=0.0, top_n=10, precision=prec)
        e = Embeddings(min_similarity=0.0, top_n=10, precision=prec)
        tg, te = [], []
        for it in range(a.warmup + a.rounds):
            t1, dg = wall_ms(lambda: g.match(names))
            t2, de = wall_ms(lambda: e.match(names, embeddings_from=E, embeddings_to=E))
            if it >= a.warmup:
                tg.append(t1); te.append(t2)
        e2e[prec] = dict(gensim_match_ms=float(np.median(tg)), embeddings_match_ms=float(np.median(te)), frames_equal=bool(dg.equals(de)))
    res["end_to_end_self_match_top10"] = e2e
    print(json.dumps(res), flush=True)

    # the reference's _embed on a sample, one thread
    ref = os.path.join(ROOT, "oracle", "_ref")
    if a.ref_sample and os.path.isdir(os.path.join(ref, "polyfuzz")):
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import gensim_oracle as go
        go.install_gensim(ref)
        from polyfuzz.models._gensim import GensimEmbeddings as RefGensim
        rm = RefGensim(go.KeyedVectorsStandIn(kv.index_to_key, V, k2i))
        sample = names[:a.ref_sample]
        t0 = time.perf_counter(); R = np.asarray(rm._embed(sample), np.float64); t = time.perf_counter() - t0
        res["reference_embed"] = dict(sample=len(sample), seconds=t, extrapolated_s_per_100k=t * 100_000 / len(sample),
                                      bit_equal_to_device=bool(np.array_equal(R.view(np.uint64), E[:len(sample)].view(np.uint64))))
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
