"""Developer tool: the device cost of the multi-GPU TF-IDF fit for code spaces above 2^24 (DESIGN.md section 5), emulated on
one GPU without NCCL.  100 000 synthetic company names at n_gram_range (3, 5), clean: the single-GPU fit against G = 8 shards,
each shard's local phase (stage A + gather + sort + run-length of its distinct codes), then what every rank runs on the
gathered buffer (the union sort + run-length) and one rank's df scatter.  The emulated global vocabulary and the summed df are
checked against the single-GPU fit.

    python tools/dist_vocab_time.py [--n 100000] [--shards 8] [--runs 11] [--warmup 2] [--json OUT]

Every time is the median over --runs of CUDA events around the phase, after --warmup.  The collectives are not run: the bytes
they would move are reported instead.  Multi-GPU wall time is not measured by this tool."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        return r.stdout.strip() or r.stderr.strip()
    except OSError as e:
        return f"nvidia-smi not available: {e}"


def timed(fn, runs, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ts, out = [], None
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--runs", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dist_vocab_time.py needs a CUDA device")
    from polyfuzz_b200 import _lib, engine, synth
    from polyfuzz_b200.distributed import shard_bounds
    from polyfuzz_b200.engine import _p, _pow2, _sorted_unique, _stream, _vocab_of_rows

    names = synth.company_names(args.n)
    G, dev = args.shards, torch.device("cuda", torch.cuda.current_device())
    res = {"card": card(), "device": torch.cuda.get_device_name(), "n": args.n, "n_gram_range": [3, 5], "clean": True,
           "shards": G, "runs": args.runs, "warmup": args.warmup}

    # single GPU: the whole fit (stage A, vocabulary, idf, the stats read) and its vocabulary step alone
    v = engine.NgramTfidf((3, 5), True, True)
    assert v.code_space() > engine.DENSE_CODE_SPACE_MAX
    S = v.stage(names)
    res["single_fit_ms"], _ = timed(lambda: v.fit_staged([S]), args.runs, args.warmup)
    rows = v._stage_a(S, None, fit=True)
    nv = torch.zeros(1, dtype=torch.int32, device=dev)
    res["single_vocab_ms"], _ = timed(lambda: _vocab_of_rows([rows], nv), args.runs, args.warmup)
    V = v.n_vocab

    # each shard's local phase
    shards = []
    for r in range(G):
        lo, hi = shard_bounds(len(names), G, r)
        St = v.stage(names[lo:hi])
        loc_nv = torch.zeros(1, dtype=torch.int32, device=dev)

        def local(St=St, loc_nv=loc_nv):
            return _vocab_of_rows([v._stage_a(St, None, fit=True)], loc_nv)
        ms, (keys, df) = timed(local, args.runs, args.warmup)
        shards.append((ms, keys, df, loc_nv, int(loc_nv.item())))
    lens = [s[4] for s in shards]
    L = max(max(lens), 1)
    gathered = torch.full((G, L), -1, dtype=torch.int64, device=dev)
    for r, (_, keys, _, _, n) in enumerate(shards):
        gathered[r, :n] = keys[:n]
    n_keys = sum(lens)
    d_n = torch.tensor([n_keys], dtype=torch.int64, device=dev)
    g_nv = torch.zeros(1, dtype=torch.int32, device=dev)

    # every rank: the union sort + run-length of the gathered buffer
    def union():
        keys = torch.full((_pow2(gathered.numel()),), -1, dtype=torch.int64, device=dev)
        keys[:gathered.numel()] = gathered.reshape(-1)
        return _sorted_unique(keys, d_n, max(n_keys, 1), g_nv)
    res["union_sort_ms"], (g_vocab, _) = timed(union, args.runs, args.warmup)
    Vg = int(g_nv.item())

    # one rank's df scatter (rank 0), and the df the all-reduce would produce
    def scatter(r):
        _, keys, df, loc_nv, _ = shards[r]
        out = torch.zeros(Vg, dtype=torch.int32, device=dev)
        _lib.call("pfz_df_scatter", _p(keys), _p(df), _p(loc_nv), int(keys.numel()), _p(g_vocab), Vg, _p(out), _stream())
        return out
    res["df_scatter_ms"], _ = timed(lambda: scatter(0), args.runs, args.warmup)
    df_sum = torch.stack([scatter(r) for r in range(G)]).sum(0)
    same = (Vg == V and np.array_equal(g_vocab[:Vg].cpu().numpy().view(np.uint64), v.vocab_keys)
            and np.array_equal(df_sum.cpu().numpy(), v.df))

    res.update({"V": V, "sum_V_r": n_keys, "max_V_r": L, "shard_local_ms": [round(s[0], 3) for s in shards],
                "shard_local_max_ms": round(max(s[0] for s in shards), 3),
                "allgather_bytes_per_rank": G * L * 8, "allreduce_bytes": V * 4, "identical_to_single_gpu": bool(same),
                "multi_gpu_wall_time": "not measured"})
    for k in ("single_fit_ms", "single_vocab_ms", "union_sort_ms", "df_scatter_ms"):
        res[k] = round(res[k], 3)
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    if not same:
        raise SystemExit("the emulated sharded vocabulary / df differ from the single-GPU fit")


if __name__ == "__main__":
    main()
