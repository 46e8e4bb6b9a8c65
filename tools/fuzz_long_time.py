"""Developer tool: time K3b (pfz_fuzz_rows, arg-best) on long from-strings, per word class, for WRatio, partial_ratio and
token_set_ratio.

    python tools/fuzz_long_time.py [--runs 10] [--warmup 1] [--n-from 16] [--n-self 128] [--json OUT]

Input: seeded long strings made of movie titles (the c3 fixture, or its synthetic stand-in) joined with spaces until they
reach a length drawn in the class's range: 200..256 code points (4 words), 300..512 (8 words, one CTA per row) and
513..1 000 (16 words).  Each class is scored against the IMDB list (--n-from rows x 80 852) and against itself (--n-self
rows, self-match).  Kernel time: CUDA events recorded on the stream right before and after each pfz_fuzz_rows call (the
host staging of the call runs before the first event, and a short device sleep queued ahead of it keeps the entry point's
own host set-up out of the interval), summed over the call's launches; the median of --runs calls after
--warmup is reported with pairs/s.  The card's name, power limit and SM clocks are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

SCORERS = ("WRatio", "partial_ratio", "token_set_ratio")
CLASSES = ((4, 200, 256), (8, 300, 512), (16, 513, 1000))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True)
        return r.stdout.strip() or r.stderr.strip()
    except OSError as e:
        return f"nvidia-smi not available: {e}"


def long_strings(titles, n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        want = int(rng.integers(lo, hi + 1))
        s = ""
        while len(s) < want:
            s += (" " if s else "") + titles[int(rng.integers(len(titles)))]
        out.append(s[:want].strip())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n-from", type=int, default=16)
    ap.add_argument("--n-self", type=int, default=128)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fuzz_long_time.py needs a CUDA device")
    from polyfuzz_b200 import _lib, datasets, fuzzy

    titles, kind = datasets.load_movie_titles()
    imdb = titles["IMDB"]
    pool = titles["Netflix"] + imdb
    kernel_ms = []

    class Timed:                                            # events around the pfz_fuzz_rows launches of one call
        @staticmethod
        def call(name, *a):
            if name != "pfz_fuzz_rows":
                return _lib.call(name, *a)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(4_000_000)                    # ~2 ms of device work ahead of e0: the call's host set-up
            e0.record()                                     # (counter reset, attributes, occupancy query) ends before e0 fires
            r = _lib.call(name, *a)
            e1.record()
            kernel_ms.append((e0, e1))
            return r

    fuzzy._lib = Timed
    out = {"card_before": card(), "data": kind, "runs": args.runs, "results": []}
    print(f"data: {kind} movie titles")
    for nw, lo, hi in CLASSES:
        frm = long_strings(pool, args.n_from, lo, hi, seed=nw)
        selfl = long_strings(pool, args.n_self, lo, hi, seed=100 + nw)
        assert set(fuzzy.word_class(np.array([len(s) for s in frm + selfl]))) == {nw}
        for against, (a, b, ex) in (("IMDB", (frm, imdb, False)), ("self", (selfl, selfl, True))):
            for scorer in SCORERS:
                times = []
                for r in range(args.warmup + args.runs):
                    kernel_ms.clear()
                    fuzzy.fuzz_argbest(a, b, scorer, exclude_self=ex)
                    torch.cuda.synchronize()
                    if r >= args.warmup:
                        times.append(sum(e0.elapsed_time(e1) for e0, e1 in kernel_ms))
                t = float(np.median(times))
                pairs = len(a) * len(b)
                res = {"n_words": nw, "from_len": [lo, hi], "against": against, "scorer": scorer, "n_from": len(a), "n_to": len(b),
                       "kernel_ms": t, "spread_ms": float(np.max(times) - np.min(times)), "pairs_per_s": pairs / (t / 1e3)}
                out["results"].append(res)
                print(f"{nw:2d} words {against:5s} {scorer:16s} {len(a):5d} x {len(b):6d}  kernel {t:9.3f} ms "
                      f"(spread {res['spread_ms']:.3f})  {res['pairs_per_s']:.3e} pairs/s", flush=True)
    out["card_after"] = card()
    print(f"card (name, power limit, SM clock, max SM clock) before: {out['card_before']}\nafter: {out['card_after']}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
