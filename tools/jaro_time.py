"""Developer tool: time the Jaro-Winkler mode of K3 against fuzz.ratio and normalized Levenshtein on the real movie titles
(Netflix 6 172 x IMDB 80 852, per-row best match), and check a 300-row sample of its arg-best against the CPU oracle.

    python tools/jaro_time.py [--runs 15] [--warmup 3] [--sample 300] [--json OUT]

The lists are staged once (EditQueries / EditTargets); each timed call is edit_argbest_staged (to-list packing per alphabet
batch, the kernels, the split merge), bracketed by CUDA events.  The three metrics alternate call by call after warm-up and
the median of --runs calls is reported.  word_steps32 counts (text symbol x 32-bit pattern word) steps the recurrence needs:
every text symbol for Levenshtein / Indel, the first min(n, m + R) for Jaro (later ones have an empty match window)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

METRICS = ("jaro_winkler", "ratio", "norm_lev")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True)
        return r.stdout.strip() or r.stderr.strip()
    except OSError as e:
        return f"nvidia-smi not available: {e}"


def word_steps32(from_lens, to_lens, jaro):
    """Sum over all pairs of (text symbols the recurrence visits) x (32-bit words of the pattern)."""
    w32 = np.where(from_lens <= 32, 1, 2 * np.ceil(from_lens / 64.0))
    if not jaro:
        return float(w32.sum()) * float(to_lens.sum())
    hist = np.bincount(to_lens)
    n = np.arange(len(hist))
    total = 0.0
    for m, cnt in zip(*np.unique(from_lens, return_counts=True)):
        r = np.maximum(0, np.maximum(m, n) // 2 - 1)
        steps = np.minimum(n, m + r) if m > 0 else np.zeros_like(n)
        total += float(cnt) * float((w32[from_lens == m][0]) * (hist * steps).sum())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=300)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("jaro_time.py needs a CUDA device")
    from polyfuzz_b200 import datasets, editdist
    import jaro_oracle

    titles, kind = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    Q = editdist.EditQueries(frm); T = editdist.EditTargets(to)
    pairs = float(len(frm)) * len(to)
    out = {"card": card(), "data": kind, "n_from": len(frm), "n_to": len(to), "pairs": pairs, "runs": args.runs}
    steps = {m: word_steps32(Q.lens, T.lens, m.startswith("jaro")) for m in METRICS}
    for _ in range(args.warmup):
        for m in METRICS:
            editdist.edit_argbest_staged(Q, T, m)
    torch.cuda.synchronize()
    times = {m: [] for m in METRICS}
    for _ in range(args.runs):
        for m in METRICS:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            editdist.edit_argbest_staged(Q, T, m)
            b.record()
            b.synchronize()
            times[m].append(a.elapsed_time(b))
    for m in METRICS:
        t = float(np.median(times[m]))
        out[m] = {"ms": t, "ms_each": [round(x, 3) for x in times[m]], "spread_ms": float(np.max(times[m]) - np.min(times[m])),
                  "pairs_per_s": pairs / (t * 1e-3), "word_steps32": steps[m], "word_steps32_per_s": steps[m] / (t * 1e-3)}
        print(f"{m:13s} median {t:8.3f} ms  (min {min(times[m]):.3f}, max {max(times[m]):.3f})  pairs/s {pairs / (t * 1e-3):.3e}  "
              f"word-steps32/s {steps[m] / (t * 1e-3):.3e}")

    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(frm), min(args.sample, len(frm)), replace=False))
    sub = [frm[i] for i in rows]
    bi, bs, bd = editdist.edit_argbest(sub, to, "jaro_winkler")
    oi, os_, od = jaro_oracle.jaro_argbest(sub, to, "jaro_winkler", n_threads=os.cpu_count() or 1)
    ok = (np.array_equal(bi.cpu().numpy(), oi) and np.array_equal(bs.cpu().numpy(), os_) and np.array_equal(bd.cpu().numpy(), od))
    out["oracle_check"] = {"rows": len(sub), "equal": bool(ok)}
    print(f"card: {out['card']}")
    print(f"oracle check ({len(sub)} rows x {len(to)}, jaro_winkler): {'equal' if ok else 'DIFFERENT'}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
