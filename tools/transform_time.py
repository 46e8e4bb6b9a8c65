"""Developer tool: the cost of PolyFuzz's fit / transform path for RapidFuzz (WRatio, K3b) and RapidFuzz(scorer="ratio") (K3) on
the real movie titles: a fit on Netflix titles against IMDB (80 852), then transform calls of 100 and 1 000 new Netflix
titles, re-staging the to-list on every call (re_train=True) or scoring against the kept to-side (re_train=False, what
PolyFuzz.transform passes); and one full Netflix x IMDB WRatio match with its to-side staging timed apart.

    python tools/transform_time.py [--runs 11] [--warmup 2] [--parent DIR] [--json OUT]

Each time is a host clock around one call that ends in a device synchronise; the median of --runs calls after --warmup is
reported.  --parent DIR times the same full WRatio match with the polyfuzz_b200 package under DIR (an earlier build) in a
subprocess of the same session, and checks that both builds return the same indices and scores."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

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
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    return ts[len(ts) // 2] * 1e3, out


def full_match(root, runs, warmup, out_path):
    """The full Netflix x IMDB WRatio fuzz_argbest with the package under root; saves the result to out_path."""
    sys.path.insert(0, root)
    import numpy as np
    from polyfuzz_b200 import datasets, fuzzy
    titles, _ = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    ms, (idx, score) = timed(lambda: fuzzy.fuzz_argbest(frm, to, "WRatio"), runs, warmup)
    np.savez(out_path, idx=idx.cpu().numpy(), score=score.cpu().numpy())
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--json", default=None)
    ap.add_argument("--full-only", default=None, help=argparse.SUPPRESS)     # subprocess mode: root,out.npz
    args = ap.parse_args()
    if args.full_only:
        root, out = args.full_only.split(",")
        print(json.dumps({"full_ms": full_match(root, args.runs, args.warmup, out)}))
        return
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("transform_time.py needs a CUDA device")
    from polyfuzz_b200 import RapidFuzz, datasets, editdist, fuzzy

    titles, kind = datasets.load_movie_titles()
    netflix, imdb = titles["Netflix"], titles["IMDB"]
    res = {"card": card(), "data": kind, "n_to": len(imdb), "runs": args.runs, "warmup": args.warmup, "transform": {}}
    fit_list = netflix[:1000]
    for scorer in ("WRatio", "ratio"):
        m = RapidFuzz(scorer=scorer)
        m.match(fit_list, imdb)                                  # the fit keeps IMDB's staged to-side
        for n_new in (100, 1000):
            new = netflix[1000:1000 + n_new]
            restage_ms, a = timed(lambda: m.match(new, imdb), args.runs, args.warmup)
            kept_ms, b = timed(lambda: m.match(new, imdb, re_train=False), args.runs, args.warmup)
            assert a.equals(b), f"{scorer}: the kept to-side changed the frame"
            res["transform"][f"{scorer} x{n_new}"] = {"restage_ms": round(restage_ms, 2), "kept_ms": round(kept_ms, 2),
                                                     "speedup": round(restage_ms / kept_ms, 1)}
            print(scorer, n_new, res["transform"][f"{scorer} x{n_new}"], flush=True)

    # one full Netflix x IMDB WRatio match: the whole call, the to-side staging alone, and the rest (from-side staging,
    # vocabulary join, kernels) against a kept to-side
    stage_ms, _ = timed(lambda: fuzzy.FuzzTargets(imdb), args.runs, args.warmup)
    kept = editdist.KeptTargets()
    kept.stage(("k3b", 0), imdb, fuzzy.FuzzTargets, False)
    rest_ms, _ = timed(lambda: fuzzy.fuzz_argbest(netflix, imdb, "WRatio", kept=kept, reuse=True), args.runs, args.warmup)
    with tempfile.TemporaryDirectory() as tmp:
        cur = os.path.join(tmp, "cur.npz")
        full_ms = full_match(ROOT, args.runs, args.warmup, cur)
        res["full_wratio"] = {"call_ms": round(full_ms, 1), "to_side_staging_ms": round(stage_ms, 1),
                              "from_staging_and_kernels_ms": round(rest_ms, 1)}
        if args.parent:
            par = os.path.join(tmp, "parent.npz")
            r = subprocess.run([sys.executable, __file__, "--runs", str(args.runs), "--warmup", str(args.warmup), "--full-only",
                                f"{os.path.abspath(args.parent)},{par}"], capture_output=True, text=True, cwd=tmp)
            if r.returncode:
                raise SystemExit("parent run failed:\n" + r.stderr[-3000:])
            res["full_wratio"]["parent_call_ms"] = round(json.loads(r.stdout.strip().splitlines()[-1])["full_ms"], 1)
            a, b = np.load(cur), np.load(par)
            res["full_wratio"]["same_as_parent"] = bool(np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"], b["score"]))
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
