"""Developer tool: where the time of one headline step goes (100k company names self-match, TF-IDF top-10, one GPU).

    python tools/k2_breakdown.py [--lib PATH] [--timing-lib PATH] [--steps 5] [--warmup 3] [--out DIR]

Runs the bench.py step (K1 + index + K2, the L2 flushed before every step, `--warmup` untimed steps first) and reports
  * the card: name, power limit, current and maximum SM clock;
  * the step time from CUDA events (profiler off);
  * per-kernel device times from torch.profiler, in a run of its own (summed over the profiled steps, divided by --steps);
  * the candidates the block kernel's filter left per from-row for exact re-scoring (its `gcnt` array): mean and maximum,
    to set against tools/k2_cand_count.py (the numbers differ somewhat: fixed point and group order);
  * with --timing-lib (a library built with PFZ_NVCC_EXTRA=-DPFZ_B3_TIMING), the block kernel's per-phase split of SM
    cycles, measured in a subprocess that loads that library.
--lib loads another build of libpfz.so instead of the package's (A/B of two builds in one session); entry points that build
does not have are left out.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libpfz.so to load instead of the package's")
    ap.add_argument("--timing-lib", default=None, help="library built with -DPFZ_B3_TIMING: adds the per-phase split")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the profiler table and the JSON record")
    ap.add_argument("--phases", action="store_true", help=argparse.SUPPRESS)   # subprocess mode: per-phase split only
    return ap.parse_args()


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:  # noqa: BLE001 -- the record says why it is missing
        return {"error": repr(e)}


def setup(args):
    from polyfuzz_b200 import _lib
    if args.lib:
        _lib._LIB_PATH = os.path.abspath(args.lib)
        other = ctypes.CDLL(_lib._LIB_PATH)
        for name in [n for n in _lib._PROTOS if not hasattr(other, n)]:
            del _lib._PROTOS[name]
    import torch
    from polyfuzz_b200 import datasets, engine
    from polyfuzz_b200.distributed import tfidf_topk_sharded
    if not torch.cuda.is_available():
        raise SystemExit("k2_breakdown needs a CUDA device")
    torch.cuda.set_device(0)
    names, kind = datasets.load_company_names(100_000, seed=0)
    staged = engine.NgramTfidf((3, 3), True, True).stage(names)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    out = {}

    def step():
        vec = engine.NgramTfidf((3, 3), True, True)
        out["r"] = tfidf_topk_sharded(vec, staged, staged, 0, 10, 0.0, self_match=True, from_index_base=0, fit=True,
                                      fit_on_from=False, comm=None, n_docs_total=len(names))
    return torch, step, flush, kind, out


def candidate_counts(torch, step, flush):
    """gcnt of one step: the block kernel's workspace is kept while the call runs and read back afterwards."""
    from polyfuzz_b200 import _lib, engine
    lib = _lib.load()
    orig_block, orig_ws = engine._spcos_block, engine._ws
    seen = []

    def block(a, index, k, *rest):
        kept = []
        engine._ws = lambda nbytes: kept.append(orig_ws(nbytes)) or kept[-1]
        try:
            r = orig_block(a, index, k, *rest)
        finally:
            engine._ws = orig_ws
        n_from, n_splits = a.n_rows, rest[-1]
        shape = (n_from, int(a.indices.numel()), index.n_vocab, n_splits)
        if hasattr(lib, "pfz_spcos_block_gcnt_offset"):
            off = lib.pfz_spcos_block_gcnt_offset(*shape)
        else:                          # older builds: gcnt, then 192 candidate slots per entry, end the workspace
            a256 = lambda x: (x + 255) // 256 * 256  # noqa: E731
            off = lib.pfz_spcos_block_ws_bytes(*shape) - a256(n_splits * n_from * 192 * 4) - a256(n_splits * n_from * 4)
        seen.append((kept[0], off, n_splits * n_from))
        return r

    engine._spcos_block = block
    try:
        flush.zero_(); step()
        torch.cuda.synchronize()
    finally:
        engine._spcos_block = orig_block
    g = torch.cat([ws[off:off + 4 * n].view(torch.int32).to(torch.int64) for ws, off, n in seen])
    return {"rows": int(g.numel()), "mean": round(float(g.double().mean()), 3), "max": int(g.max())}


def run_phases(args):
    torch, step, flush, _kind, _ = setup(args)
    from polyfuzz_b200 import _lib, engine
    lib = _lib.load()
    lib.pfz_debug_b3_cycles.argtypes = [ctypes.c_void_p, ctypes.c_int32]
    c = (ctypes.c_ulonglong * 8)()
    for _ in range(args.warmup):
        flush.zero_(); step()
    torch.cuda.synchronize()
    lib.pfz_debug_b3_cycles(c, 1)
    for _ in range(args.steps):
        flush.zero_(); step()
    torch.cuda.synchronize()
    lib.pfz_debug_b3_cycles(c, 1)
    x = [float(v) for v in c]
    labels = ["table", "wait A", "items", "wait B", "scan (+prologue)", "exact at block end", "wait block end", "-"]
    tot = sum(x) or 1.0
    print(json.dumps({"phases": {k: {"share": v / tot, "gcycles_per_step": v / args.steps / 1e9} for k, v in zip(labels, x) if k != "-"},
                      "block_rows": engine.BLOCK_ROWS}))


def main():
    args = parse()
    if args.phases:
        return run_phases(args)
    torch, step, flush, kind, out = setup(args)
    from polyfuzz_b200 import engine
    rec = {"card": card(), "data": kind, "lib": args.lib or "package", "block_rows": engine.BLOCK_ROWS}
    for _ in range(args.warmup):
        flush.zero_(); step()
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.steps):
        flush.zero_(); torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); step(); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    rec["step_ms"] = [round(v, 3) for v in ms]
    rec["tile"] = out["r"][3].tile
    rec["gcnt"] = candidate_counts(torch, step, flush)
    print(f"candidates left for exact re-scoring per from-row (gcnt): mean {rec['gcnt']['mean']}, max {rec['gcnt']['max']}")
    # per-kernel device times: a run of its own, the profiler on
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            flush.zero_(); step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            per[ev.key] = (t / 1e3 / args.steps, ev.count // args.steps)
    top = sorted(per.items(), key=lambda kv: -kv[1][0])
    rec["kernels_ms_per_step"] = {k[:90]: round(v[0], 4) for k, v in top[:25]}
    rec["card_after"] = card()
    print(f"card: {rec['card']}  data: {kind}  tile {rec['tile']}  rows {rec['block_rows']}")
    print(f"step ms (events, profiler off): {rec['step_ms']}")
    for k, (t, n) in top[:25]:
        print(f"  {t:8.3f} ms  x{n:<4d} {k[:110]}")
    if args.timing_lib:
        cmd = [sys.executable, os.path.abspath(__file__), "--phases", "--lib", args.timing_lib, "--steps", str(args.steps), "--warmup", str(args.warmup)]
        r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ))
        line = [l for l in r.stdout.splitlines() if l.startswith("{")]
        rec["phases"] = json.loads(line[-1])["phases"] if line else {"error": r.stderr[-2000:]}
        if line:
            for k, v in rec["phases"].items():
                print(f"  phase {k:20s} {100 * v['share']:5.1f} %  {v['gcycles_per_step']:.3f} G warp-cycles per step")
        else:
            print("phase split failed:\n" + r.stderr[-2000:])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "k2_breakdown.json"), "a") as f:
            f.write(json.dumps(rec) + "\n")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
