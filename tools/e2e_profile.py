"""Developer tool: wall-clock breakdown of TFIDF.match (host + device) on the 100k company-names workload."""
import sys, os, time
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np, torch
import polyfuzz_b200
from polyfuzz_b200 import datasets, engine
from polyfuzz_b200.matchers import _utils as U
names, _ = datasets.load_company_names(100_000)
def sync(): torch.cuda.synchronize()
for rep in range(5):
    T = {}
    t0 = time.perf_counter()
    vec = engine.NgramTfidf((3, 3), True, True)
    S = vec.stage(names); sync(); t1 = time.perf_counter(); T["stage(pack+H2D)"] = t1 - t0
    (rows,) = vec.fit_staged([S]); sync(); t2 = time.perf_counter(); T["fit"] = t2 - t1
    csr = vec.emit(rows); sync(); t3 = time.perf_counter(); T["emit"] = t3 - t2
    ix = engine.index_for(csr, vec); sync(); t4 = time.perf_counter(); T["index"] = t4 - t3
    oi, ov = engine.spcos_topk(csr, ix, 10, 0.0, self_match=True); sync(); t5 = time.perf_counter(); T["K2 " + ix.variant] = t5 - t4
    fa = U.arrow_from_staged(S); t6 = time.perf_counter(); T["from arrow"] = t6 - t5
    df = U.assemble_matches_device(fa, S.d_blob, S.d_off, oi, ov); t7 = time.perf_counter(); T["tail K5 + D2H + wrap"] = t7 - t6
    t9 = time.perf_counter(); m = polyfuzz_b200.TFIDF(min_similarity=0, top_n=10); d2 = m.match(names); t10 = time.perf_counter()
    if rep >= 2:
        print(" | ".join(f"{k} {v*1e3:.2f}" for k, v in T.items()), f"| sum {1e3*(t7-t0):.1f} | match() {1e3*(t10-t9):.1f} ms", flush=True)
# inside the tail
import ctypes
from polyfuzz_b200 import _lib
from polyfuzz_b200.engine import _p, _stream, _ws
n, k = oi.shape
for rep in range(3):
    sync(); a = time.perf_counter()
    sims = torch.empty(k * n, dtype=torch.float64, device="cuda"); pos = torch.empty(k * n + 1, dtype=torch.int64, device="cuda")
    bitmap = torch.empty(k * ((n + 31) // 32), dtype=torch.int32, device="cuda"); ws = _ws(_lib.load().pfz_frame_tail_ws_bytes(k * n))
    _lib.call("pfz_frame_tail_count", _p(oi.contiguous()), _p(ov.contiguous()), n, k, _p(S.d_off), _p(sims), _p(pos), _p(bitmap), _p(ws),
              ws.numel(), _stream())
    total = int(pos[-1].item()); b = time.perf_counter()
    offsets = torch.empty(k * (n + 1), dtype=torch.int64, device="cuda"); data = torch.empty(max(total, 1), dtype=torch.uint8, device="cuda")
    _lib.call("pfz_frame_tail_copy", _p(oi.contiguous()), n, k, _p(S.d_blob), _p(S.d_off), _p(pos), _p(offsets), _p(data), _stream()); sync(); c = time.perf_counter()
    parts = [sims.view(torch.uint8), offsets.view(torch.uint8), bitmap.view(torch.uint8), data[:total]]
    cat = torch.cat(parts); sync(); d = time.perf_counter()
    host = cat.cpu(); e = time.perf_counter()
    hn = host.numpy(); f = time.perf_counter()
    print(f"tail: count+scan+sync {1e3*(b-a):.2f} | copy kernel {1e3*(c-b):.2f} | cat {1e3*(d-c):.2f} | D2H {host.numel()/1e6:.1f} MB {1e3*(e-d):.2f} | numpy {1e3*(f-e):.2f}", flush=True)
