"""Run under torchrun (N >= 2 GPUs): TFIDF(distributed=True).match on every rank must equal the single-GPU result.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/dist_check.py"""
import os, sys
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch, torch.distributed as dist
rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
import polyfuzz_b200
from polyfuzz_b200 import synth
to = synth.company_names(7001, seed=5); frm = synth.company_names(1503, seed=6)
ok = True
for kw in (dict(a=(frm, to)), dict(a=(to[:3000],)), dict(a=(to,), from_block=(1000, 2200))):
    args = kw.pop("a")
    d = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=7, distributed=True).match(*args, **kw)
    s = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=7, distributed=False).match(*args, **kw)
    same = d.equals(s)
    ok = ok and same
    print(f"rank {rank}/{world} case {list(kw) or 'plain'} n_from={len(d)} identical_to_single_gpu={same}", flush=True)
# fit / transform with the sharded index kept on every rank
m = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=3, distributed=True); m.match(frm, to)
t1 = m.match(frm[:200], to, re_train=False)
m2 = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=3); m2.match(frm, to)
t2 = m2.match(frm[:200], to, re_train=False)
print(f"rank {rank} transform identical={t1.equals(t2)}", flush=True)
ok = ok and t1.equals(t2)
# top_n > 32 across shards, and the edit-distance / embedding matchers sharded the same way
d = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=40, distributed=True).match(frm[:300], to)
s1 = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=40).match(frm[:300], to)
print(f"rank {rank} top_n=40 identical={d.equals(s1)}", flush=True); ok = ok and d.equals(s1)
from polyfuzz_b200 import RapidFuzz, EditDistance, Embeddings
for cls, kw in ((RapidFuzz, dict(scorer="ratio")), (RapidFuzz, dict(scorer="levenshtein", score_cutoff=0.5)), (EditDistance, dict(scorer="ratio"))):
    for args in ((frm[:400], to), (to[:900],)):
        d = cls(distributed=True, **kw).match(*args); s1 = cls(**kw).match(*args)
        print(f"rank {rank} {cls.__name__} {kw} lists={len(args)} identical={d.equals(s1)}", flush=True); ok = ok and d.equals(s1)
import numpy as np
rng = np.random.default_rng(3); ef = rng.standard_normal((700, 96)).astype(np.float32); et = rng.standard_normal((5000, 96)).astype(np.float32)
fl = [f"f{i}" for i in range(700)]; tl = [f"t{i}" for i in range(5000)]
for args, kw in (((fl, tl), dict(embeddings_from=ef, embeddings_to=et)), ((tl,), dict(embeddings_from=et))):
    d = Embeddings(min_similarity=0.0, top_n=5, distributed=True).match(*args, **kw); s1 = Embeddings(min_similarity=0.0, top_n=5).match(*args, **kw)
    print(f"rank {rank} Embeddings lists={len(args)} identical={d.equals(s1)}", flush=True); ok = ok and d.equals(s1)
    d = Embeddings(min_similarity=0.0, top_n=5, distributed=True, precision="fp64").match(*args, **kw); s1 = Embeddings(min_similarity=0.0, top_n=5, precision="fp64").match(*args, **kw)
    print(f"rank {rank} Embeddings fp64 lists={len(args)} identical={d.equals(s1)}", flush=True); ok = ok and d.equals(s1)
    # top_n > 32 on each shard (DESIGN.md 4.7), merged by merge_topk_any; like this whole script it needs two GPUs
    d = Embeddings(min_similarity=0.0, top_n=50, distributed=True, precision="fp64").match(*args, **kw); s1 = Embeddings(min_similarity=0.0, top_n=50, precision="fp64").match(*args, **kw)
    print(f"rank {rank} Embeddings fp64 top_n=50 lists={len(args)} identical={d.equals(s1)}", flush=True); ok = ok and d.equals(s1)
flag = torch.tensor([int(ok)], device="cuda"); dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print("DIST_CHECK", "PASS" if int(flag.item()) == 1 else "FAIL", flush=True)
dist.destroy_process_group()
