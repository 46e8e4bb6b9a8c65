"""Run under torchrun (N >= 2 GPUs): TFIDF(distributed=True) with n-gram code spaces above 2^24 (the fit all-gathers the ranks'
local vocabularies, DESIGN.md section 5) returns on every rank the frames of the single-GPU matcher: match, self-match and
transform, for (3, 5) clean and (3, 4) raw.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/dist_vocab_check.py"""
import os, sys
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch, torch.distributed as dist
rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"]); world = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
import polyfuzz_b200
from polyfuzz_b200 import engine, synth
to = synth.titles(6001, seed=51); frm = synth.titles(1503, seed=52) + ["", "x", "Ünïcødé Çafé", to[3]]
ok = True
for rng, clean in (((3, 5), True), ((3, 4), False)):
    kw = dict(n_gram_range=rng, clean_string=clean, min_similarity=0.0, top_n=5)
    for args in ((frm, to), (to[:2500],)):
        d = polyfuzz_b200.TFIDF(distributed=True, **kw); s = polyfuzz_b200.TFIDF(**kw)
        fd, fs = d.match(*args), s.match(*args)
        large = d.vectorizer.code_space() > engine.DENSE_CODE_SPACE_MAX
        same = large and fd.equals(fs)
        print(f"rank {rank}/{world} {rng} clean={clean} lists={len(args)} code_space={d.vectorizer.code_space()} "
              f"identical_to_single_gpu={same}", flush=True)
        ok = ok and same
        if len(args) == 2:                                    # transform against the kept shard index
            td = d.match(frm[:300] + ["zz", to[7]], to, re_train=False)
            ts = s.match(frm[:300] + ["zz", to[7]], to, re_train=False)
            print(f"rank {rank} {rng} clean={clean} transform identical={td.equals(ts)}", flush=True)
            ok = ok and td.equals(ts)
flag = torch.tensor([int(ok)], device="cuda"); dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print("DIST_VOCAB_CHECK", "PASS" if int(flag.item()) == 1 else "FAIL", flush=True)
dist.destroy_process_group()
