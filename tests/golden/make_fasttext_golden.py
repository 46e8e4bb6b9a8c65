"""Generate tests/golden/fasttext_c1.npz by running the UNMODIFIED reference's GensimEmbeddings (/root/reference, imported through
oracle/ref_shim.py, with gensim stubbed by tests/gensim_oracle.py) on a FastText stand-in (tests/fasttext_oracle.py) whose
get_vector is gensim 4's.  Re-run:

    python tests/golden/make_fasttext_golden.py

What is recorded: the README lists and the title slice of gensim_c1.npz (its d25 strings); a vocabulary of their tokens less a
seeded 30 % held out, so that unknown tokens take the subword path (the keys and the row each key maps to); the seeds, d,
min_n, max_n and bucket of the float32 tables, which fasttext_oracle.golden_tables regenerates rather than the file storing
them; the reference's _embed of the strings; and its match frames (cosine_method="sklearn", top_n 1..3, min_similarity 0 and
0.75, two lists and self-match).  Regenerating is byte-identical."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
from make_golden import FROM, TO, df_to_json, savez_fixed  # noqa: E402  (also installs the reference's import shim)
import gensim_oracle as go  # noqa: E402
import fasttext_oracle as fo  # noqa: E402

D, MIN_N, MAX_N, BUCKET = 25, 3, 6, 20011
VECTORS_SEED, NGRAMS_SEED = 4100, 4101


def main():
    assert go.install_gensim(), "the gensim stub needs gensim to be absent"
    from polyfuzz.models._gensim import GensimEmbeddings
    strings = np.load(os.path.join(HERE, "gensim_c1.npz"))["d25_strings"].tolist()
    readme = FROM + TO
    assert strings[:len(readme)] == readme
    picked = strings[len(readme):]
    tokens = list(dict.fromkeys(t for s in strings for t in s.split(" ")))
    rng = np.random.default_rng(4099)
    held = set(rng.choice(tokens, size=3 * len(tokens) // 10, replace=False).tolist())
    keys = [t for t in tokens if t not in held]
    perm = rng.permutation(len(keys))
    out = {"keys": np.array(keys), "rows": perm.astype(np.int64), "d": np.int64(D), "min_n": np.int64(MIN_N),
           "max_n": np.int64(MAX_N), "bucket": np.int64(BUCKET), "vectors_seed": np.int64(VECTORS_SEED),
           "ngrams_seed": np.int64(NGRAMS_SEED), "strings": np.array(strings)}
    ft = fo.golden_model(out)
    emb = np.asarray(GensimEmbeddings(ft)._embed(strings), np.float64)
    assert emb.dtype == np.float64 and np.array_equal(go.bits(emb), go.bits(fo.embed(ft, strings)))
    # pooled rows that coincide tie in every cosine: the title slice has none
    assert np.unique(go.bits(emb[len(readme):]), axis=0).shape[0] == len(picked)
    out["embed"] = emb
    lists = {"readme": (FROM, TO), "titles": (picked[:120], picked[120:])}
    for lname, (frm, to) in lists.items():
        for top_n in (1, 2, 3):
            for ms in (0.0, 0.75):
                for two in (True, False):
                    m = GensimEmbeddings(ft, min_similarity=ms, top_n=top_n, cosine_method="sklearn")
                    df = m.match(frm, to) if two else m.match(frm)
                    key = f"{lname}_{'two' if two else 'self'}_top{top_n}_ms{ms}"
                    out[key + "_frame"] = np.array(json.dumps(df_to_json(df)))
    savez_fixed(os.path.join(HERE, "fasttext_c1.npz"), out)
    print("written", os.path.join(HERE, "fasttext_c1.npz"))


if __name__ == "__main__":
    main()
