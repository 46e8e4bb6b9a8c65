"""Generate tests/golden/gensim_c1.npz by running the UNMODIFIED reference's GensimEmbeddings (/root/reference, imported through
oracle/ref_shim.py, with gensim stubbed by tests/gensim_oracle.py) in the build container.  Re-run:

    python tests/golden/make_gensim_golden.py

What is recorded: seeded stand-in vocabularies of d = 25 and d = 300 (keys, the row each key maps to, float32 vectors and a
float64 copy; the tokens of the README lists and of titles from tests/golden/data, non-ASCII ones included, less a seeded 10 %
held out as missing); the reference's _embed of those strings for both vector dtypes; and its match frames
(cosine_method="sklearn", top_n 1..3, min_similarity 0 and 0.75, two lists and self-match).  Regenerating is byte-identical."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
from make_golden import FROM, TO, df_to_json, savez_fixed  # noqa: E402  (also installs the reference's import shim)
import gensim_oracle as go  # noqa: E402


def main():
    assert go.install_gensim(), "the gensim stub needs gensim to be absent"
    from polyfuzz.models._gensim import GensimEmbeddings
    titles = list(dict.fromkeys(json.load(open(os.path.join(HERE, "data", "movie_titles.json")))["Netflix"]))
    ascii_t = [t for t in titles if t.isascii()]
    other_t = [t for t in titles if not t.isascii()]
    out = {}
    for tag, d, n_titles in (("d25", 25, 510), ("d300", 300, 24)):
        picked = ascii_t[:n_titles - n_titles // 6] + other_t[:n_titles // 6]
        readme = FROM + TO
        tokens = list(dict.fromkeys(t for s in readme + picked for t in s.split(" ")))
        rng = np.random.default_rng(2500 + d)
        held = set(rng.choice([t for t in tokens if t not in readme], size=len(tokens) // 10, replace=False))
        keys = [t for t in tokens if t not in held]
        V = go.random_vectors(len(keys), d, seed=d)
        k2i = {keys[j]: j for j in rng.permutation(len(keys))}          # dict order differs from the row order
        # pooled rows that coincide ("a b" and "b a") tie in every cosine: keep one string of each
        pooled = go.embed(k2i, V, picked)
        _, first = np.unique(go.bits(pooled), axis=0, return_index=True)
        picked = [picked[i] for i in sorted(first)]
        out[tag + "_keys"] = np.array(keys)
        out[tag + "_rows"] = np.array([k2i[k] for k in keys], dtype=np.int64)
        out[tag + "_vectors_f32"] = V
        out[tag + "_vectors_f64"] = V.astype(np.float64)
        out[tag + "_strings"] = np.array(readme + picked)
        for dt in ("f32", "f64"):
            kv = go.KeyedVectorsStandIn(sorted(k2i, key=k2i.get), out[f"{tag}_vectors_{dt}"], k2i)
            out[f"{tag}_embed_{dt}"] = np.asarray(GensimEmbeddings(kv)._embed(readme + picked), np.float64)
        kv = go.KeyedVectorsStandIn(sorted(k2i, key=k2i.get), V, k2i)
        lists = {"readme": (FROM, TO)}
        if tag == "d25":
            lists["titles"] = (picked[:120], picked[120:])
        for lname, (frm, to) in lists.items():
            for top_n in (1, 2, 3):
                for ms in (0.0, 0.75):
                    for two in (True, False):
                        m = GensimEmbeddings(kv, min_similarity=ms, top_n=top_n, cosine_method="sklearn")
                        df = m.match(frm, to) if two else m.match(frm)
                        key = f"{tag}_{lname}_{'two' if two else 'self'}_top{top_n}_ms{ms}"
                        out[key + "_frame"] = np.array(json.dumps(df_to_json(df)))
    savez_fixed(os.path.join(HERE, "gensim_c1.npz"), out)
    print("written", os.path.join(HERE, "gensim_c1.npz"))


if __name__ == "__main__":
    main()
