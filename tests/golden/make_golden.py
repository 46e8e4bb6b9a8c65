"""Generate tests/golden/*.npz|json by running the UNMODIFIED reference (/root/reference, imported
through oracle/ref_shim.py) in the build container.  The reference cannot travel to the GPU box, so
its inputs/outputs are committed as small fixtures.  Re-run:  python tests/golden/make_golden.py

What is recorded (SURVEY.md section 8c "Golden vectors"):
  c1_tfidf.npz        reference TFIDF._extract_tf_idf CSR (two-list and self-match) on the README /
                      tests/utils.py 6-vs-3 lists for every n-gram range the reference tests use
                      (tests/models/test_tfidf.py:20, tests/test_polyfuzz.py:111), vocabulary + idf
  c1_match.json       reference TFIDF.match DataFrames (sklearn branch, the only numeric branch
                      runnable here) for top_n 1..3, two-list and self-match
  company_slice.npz   company_names[20000:23000] self-match: reference CSR, and reference
                      cosine_similarity(method="sklearn") top-10 indices + 3-dp scores
  clean_survivors.json  exhaustive probe of _clean_string over all code points
  dense_c1.npz        reference tests/from_list.npy|to_list.npy + reference sklearn-branch result
  k1_edges.npz        reference TFIDF._extract_tf_idf on the lists of tests/k1_cases.py, at the places where the GPU
                      vectoriser changes path: rows of 255..257 and 8 191..8 192 n-gram slots, a code space of exactly
                      2^24 and one just above it, n-gram codes >= 2^63; fit CSR of both lists, idf, vocabulary, the CSR
                      of a transformed list with unseen symbols and n-grams, and a digest of the inputs.
                      Write only this fixture:  python tests/golden/make_golden.py --k1-edges
"""
import io
import zipfile
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
warnings.filterwarnings("ignore")

from oracle import ref_shim  # noqa: E402

ref_shim.install()
from polyfuzz.models import TFIDF  # noqa: E402
from polyfuzz.models._tfidf import _clean_string  # noqa: E402
from polyfuzz.models._utils import cosine_similarity  # noqa: E402

FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]
RANGES = [(1, 1), (1, 2), (1, 3), (2, 2), (2, 3), (3, 3), (3, 6)]


def csr_parts(prefix, m, out):
    m = m.tocsr(); m.sort_indices()
    out[prefix + "_indptr"] = m.indptr.astype(np.int32)
    out[prefix + "_indices"] = m.indices.astype(np.int32)
    out[prefix + "_data"] = m.data.astype(np.float64)
    out[prefix + "_shape"] = np.array(m.shape, dtype=np.int64)


def df_to_json(df):
    return {c: [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] for c in df.columns}


def savez_fixed(path, arrays):
    """np.savez_compressed with fixed zip timestamps, so that regenerating a fixture is byte-identical."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name, arr in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arr), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def k1_edges():
    """The reference's output for the K1 edge cases of tests/k1_cases.py (the inputs are rebuilt there, not stored)."""
    sys.path.insert(0, os.path.join(HERE, ".."))
    import k1_cases
    out = {}
    for c in k1_cases.cases():
        name = c["name"]
        m = TFIDF(n_gram_range=tuple(c["ngram_range"]), clean_string=c["clean"], remove_space_ngrams=c["remove_space"])
        f, t = m._extract_tf_idf(c["frm"], c["to"], True)
        csr_parts(name + "_from", f, out); csr_parts(name + "_to", t, out)
        out[name + "_idf"] = m.vectorizer.idf_.astype(np.float64)
        out[name + "_vocabulary"] = np.array(sorted(m.vectorizer.vocabulary_, key=m.vectorizer.vocabulary_.get))
        nw, _ = m._extract_tf_idf(c["new"], c["to"], False)                 # transform with the fitted vectoriser
        csr_parts(name + "_new", nw, out)
        out[name + "_inputs_sha256"] = np.array(k1_cases.digest(c))
    savez_fixed(os.path.join(HERE, "k1_edges.npz"), out)


def main():
    # ---- C1 vectoriser -------------------------------------------------------------------
    out = {}
    vocabs = {}
    for lo, hi in RANGES:
        for clean in (True, False):
            for rs in (True, False):
                tag = f"r{lo}{hi}_c{int(clean)}_s{int(rs)}"
                m = TFIDF(n_gram_range=(lo, hi), clean_string=clean, remove_space_ngrams=rs)
                f, t = m._extract_tf_idf(FROM, TO, True)
                csr_parts(tag + "_two_from", f, out); csr_parts(tag + "_two_to", t, out)
                voc = sorted(m.vectorizer.vocabulary_, key=m.vectorizer.vocabulary_.get)
                vocabs[tag + "_two"] = voc
                out[tag + "_two_idf"] = m.vectorizer.idf_.astype(np.float64)
                m2 = TFIDF(n_gram_range=(lo, hi), clean_string=clean, remove_space_ngrams=rs)
                f2, t2 = m2._extract_tf_idf(FROM, None, True)
                csr_parts(tag + "_self", f2, out)
                vocabs[tag + "_self"] = sorted(m2.vectorizer.vocabulary_, key=m2.vectorizer.vocabulary_.get)
                out[tag + "_self_idf"] = m2.vectorizer.idf_.astype(np.float64)
    np.savez_compressed(os.path.join(HERE, "c1_tfidf.npz"), **out)
    json.dump(vocabs, open(os.path.join(HERE, "c1_vocab.json"), "w"))

    # ---- C1 match DataFrames (sklearn branch; `sparse` silently falls to it w/o the package) ----
    match = {}
    for top_n in (1, 2, 3):
        for ms in (0.0, 0.75):
            m = TFIDF(min_similarity=ms, top_n=top_n, cosine_method="sklearn")
            match[f"two_top{top_n}_ms{ms}"] = df_to_json(m.match(FROM, TO))
            m = TFIDF(min_similarity=ms, top_n=top_n, cosine_method="sklearn")
            match[f"self_top{top_n}_ms{ms}"] = df_to_json(m.match(FROM))
    # transform path (re_train=False), polyfuzz/polyfuzz.py:235
    m = TFIDF(min_similarity=0, top_n=1, cosine_method="sklearn")
    m.match(FROM, TO)
    match["transform_unseen"] = df_to_json(m.match(["apples", "mouses", "zzz"], TO, re_train=False))
    json.dump(match, open(os.path.join(HERE, "c1_match.json"), "w"), indent=0)

    # ---- company slice ---------------------------------------------------------------------
    names = json.load(open(os.path.join(ref_shim.REFERENCE_ROOT, "data", "company_names.json")))[20000:23000]
    m = TFIDF(n_gram_range=(3, 3), min_similarity=0, top_n=10, cosine_method="sklearn")
    f, t = m._extract_tf_idf(names, None, True)
    out = {}
    csr_parts("csr", f, out)
    out["idf"] = m.vectorizer.idf_.astype(np.float64)
    k = 10
    df = cosine_similarity(f, t, names, None, 0.0, top_n=k, method="sklearn")
    # recover what the reference computed: scores (3 dp) per rank and the matched strings
    sims = np.stack([df["Similarity" if r == 0 else f"Similarity_{r+1}"].to_numpy() for r in range(k)], 1)
    out["ref_sims"] = sims.astype(np.float64)
    # the reference's own index array (before DataFrame assembly), _utils.py:95-101
    from sklearn.metrics.pairwise import cosine_similarity as skcos
    sm = skcos(f, t); np.fill_diagonal(sm, 0)
    out["ref_idx"] = np.flip(np.argsort(sm, axis=-1), axis=1)[:, :k].astype(np.int32)
    srt = np.flip(np.sort(sm, axis=-1), axis=1)[:, :k + 1]
    out["ref_tiefree"] = (np.diff(srt, axis=1) != 0).all(axis=1)     # rows with no exact tie in ranks 1..k+1
    out["ref_topvals"] = srt[:, :k].astype(np.float64)
    np.savez_compressed(os.path.join(HERE, "company_slice.npz"), **out)
    json.dump({"names": names}, open(os.path.join(HERE, "company_slice_names.json"), "w"))

    # ---- movie titles slice (non-ASCII, punctuation): raw and clean vectoriser, (1,3)- and 3-grams ----------
    mt = json.load(open(os.path.join(ref_shim.REFERENCE_ROOT, "data", "movie_titles.json")))
    titles_to = mt["IMDB"][2000:2600]; titles_from = mt["Netflix"][:300]
    out = {}
    for tag, rng, clean in (("raw33", (3, 3), False), ("clean13", (1, 3), True), ("raw12", (1, 2), False)):
        m = TFIDF(n_gram_range=rng, clean_string=clean, min_similarity=0, top_n=3, cosine_method="sklearn")
        f, t = m._extract_tf_idf(titles_from, titles_to, True)
        csr_parts(tag + "_from", f, out); csr_parts(tag + "_to", t, out)
        out[tag + "_idf"] = m.vectorizer.idf_.astype(np.float64)
    np.savez_compressed(os.path.join(HERE, "titles_slice.npz"), **out)
    json.dump({"from": titles_from, "to": titles_to}, open(os.path.join(HERE, "titles_slice_names.json"), "w"))

    # ---- _clean_string exhaustive probe -----------------------------------------------------------
    surv = {}
    for cp in range(0x110000):
        if 0xD800 <= cp <= 0xDFFF:
            continue
        r = _clean_string("a" + chr(cp) + "b")
        if cp >= 128 and r != "ab":
            surv[str(cp)] = r
    ascii_map = {str(cp): _clean_string("a" + chr(cp) + "b") for cp in range(128)}
    json.dump({"non_ascii_survivors": surv, "ascii": ascii_map,
               "examples": {s: _clean_string(s) for s in
                            ["  Hello,  World!! ", "A\tB\nC", "İstanbul Kelvin K", "--", "", " a  b ", "ÀÉ x9"]}},
              open(os.path.join(HERE, "clean_survivors.json"), "w"))

    # ---- dense fixture ------------------------------------------------------------------------
    fv = np.load(os.path.join(ref_shim.REFERENCE_ROOT, "tests", "from_list.npy"))
    tv = np.load(os.path.join(ref_shim.REFERENCE_ROOT, "tests", "to_list.npy"))
    d = {"from_vec": fv, "to_vec": tv, "prod": fv @ tv.T}
    for top_n in (1, 2, 3):
        df = cosine_similarity(fv, tv, FROM, TO, 0.0, top_n=top_n, method="sklearn")
        d[f"sims_top{top_n}"] = np.stack([df["Similarity" if r == 0 else f"Similarity_{r+1}"].to_numpy()
                                          for r in range(top_n)], 1)
        json.dump(df_to_json(df), open(os.path.join(HERE, f"dense_c1_top{top_n}.json"), "w"))
    np.savez_compressed(os.path.join(HERE, "dense_c1.npz"), **d)
    k1_edges()
    print("golden fixtures written to", HERE)


if __name__ == "__main__":
    if "--k1-edges" in sys.argv:
        k1_edges()
    else:
        main()
