"""oracle/assemble.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restatement of the reference's result-assembly tail, polyfuzz/models/_utils.py:104-125:
columns From, To, Similarity, To_2, Similarity_2, ...; similarities rounded to 3 decimals
(_utils.py:70,102,143); Similarity < 0.001 -> 0 and To -> None (_utils.py:119-123)."""
import numpy as np
import pandas as pd


def assemble(from_list, to_list, top_idx, top_val):
    if to_list is None:
        to_list = list(from_list)
    n, k = top_idx.shape
    cols = {"From": list(from_list)}
    for r in range(k):
        sims = np.round(np.asarray(top_val[:, r], dtype=np.float64), 3)
        names = [to_list[j] if j >= 0 else None for j in top_idx[:, r]]
        # an empty slot of the top-k arrays (index -1) is blank whatever score it carries; the reference has no empty
        # slots, and the kernels write them as (-1, 0.0)
        low = (sims < 0.001) | (np.asarray(top_idx[:, r]) < 0)
        sims = np.where(low, 0.0, sims)
        names = [None if l else nm for l, nm in zip(low, names)]
        cols["To" if r == 0 else f"To_{r + 1}"] = names
        cols["Similarity" if r == 0 else f"Similarity_{r + 1}"] = sims
    return pd.DataFrame(cols)


def cosine_topk_dense(x_from, y_to, k, min_similarity=0.0, self_match=False, normalize=False):
    """fp64 dense statement of the canonical contract for the Embeddings path (_utils.py:94-102
    re-normalises in the sklearn branch; the sparse branch does not, SURVEY 3.3)."""
    x = np.asarray(x_from, dtype=np.float64); y = np.asarray(y_to, dtype=np.float64)
    if normalize:
        x = x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-300)
        y = y / np.maximum(np.linalg.norm(y, axis=1, keepdims=True), 1e-300)
    s = x @ y.T
    n, m = s.shape
    idx = np.full((n, k), -1, dtype=np.int32); val = np.zeros((n, k), dtype=np.float64)
    for i in range(n):
        row = s[i]
        ok = row > min_similarity
        if self_match and i < m:
            ok[i] = False
        js = np.nonzero(ok)[0]
        order = js[np.lexsort((js, -row[js]))][:k]
        idx[i, :len(order)] = order; val[i, :len(order)] = row[order]
    return idx, val
