"""K5 (the frame tail on the device, csrc/pfz_assemble.cu) called directly with constructed top-k arrays, compared with
`==` against the host Arrow path (`assemble_matches`) and against the restated reference tail (oracle/assemble.py, the
reference's polyfuzz/models/_utils.py:104-125): scores on the 3-decimal rounding and the 0.001 blanking edges, bitmap
words that are partial or full, blank columns and frames, empty matched strings, the matcher paths, and a frame whose
matched strings total more than 2^31 bytes (64-bit byte positions)."""
import gc
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle.assemble import assemble as oracle_assemble

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tail():
    import pyarrow as pa
    from polyfuzz_b200.matchers import _utils
    assert _utils._str_dtype() is not None, "K5 needs pandas' Arrow-backed str dtype"
    return pa, _utils


def _dev_to_list(to_list):
    """The device-resident to-list as K5 takes it: int32 code points of an ASCII list and int64 offsets."""
    b = "".join(to_list).encode("ascii")
    off = np.zeros(len(to_list) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in to_list])
    blob = torch.from_numpy(np.frombuffer(b, dtype=np.uint8).astype(np.int32)) if b else torch.zeros(1, dtype=torch.int32)
    return blob.cuda(), torch.from_numpy(off).cuda()


def _col(df, c):
    if c.startswith("Similarity"):
        return df[c].to_numpy(dtype=np.float64).view(np.uint64).tolist()          # bit for bit (+0.0 is not -0.0)
    return [None if (isinstance(v, float) and np.isnan(v)) or v is None or v is pd.NA else v for v in df[c].tolist()]


def _frames_eq(got, exp):
    assert list(got.columns) == list(exp.columns)
    assert len(got) == len(exp)
    for c in exp.columns:
        assert _col(got, c) == _col(exp, c), c


def _device_frame(tail, from_list, to_list, idx, val):
    pa, u = tail
    blob, off = _dev_to_list(to_list)
    df = u.assemble_matches_device(pa.array(from_list, type=pa.large_string()), blob, off,
                                   torch.from_numpy(idx).cuda(), torch.from_numpy(val).cuda())
    assert u.LAST_TAIL["device"]
    return df


def _check(tail, from_list, to_list, idx, val):
    _, u = tail
    got = _device_frame(tail, from_list, to_list, idx, val)
    host = u.assemble_matches(from_list, to_list, idx, val)
    assert not u.LAST_TAIL["device"]
    ref = oracle_assemble(from_list, to_list, idx, val)
    _frames_eq(host, ref)
    _frames_eq(got, ref)
    return got


def _edge_scores():
    """Doubles x with x * 1000 == k + 1/2 exactly (rint rounds half to even), their neighbours, and the 0.001 edge."""
    nxt = lambda x, s: np.nextafter(x, s * np.inf)                         # noqa: E731
    out = [0.001, 0.0009995, 0.0005, 0.0015, 0.0025, 0.9995, 0.0, -0.0, -0.0004, -0.001, -0.5, 1.0, nxt(1.0, 1), 0.5, 0.123456]
    for k in (0, 1, 2, 3, 9, 10, 99, 123, 500, 998, 999):
        t = (k + 0.5) / 1000.0
        for d in range(-3, 4):                                             # the doubles around t that hit k + 1/2 exactly
            x = t
            for _ in range(abs(d)):
                x = nxt(x, np.sign(d))
            if x * 1000.0 == k + 0.5:
                out.append(x)
    half = [x for x in out if x * 1000.0 == np.floor(x * 1000.0) + 0.5]
    assert len(half) >= 10                                                  # the half-way cases are really there
    for x in list(out):
        out += [nxt(x, 1), nxt(x, -1), nxt(nxt(x, 1), 1), nxt(nxt(x, -1), -1)]
    return np.array(out, dtype=np.float64)


def _to_list(m, seed):
    rng = np.random.default_rng(seed)
    alpha = np.array(list("abcdefghijklmnopqrstuvwxyz0123456789 -.&ABCXYZ"))
    out = ["".join(rng.choice(alpha, int(rng.integers(1, 70)))) for _ in range(m)]
    out[3] = ""                                                             # a valid match may be the empty string
    out[7] = out[8]
    return out


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("k", [1, 2, 32, 40])
def test_frame_tail_rounding_and_shapes(tail, n, k):
    rng = np.random.default_rng(n * 100 + k)
    to_list = _to_list(300, seed=n + k)
    from_list = [f"from {i}" for i in range(n)]
    scores = _edge_scores()
    val = scores[rng.integers(0, len(scores), (n, k))]
    idx = rng.integers(0, len(to_list), (n, k)).astype(np.int32)
    idx[rng.random((n, k)) < 0.1] = -1                                      # empty slots, some with a non-zero score
    val[idx == -1] = np.where(rng.random(int((idx == -1).sum())) < 0.5, 0.9, 0.0)
    idx[0, 0], val[0, 0] = 3, 0.5                                           # "" with a valid score: "" and not null
    if k > 1:
        val[:, -1] = 0.0004999                                              # a column where every slot is blank
    got = _check(tail, from_list, to_list, idx, val)
    sims = got["Similarity"].to_numpy()
    assert got["To"].tolist()[0] == "" and sims[0] == 0.5
    if k > 1:
        assert got[f"To_{k}"].isna().all() and (got[f"Similarity_{k}"].to_numpy() == 0.0).all()
    # the edge values were hit on both sides of the blanking threshold
    r = np.round(val, 3)
    assert ((r == 0.001) & (idx >= 0)).any() or n * k < 64
    assert ((r < 0.001) & (idx >= 0)).any() or n * k < 64


def test_frame_tail_half_way_scores_round_to_even(tail):
    """One row per edge score, so that every score is checked, at rank 0 and at rank 1 of a 2-column frame."""
    scores = _edge_scores()
    n = len(scores)
    to_list = _to_list(40, seed=1)
    idx = np.stack([np.arange(n) % 40, (np.arange(n) + 1) % 40], 1).astype(np.int32)
    val = np.stack([scores, scores[::-1]], 1)
    got = _check(tail, [str(i) for i in range(n)], to_list, idx, val)
    # spot checks against the hand-derived values: 0.0005 -> 0.0 (blank); 0.0015 -> 0.002; 0.0025 -> 0.002; 0.001 stays
    s = dict(zip(scores.tolist(), got["Similarity"].tolist()))
    assert s[0.0005] == 0.0 and s[0.0015] == 0.002 and s[0.0025] == 0.002 and s[0.001] == 0.001 and s[0.0009995] == 0.001
    assert s[-0.0] == 0.0 and s[-0.5] == 0.0


def test_frame_tail_every_slot_blank(tail):
    """Total bytes 0: every slot empty or below 0.001."""
    n, k = 45, 3
    idx = np.full((n, k), -1, dtype=np.int32)
    idx[::2, 1] = 5
    val = np.full((n, k), 0.0004, dtype=np.float64)
    val[1::3, 0] = 0.7                                                      # idx -1 with a score: still blank
    got = _check(tail, [f"f{i}" for i in range(n)], _to_list(10, seed=2), idx, val)
    for c in ("To", "To_2", "To_3"):
        assert got[c].isna().all()


def test_frame_tail_matcher_paths(tail, monkeypatch):
    """TFIDF.match, a from_block self-match and re_train=False give the same frame with K5 as on the host Arrow path."""
    import polyfuzz_b200
    from polyfuzz_b200 import synth
    from polyfuzz_b200.matchers import _tfidf
    _, u = tail
    to = synth.company_names(3000, seed=21)
    frm = synth.company_names(700, seed=22) + ["", to[5]]
    new = synth.company_names(300, seed=23) + [""]

    def run(device):
        if not device:
            monkeypatch.setattr(_tfidf, "device_tail_available", lambda *a: False)
        m = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=5)
        out = [m.match(frm, to)]
        assert u.LAST_TAIL["device"] == device
        out.append(m.match(new, to, re_train=False))
        assert u.LAST_TAIL["device"] == device
        out.append(polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=4).match(to, from_block=(1000, 1033)))
        assert u.LAST_TAIL["device"] == device
        monkeypatch.undo()
        return out

    for got, exp in zip(run(True), run(False)):
        _frames_eq(got, exp)


def _big_tail_resources():
    need_dev = 5 << 30                           # 2.25 GB of bytes + the one-buffer copy of them + small arrays
    need_host = 5 << 30                          # the pinned result buffer (pool sizes are powers of two: 4 GiB) + headroom
    if not torch.cuda.is_available():
        return "no CUDA device"
    free, _ = torch.cuda.mem_get_info()
    if free < need_dev:
        return f"needs {need_dev >> 30} GiB of free device memory, {free / 2**30:.1f} GiB available"
    try:
        avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        avail = 0
    if avail < need_host:
        return f"needs {need_host >> 30} GiB of free host memory for pinned buffers, {avail / 2**30:.1f} GiB available"
    return None


def test_frame_tail_over_2_31_bytes(tail):
    """n = 1 100 rows x k = 32 ranks of 64 000-byte matches: 2.25e9 bytes in one frame, past the int32 range.  Byte
    positions and column offsets are 64-bit: the last columns start beyond 2^31."""
    reason = _big_tail_resources()
    if reason:
        pytest.skip(reason)
    from polyfuzz_b200 import engine
    _, u = tail
    n, k, L, m = 1100, 32, 64000, 8
    rng = np.random.default_rng(31)
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    to_list = [rng.choice(letters, L).tobytes().decode("ascii") for _ in range(m)]
    idx = ((np.arange(n)[:, None] + np.arange(k)[None, :]) % m).astype(np.int32)
    val = np.full((n, k), 0.5)
    val[5, 3], idx[7, 31] = 0.0004, -1                                      # two blank slots
    lens = np.where((val >= 0.001) & (idx >= 0), L, 0)
    assert int(lens.sum()) > 2 ** 31
    try:
        df = _device_frame(tail, [f"r{i}" for i in range(n)], to_list, idx, val)
        assert u.LAST_TAIL["d2h_bytes"] > 2 ** 31
        start = 0
        for r in range(k):
            c = "To" if r == 0 else f"To_{r + 1}"
            ch = df[c].array._pa_array
            assert ch.num_chunks == 1
            a = ch.chunk(0)
            offs = np.frombuffer(a.buffers()[1], dtype=np.int64)[a.offset:a.offset + n + 1]
            assert offs[0] == 0 and offs[-1] == int(lens[:, r].sum())     # the final offset of each column
            assert (np.diff(offs) >= 0).all()                              # offsets never decrease
            np.testing.assert_array_equal(np.diff(offs), lens[:, r])
            start += int(offs[-1])
        assert start == int(lens.sum())
        assert df["To_4"].isna().tolist()[5] and df["To_32"].isna().tolist()[7]
        # a sample of rows byte for byte, including the last ranks, whose bytes lie beyond 2^31 in the device buffer
        for i, r in [(0, 0), (1, 1), (n - 1, 15), (3, 30), (n // 2, 31), (n - 1, 31), (n - 2, 31), (6, 31)]:
            c = "To" if r == 0 else f"To_{r + 1}"
            assert df[c].iloc[i] == to_list[idx[i, r]], (i, r)
        np.testing.assert_array_equal(df["Similarity_32"].to_numpy(), np.where(idx[:, 31] >= 0, 0.5, 0.0))
    finally:
        df = None
        gc.collect()
        engine._PINNED_OUT.free = [(b, e) for b, e in engine._PINNED_OUT.free if b.numel() < (1 << 30)]
        torch.cuda.empty_cache()
