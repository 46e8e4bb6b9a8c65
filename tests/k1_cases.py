"""Case generators for the K1 edge tests (TEST INFRASTRUCTURE, NOT PRODUCT CODE; no GPU needed).

String lists at the places where the GPU vectoriser changes path: rows of 255 / 256 / 257 and 8 191 / 8 192 n-gram slots
(the warp kernel's limit and the long kernel's key arena), raw alphabets whose code space is exactly 2^24 and just above
it, and n-gram codes >= 2^63.  tests/golden/make_golden.py --k1-edges records the unmodified reference's output for them
in tests/golden/k1_edges.npz together with a digest of the inputs, so a changed generator fails loudly instead of being
compared with another input's output."""
import hashlib
import json

import numpy as np

# n-gram slots of a string of L code points (strings.ngram_slot_bounds): sum over n in lo..hi of max(0, L - n + 1).
# (3,3): L - 2.  (1,3): 3L - 3.  (3,6): 4L - 14.  (1,8): 8L - 28.  (8,8): L - 7.
CLEAN_ALPHA = "abcdefghijklmnopqrstuvwxyz0123456789"
RAW_ALPHA = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJ0123456789éüñİK中文"
LONG_ALPHA = "abé"              # rows of >= 1 000 code points: few distinct n-grams, so the fixture stays small
NAMES = ["slots33_clean", "slots33_raw", "slots13_clean", "slots36_raw", "slots18_raw", "space255_raw33", "space256_raw33",
         "codes64_raw18", "codes64_raw88"]


def _text(rng, n, alpha):
    """n code points over alpha, single spaces between words, none at either end (cleaning keeps the length)."""
    out = []
    for i in range(n):
        if 0 < i < n - 1 and out[-1] != " " and rng.random() < 0.18:
            out.append(" ")
        else:
            out.append(alpha[int(rng.integers(len(alpha)))])
    return "".join(out)


def alphabet(n_syms):
    """n_syms code points: the space, a run above U+00FF spaced 7 apart (past Latin-1, no surrogates) and one astral."""
    return "".join(chr(c) for c in [0x20] + [0x100 + 7 * i for i in range(n_syms - 2)] + [0x1F600])


def cases():
    """[{name, ngram_range, clean, remove_space, frm, to, new, slots}]: fit on to + frm (as the reference does), then
    transform `new`; `slots` are the slot counts the lists provably contain."""
    rng = np.random.default_rng(20261017)
    out = []
    shorts = ["", "ab", "abc", "  lead and trail  ", "many    spaces  in   a row", "İstanbul KELVIN K", "x"]
    unseen = ["", "zzzz yyyy", "Ω≈ç√∫ never seen", "ab", "   ", "中文中文 new"]

    def case(name, rng_, clean, rs, long_lengths, alpha, extra_from=(), extra_to=(), slots=(), new=(), short=shorts):
        longs = [_text(rng, L, alpha if L < 1000 else LONG_ALPHA) for L in long_lengths]
        mid = [_text(rng, int(rng.integers(3, 40)), alpha) for _ in range(12)]
        frm = short[:4] + longs[0::2] + mid[:6] + list(extra_from)
        to = short[4:] + longs[1::2] + mid[6:] + list(extra_to)
        out.append(dict(name=name, ngram_range=list(rng_), clean=clean, remove_space=rs, frm=frm, to=to,
                        new=unseen + mid[:3] + list(new), slots=list(slots)))

    # slot boundaries of the warp kernel (256) and of the long kernel's key arena (8 192), with short and empty rows in
    # the same launch; the long-kernel contents: one n-gram of tf 8 192, rows of > 32 and > 256 distinct terms, a clean
    # row of mostly punctuation (raw slots > 256, few symbols after cleaning) and one that cleans to ""
    case("slots33_clean", (3, 3), True, True, [257, 258, 259, 8193, 8194, 700], CLEAN_ALPHA + CLEAN_ALPHA.upper(),
         extra_from=["a" * 8194, "x" + "!.,;" * 100 + "y z", "?!" * 200],
         extra_to=["k" + "-+" * 150 + "elvin  K"], slots=[255, 256, 257, 8191, 8192])
    case("slots33_raw", (3, 3), False, False, [257, 258, 259, 8193, 8194, 700], RAW_ALPHA,
         extra_from=["a" * 8194], slots=[255, 256, 257, 8191, 8192])
    case("slots13_clean", (1, 3), True, True, [85, 86, 87, 2731], CLEAN_ALPHA, slots=[252, 255, 258, 8190])
    case("slots36_raw", (3, 6), False, True, [67, 68, 2051], RAW_ALPHA, slots=[254, 258, 8190])
    case("slots18_raw", (1, 8), False, True, [35, 36, 1027, 300], RAW_ALPHA, slots=[252, 260, 8188])

    # the next cases fit on exactly the symbols of `alpha`: their short rows are made of it too
    def own_shorts(a):
        return ["", a[1:3], a[3:6], "  " + a[6:12] + "  " + a[12:15] + " ", a[15:19] + "   " + a[19:30], a[30]]

    # code space of the raw (3,3) vectoriser: (|alphabet| + 1)^3 = 2^24 keeps the direct-addressed df table, 257^3 does not
    for n_syms, name in ((255, "space255_raw33"), (256, "space256_raw33")):
        a = alphabet(n_syms)
        case(name, (3, 3), False, True, [300, 40], a, extra_to=[a[1:]], new=[a[5:40] + "a", a[::-3]], short=own_shorts(a))
    # 64-bit codes: 255^8 ~ 1.78e19, so n-grams starting with a high symbol have codes >= 2^63
    a = alphabet(254)
    pairs = " ".join(a[i:i + 2] for i in range(1, len(a), 2))             # every symbol, in few n-grams once spaces are removed
    case("codes64_raw18", (1, 8), False, True, [60], a, extra_to=[pairs], new=[a[::-1], a[100:140] + "Z"], short=own_shorts(a))
    case("codes64_raw88", (8, 8), False, False, [60, 300], a, extra_to=[a[1:]], new=[a[::-1], a[100:140] + "Z"],
         short=own_shorts(a))
    assert [c["name"] for c in out] == NAMES
    return out


def digest(c):
    """sha256 of one case's inputs and settings."""
    key = [c["ngram_range"], c["clean"], c["remove_space"], c["frm"], c["to"], c["new"]]
    return hashlib.sha256(json.dumps(key, ensure_ascii=False).encode("utf-8")).hexdigest()


def load(golden_dir):
    """{name: case} with the reference's recorded output under case["g"] (a dict of arrays) and case["vocabulary"];
    asserts that the generator still makes the inputs the fixture was recorded from."""
    import os
    g = np.load(os.path.join(golden_dir, "k1_edges.npz"))
    out = {}
    for c in cases():
        name = c["name"]
        assert str(g[name + "_inputs_sha256"]) == digest(c), f"{name}: the inputs differ from those k1_edges.npz was made from"
        c["vocabulary"] = g[name + "_vocabulary"].tolist()
        c["g"] = {k[len(name) + 1:]: g[k] for k in g.files if k.startswith(name + "_")}
        out[name] = c
    return out
