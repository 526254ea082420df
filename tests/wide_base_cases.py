"""Scalars S that reach the corners of the signed radix-2^w recoding of the table-driven verify's fixed-base table
(sc_recode_wide / sc_digit_wide in agentfield_b200/csrc/afc_sc.cuh), and the recoding restated on Python integers."""
import numpy as np

from oracle import go_ed25519 as G

WINDOWS = list(range(16, 23))          # every window AFC_VERIFY_BASE_WINDOW accepts


def rows(w):
    return -(-254 // w)


def recode(s, w):
    """Signed digits: rows - 1 digits in [-2^(w-1), 2^(w-1)) and the top digit, everything above, unsigned."""
    r = rows(w)
    t = s + sum(1 << (w * i + w - 1) for i in range(r - 1))
    return [((t >> (w * i)) & ((1 << w) - 1)) - (1 << (w - 1)) for i in range(r - 1)] + [t >> (w * (r - 1))]


def compose(d, w):
    return sum(x << (w * i) for i, x in enumerate(d))


def scalars(w, seed=0xAF21):
    """name -> S < L."""
    r, h = rows(w), 1 << (w - 1)
    out = {"0": 0, "1": 1, "L-1": G.L - 1,
           "every digit -2^(w-1)": compose([-h] * (r - 1) + [1], w),
           "every digit 2^(w-1)-1": compose([h - 1] * (r - 1) + [0], w),
           "digits alternate at both ends": compose([(-h if i % 2 else h - 1) for i in range(r - 1)] + [1], w),
           "carries into the top row": (1 << (w * (r - 1))) - 1,
           "top row only": 1 << (w * (r - 1))}
    rng = np.random.default_rng(seed + w)
    for j in range(r):
        d = recode(int.from_bytes(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), "little") % G.L, w)
        d[j] = 0
        out["zero digit in row %d" % j] = compose(d, w)
    out = {k: v for k, v in out.items() if 0 <= v < G.L}
    return out
