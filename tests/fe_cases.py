"""Operands at the carry and reduction boundaries of afc_fe.cuh / afc_sc.cuh, and their exact results, for the tests/devsim
harness (tests/test_fe_boundaries_hostsim.py on the CPU, tests/test_fe_boundaries_gpu.py on the H100).

Every expected output comes from Python integers.  For the weakly reduced field routines the expected value is the limb
algorithm replayed on integers (each carry chain is one 256-bit addition), so the device must match it bit for bit; the
replay is itself checked against x*y % p and friends.  The replays count how often each rarely taken branch fires, and
the tests require every one of REQUIRED_BRANCHES to fire on some constructed case — a "boundary" case that misses its
branch fails the suite instead of passing quietly."""
import collections
import random

import numpy as np

P = 2**255 - 19
L = 2**252 + 27742317777372353535851937790883648493
MU = 2**512 // L
M256 = 2**256 - 1

# tests/devsim/devsim_ops.cuh, enum Op
(OP_MUL_WIDE, OP_SQ_WIDE, OP_MUL_WIDE_KARA, OP_FOLD16, OP_MUL, OP_SQ, OP_MUL_CALL, OP_SQ_CALL, OP_ADD, OP_SUB, OP_ADDSUB,
 OP_TOWORDS, OP_INVERT, OP_POW22523, OP_SC_REDUCE512, OP_SC_REDUCE256, OP_SC_MULADD, OP_COUNT) = range(18)
OP_NAMES = ["mul_wide", "sq_wide", "mul_wide_kara", "fold16", "mul", "sq", "mul_call", "sq_call", "add", "sub", "addsub_m",
            "towords", "invert", "pow22523", "sc_reduce512", "sc_reduce256", "sc_muladd"]
DEVICE_ONLY = {OP_MUL_WIDE_KARA, OP_MUL_CALL, OP_SQ_CALL}

# branch -> what reaching it means
REQUIRED_BRANCHES = {
    "add.wrap2": "fe_add: the +38 of the first wrap carries out again",
    "sub.borrow2": "fe_sub: the -38 of the first wrap borrows again",
    "addsub.add.wrap2": "fe_addsub_m (add, keep): second carry",
    "addsub.sub.borrow2": "fe_addsub_m (subtract, keep): second borrow",
    "fold.wrap2": "fe_fold16: r + 38*top carries out of 2^256",
    "fold.top38": "fe_fold16: top = 38, the largest the first fold can leave",
    "mul.wrap2": "fe_mul: the product's fold takes the second wrap",
    "towords.bit255": "fe_towords: bit 255 folded in as +19",
    "towords.ge": "fe_towords: value >= p after the fold, p subtracted",
    "sc.corr1": "Barrett estimate low by one: one conditional subtraction of L",
}


class Branches(collections.Counter):
    def hit(self, name, cond=True):
        if cond:
            self[name] += 1


NOBR = Branches()   # sink for replays whose branch counts nobody reads


# ----------------------------------------------------------------------------------------------- replays on integers
def add_ref(f, g, br=NOBR, tag="add"):
    s = f + g
    c = s >> 256
    u = (s & M256) + 38 * c
    c2 = u >> 256
    br.hit(tag + ".wrap1", c)
    br.hit(tag + ".wrap2", c2)
    return (u & M256) + 38 * c2


def sub_ref(f, g, br=NOBR, tag="sub"):
    d = f - g
    b = d < 0
    u = (d & M256) - 38 * b
    b2 = u < 0
    br.hit(tag + ".borrow1", b)
    br.hit(tag + ".borrow2", b2)
    return (u & M256) - 38 * b2


def addsub_ref(f, g, keep, sgn, br=NOBR):
    g = g if keep else 0
    if sgn:
        return sub_ref(f, g, br, "addsub.sub" if keep else "addsub.sub0")
    return add_ref(f, g, br, "addsub.add" if keep else "addsub.add0")


def fold_ref(t, br=NOBR, tag="fold"):
    s = (t & M256) + 38 * (t >> 256)
    top = s >> 256
    u = (s & M256) + 38 * top
    c2 = u >> 256
    br.hit(tag + ".top38", top == 38)
    br.hit(tag + ".wrap2", c2)
    return (u & M256) + 38 * c2


def mul_ref(a, b, br=NOBR):
    return fold_ref(a * b, br, "mul")


def sq_ref(a, br=NOBR):
    return fold_ref(a * a, br, "sq")


def towords_ref(x, br=NOBR):
    hi = x >> 255
    r = (x & (2**255 - 1)) + 19 * hi
    y = r + 19
    ge = y >> 255
    br.hit("towords.bit255", hi)
    br.hit("towords.ge", ge)
    out = (y if ge else r) & (2**255 - 1)
    assert out == x % P
    return out


def _sqn(x, n):
    for _ in range(n):
        x = sq_ref(x)
    return x


def _pow_2_250_m1(z):
    """afc_fe.cuh fe_pow_2_250_m1, step by step: (z^(2^250-1), z^11)."""
    t0 = sq_ref(z)
    t1 = mul_ref(z, _sqn(t0, 2))
    t0 = mul_ref(t0, t1)
    z11 = t0
    t1 = mul_ref(t1, sq_ref(t0))
    t1 = mul_ref(_sqn(t1, 5), t1)
    t2 = mul_ref(_sqn(t1, 10), t1)
    t2 = mul_ref(_sqn(t2, 20), t2)
    t1 = mul_ref(_sqn(t2, 10), t1)
    t2 = mul_ref(_sqn(t1, 50), t1)
    t2 = mul_ref(_sqn(t2, 100), t2)
    return mul_ref(_sqn(t2, 50), t1), z11


def invert_ref(z):
    t, z11 = _pow_2_250_m1(z)
    out = mul_ref(_sqn(t, 5), z11)
    assert out % P == pow(z, P - 2, P)
    return out


def pow22523_ref(z):
    t, _ = _pow_2_250_m1(z)
    out = mul_ref(_sqn(t, 2), z)
    assert out % P == pow(z, (P - 5) // 8, P)
    return out


def barrett_ref(x, br=NOBR):
    """sc_reduce512 on integers (HAC 14.42, b = 2^32, k = 8): returns x mod L, counting the corrective subtractions."""
    q3 = ((x >> 224) * MU) >> 288
    r = (x - q3 * L) % 2**288
    n = 0
    while r >= L and n < 2:
        r -= L
        n += 1
    br.hit("sc.corr%d" % n)
    assert r == x % L
    return r


def barrett_max_deficit():
    """An upper bound on x/L - q3 over every x < 2^512: floor(x / 2^224) drops less than 2^224/L, and mu = floor(2^512/L)
    loses (2^512/L - mu) times q1/2^288 < 1.  Below 1 means the estimate is never low by 2."""
    from fractions import Fraction
    return Fraction(2**224, L) + (Fraction(2**512, L) - MU)


def expected(op, x):
    """The exact output words (16) of op for one item x (a tuple of integers), as an integer."""
    if op in (OP_MUL_WIDE, OP_MUL_WIDE_KARA):
        return x[0] * x[1]
    if op == OP_SQ_WIDE:
        return x[0] * x[0]
    if op == OP_FOLD16:
        r = fold_ref(x[0])
    elif op in (OP_MUL, OP_MUL_CALL):
        r = mul_ref(x[0], x[1])
        assert r % P == x[0] * x[1] % P
    elif op in (OP_SQ, OP_SQ_CALL):
        r = sq_ref(x[0])
        assert r % P == x[0] * x[0] % P
    elif op == OP_ADD:
        r = add_ref(x[0], x[1])
        assert r % P == (x[0] + x[1]) % P
    elif op == OP_SUB:
        r = sub_ref(x[0], x[1])
        assert r % P == (x[0] - x[1]) % P
    elif op == OP_ADDSUB:
        r = addsub_ref(*x)
        assert r % P == (x[0] + (-1 if x[3] else 1) * (x[1] if x[2] else 0)) % P
    elif op == OP_TOWORDS:
        return x[0] % P
    elif op == OP_INVERT:
        r = invert_ref(x[0])
    elif op == OP_POW22523:
        r = pow22523_ref(x[0])
    elif op == OP_SC_REDUCE512:
        return x[0] % L
    elif op == OP_SC_REDUCE256:
        return x[0] % L
    elif op == OP_SC_MULADD:
        return (x[0] * x[1] + x[2]) % L
    else:
        raise ValueError(op)
    assert 0 <= r < 2**256
    return r


def count_branches(op, x, br):
    """Replay op on x, counting branches into br (the expected value itself comes from expected())."""
    if op == OP_FOLD16:
        fold_ref(x[0], br)
    elif op in (OP_MUL, OP_MUL_CALL):
        mul_ref(x[0], x[1], br)
    elif op in (OP_SQ, OP_SQ_CALL):
        sq_ref(x[0], br)
    elif op == OP_ADD:
        add_ref(x[0], x[1], br)
    elif op == OP_SUB:
        sub_ref(x[0], x[1], br)
    elif op == OP_ADDSUB:
        addsub_ref(*x, br=br)
    elif op == OP_TOWORDS:
        towords_ref(x[0], br)
    elif op in (OP_SC_REDUCE512, OP_SC_REDUCE256):
        barrett_ref(x[0], br)
    elif op == OP_SC_MULADD:
        barrett_ref(x[0] * x[1] + x[2], br)


# ----------------------------------------------------------------------------------------------- packing
def _words(vals, n):
    """Integers -> uint32 array of shape (len(vals), n), little-endian limbs."""
    b = b"".join(int(v).to_bytes(4 * n, "little") for v in vals)
    return np.frombuffer(b, dtype="<u4").reshape(len(vals), n).astype(np.uint32)


def pack(op, items):
    """Items (tuples of integers) -> the harness's (n, 32) input words."""
    a = np.zeros((len(items), 32), dtype=np.uint32)
    if not items:
        return a
    if op in (OP_FOLD16, OP_SC_REDUCE512):
        a[:, :16] = _words([x[0] for x in items], 16)
        return a
    for k in range(len(items[0])):
        col = [x[k] for x in items]
        if op == OP_ADDSUB and k >= 2:
            a[:, 16 + k - 2] = np.array([1 if v else 0 for v in col], dtype=np.uint32)
        else:
            a[:, 8 * k:8 * k + 8] = _words(col, 8)
    return a


def unpack_in(op, words):
    """The inverse of pack, for inputs the device generated: (n, 32) words -> items."""
    def ints(cols):
        return [int.from_bytes(np.ascontiguousarray(r).tobytes(), "little") for r in cols]
    if op in (OP_FOLD16, OP_SC_REDUCE512):
        return [(v,) for v in ints(words[:, :16])]
    a, b, c = ints(words[:, 0:8]), ints(words[:, 8:16]), ints(words[:, 16:24])
    if op in (OP_SQ_WIDE, OP_SQ, OP_SQ_CALL, OP_TOWORDS, OP_INVERT, OP_POW22523, OP_SC_REDUCE256):
        return [(x,) for x in a]
    if op == OP_ADDSUB:
        return [(x, y, int(k & 1), int(s & 1)) for x, y, k, s in zip(a, b, words[:, 16], words[:, 17])]
    if op == OP_SC_MULADD:
        return list(zip(a, b, c))
    return list(zip(a, b))


def unpack_out(words):
    return [int.from_bytes(np.ascontiguousarray(r).tobytes(), "little") for r in words]


# ----------------------------------------------------------------------------------------------- constructed operands
def _mask_val(m):
    """8-bit mask -> the 256-bit value whose limb i is 0xffffffff when bit i is set, else 0."""
    return sum(0xFFFFFFFF << (32 * i) for i in range(8) if m >> i & 1)


def _fold_window_input(rng, top, r):
    """A 512-bit t with (t mod 2^256) + 38 (t >> 256) = top 2^256 + r, or None if no t has that first fold."""
    s = (top << 256) + r
    lo_min, lo_max = max(0, s - 38 * M256), min(M256, s)
    if lo_min > lo_max:
        return None
    lo = rng.randint(lo_min, lo_max)
    lo -= (lo - s) % 38
    if lo < lo_min:
        lo += 38
    if lo > lo_max:
        return None
    return lo + (((s - lo) // 38) << 256)


def field_cases(seed=0xFE25519):
    """{op: [items]} at the boundaries of the field routines."""
    rng = random.Random(seed)
    cases = collections.defaultdict(list)
    # add / sub / addsub: sums and differences at the wraps
    sums = [2**256 - 1, 2**256, 2**256 + 37, 2**256 + 38] + list(range(2**257 - 39, 2**257 - 1))
    pairs = []
    for s in sums:
        for f in (s - M256, s // 2, M256, s - M256 + rng.randrange(M256 - (s - M256) + 1)) if s > M256 else (0, s, s // 2):
            if 0 <= f <= M256 and 0 <= s - f <= M256:
                pairs.append((f, s - f))
    for d in (-1, -38, -39):
        for f in (0, 1, 2**255, M256 + d, rng.randrange(2**256 + d)):
            if 0 <= f <= M256 and 0 <= f - d <= M256:
                pairs.append((f, f - d))
    pairs += [(0, g) for g in range(2**256 - 38, 2**256)]
    pairs += [(g, 0) for g in range(2**256 - 38, 2**256)]
    cases[OP_ADD] = pairs
    cases[OP_SUB] = pairs
    cases[OP_ADDSUB] = [(f, g, keep, sgn) for f, g in pairs for keep in (0, 1) for sgn in (0, 1)]
    # fold16: every top, the first fold's result in [2^256 - 38 top, 2^256) and just below it
    fold = [M256 << 256 | M256, M256 << 256, M256, 0]
    for top in range(39):
        for r in {2**256 - 38 * top, 2**256 - 38 * top - 1, 2**256 - 1, 2**256 - 39 * 38, 0}:
            for _ in range(3):
                if 0 <= r <= M256:
                    t = _fold_window_input(rng, top, r)
                    if t is not None:
                        fold.append(t)
        for _ in range(4):
            if top:
                t = _fold_window_input(rng, top, 2**256 - rng.randint(1, 38 * top))
                if t is not None:
                    fold.append(t)
    cases[OP_FOLD16] = [(t,) for t in fold]
    # wide products and the multiplies: every pair of all-ones/zero limb masks, single limbs, one all-ones limb
    masks = [_mask_val(m) for m in range(256)]
    mul = [(x, y) for x in masks for y in masks]
    singles = [v << (32 * i) for i in range(8) for v in (1, 0xFFFFFFFF, rng.getrandbits(32) | 1)]
    mul += [(x, y) for x in singles for y in singles]
    for i in range(8):
        for _ in range(16):
            x, y = rng.getrandbits(256), rng.getrandbits(256)
            x |= 0xFFFFFFFF << (32 * i)
            mul.append((x, y))
            mul.append((y, x))
    mul += _mul_wrap2_pairs(rng)
    for op in (OP_MUL_WIDE, OP_MUL_WIDE_KARA, OP_MUL, OP_MUL_CALL):
        cases[op] = mul
    sq = [(x,) for x in masks + singles] + [(x,) for x, _ in mul[-2048:]]
    sq += [(v,) for v in (P - 1, P, P + 1, 2**255, M256, 2**256 - 38, 2**256 - 39)]
    for op in (OP_SQ_WIDE, OP_SQ, OP_SQ_CALL):
        cases[op] = sq
    # towords: both sides of p, 2p, 2^255 and 2^256
    tw = list(range(41))
    for c in (P, 2 * P, 2**255):
        tw += [c + d for d in range(-40, 41)]
    tw += list(range(2**256 - 40, 2**256))
    cases[OP_TOWORDS] = [(x,) for x in sorted(set(v for v in tw if 0 <= v <= M256))]
    # invert / pow22523: 0, 1, p - 1 and the non-canonical spellings
    ex = [0, 1, 2, P - 1, P, P + 1, 2 * P, M256, 2**255 - 1, 2**256 - 38] + [rng.getrandbits(256) for _ in range(6)]
    cases[OP_INVERT] = [(x,) for x in ex]
    cases[OP_POW22523] = [(x,) for x in ex]
    return cases


def _mul_wrap2_pairs(rng, want=96):
    """(a, b) whose product's fold takes the second wrap: fix the first fold X = t_lo + 38 t_hi in the window, pick
    b in [2^255, 2^256), solve t = t_lo + 2^256 t_hi = X + (2^256 - 38) t_hi = 0 (mod b) for t_hi, keep it when t_lo is a
    256-bit limb string and a = t / b fits in 256 bits."""
    out = []
    inv_tries = 0
    while len(out) < want:
        inv_tries += 1
        assert inv_tries < 200000, "fe_mul second-wrap construction found too few pairs"
        top = rng.randint(1, 38)
        X = (top << 256) + 2**256 - rng.randint(1, 38 * top)
        b = rng.randrange(2**255, 2**256) | 1
        try:
            th = (-X * pow(2**256 - 38, -1, b)) % b
        except ValueError:
            continue
        while th * 38 <= X:
            tl = X - 38 * th
            if tl <= M256 and th <= M256:
                t = tl + (th << 256)
                a = t // b
                if t % b == 0 and a <= M256:
                    out.append((a, b))
            th += b
    return out


def scalar_cases(seed=0x5CA1A2):
    """{op: [items]} for the scalar routines: the existing sc_reduce512 specials, multiples of L either side, and inputs
    whose Barrett quotient estimate is one low (searched: near multiples of L with the dropped low bits large)."""
    rng = random.Random(seed)
    r512 = [M256 << 256 | M256, 0] + [L * k + d for k in (1, 2, 2**250) for d in (-1, 0, 1)]
    r512 += [L * k + d for k in (2**259, (2**512 - 1) // L, (2**512 - 1) // L - 1) for d in (-1, 0, 1)]
    low = []
    while len(low) < 64:
        x = L * rng.getrandbits(259) + rng.getrandbits(rng.randint(1, 224))
        if x < 2**512:
            br = Branches()
            barrett_ref(x, br)
            if br["sc.corr1"]:
                low.append(x)
    r512 += low + [rng.getrandbits(512) for _ in range(64)]
    r256 = [0, 1, L - 1, L, L + 1, 2 * L, 15 * L, M256, 2**255, 2**253] + [L * k + d for k in range(1, 16) for d in (-1, 0, 1)]
    low256 = []
    while len(low256) < 32:
        k = rng.randint(1, 15)
        x = L * k + rng.getrandbits(rng.randint(1, 200))
        if x <= M256:
            br = Branches()
            barrett_ref(x, br)
            if br["sc.corr1"]:
                low256.append(x)
    r256 += low256
    ma = []
    for x in low[:32] + [L * k for k in (1, 2**200, 2**259)]:
        a = rng.randrange((x >> 256) + 1, 2**256)       # so that b = x // a < 2^256
        b, c = divmod(x, a)
        ma.append((a, b, c))
    ma += [(M256, M256, M256), (L - 1, L - 1, L - 1), (0, 0, L), (L, L, L)]
    return {OP_SC_REDUCE512: [(x,) for x in r512], OP_SC_REDUCE256: [(x,) for x in r256], OP_SC_MULADD: ma}


def all_cases():
    c = field_cases()
    c.update(scalar_cases())
    return c


def mismatches(op, items, got, exact=True):
    """Items whose output words differ from the integer result: bit for bit, or (exact=False, for the exponentiation chains
    on random inputs, where replaying 265 multiplies per item in Python is too slow) as the right residue mod p."""
    bad = []
    for x, g in zip(items, got):
        if exact:
            ok = g == expected(op, x)
        elif op == OP_INVERT:
            ok = g < 2**256 and g % P == pow(x[0], P - 2, P)
        elif op == OP_POW22523:
            ok = g < 2**256 and g % P == pow(x[0], (P - 5) // 8, P)
        else:
            raise ValueError(op)
        if not ok:
            bad.append((x, g))
    return bad


def describe(op, bad, n):
    x, g = bad[0]
    return "%s: %d of %d items wrong; first %s -> %#x" % (OP_NAMES[op], len(bad), n, tuple(hex(v) for v in x), g)


def random_items(op, n, seed):
    """n random items for op, every limb 0 with probability 1/16 and all ones with probability 1/8 (as on the device)."""
    rs = np.random.default_rng(seed)
    w = rs.integers(0, 2**32, (n, 32), dtype=np.uint64).astype(np.uint32)
    sel = rs.integers(0, 16, (n, 32))
    w[sel == 0] = 0
    w[(sel == 1) | (sel == 2)] = 0xFFFFFFFF
    return w, unpack_in(op, w)


# tests/devsim/devsim.cu gen_word, for the items whose outputs devsim_bulk keeps
def device_items(op, seed, indices):
    i = np.asarray(indices, dtype=np.uint64)[:, None]
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + i * np.uint64(32) + np.arange(32, dtype=np.uint64)[None, :]
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    sel = z >> np.uint64(60)
    w = (z & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    w[sel == 0] = 0
    w[(sel == 1) | (sel == 2)] = 0xFFFFFFFF
    return unpack_in(op, w)
