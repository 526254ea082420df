"""Cases for the group routines of afc_ge.cuh and the scalar recodings of afc_sc.cuh, and their checks, for the tests/devsim
harness (tests/test_ge_boundaries_hostsim.py on the CPU, tests/test_ge_boundaries_gpu.py on the H100).

Cases are built from Python integers: the torsion points, points with x = 0, projective scales whose limbs sit at the weakly
reduced extremes (value + p, Z = 2^256 - 1), decodings that need the sqrt(-1) correction, keys of every small order.  Every
output is checked by value, never as raw limbs, in two ways:
  * against the same formula replayed on integers mod p (any input, on the curve or not: also the random items), and
  * for constructed points, against the big-integer Edwards arithmetic of oracle/go_ed25519.py (decompress, _ext_add,
    _encode): the affine result, and XY = ZT of a P3 output.
The decoding replay counts the branches of ge_frombytes, and the tests require every one of DECODE_BRANCHES to be taken by
some constructed case."""
import collections
import ctypes
import functools
import os
import random
import subprocess

import numpy as np

from oracle import go_ed25519 as GE

P, L, D = GE.P, GE.L, GE.D
D2 = 2 * D % P
M256 = 2**256 - 1
KC_GMAX, SIGN_GMAX, KR_PARTS, COMB_ROWS, COMB_COLS = 32, 8, 4, 32, 128
KR_SLICE = COMB_COLS // KR_PARTS

# tests/devsim/ge_ops.cuh, enum GeOp
(GE_DECODE, GE_ENCODE, GE_ENCODE_CALL, GE_GROUP_KC, GE_GROUP_SIGN, GE_GROUP_SIGN2, GE_DBL, GE_DBL_CALL, GE_ADDSUB,
 GE_ADDSUB_CALL, GE_TO_PRECOMP, GE_MADD, GE_CT_SELECT, GE_SMALL_MULT, GE_SMALL_MULT_CALL, GE_AFFINE_RUN, GE_AFFINE_RUN_CALL,
 GE_AFFINE_FWDBWD, GE_KEY_ROWS, GE_RECODE, GE_WELLFORMED, GE_OP_COUNT) = range(22)
OP_NAMES = ["decode", "encode", "encode_call", "group_kc", "group_sign", "group_sign2", "dbl", "dbl_call", "addsub",
            "addsub_call", "to_precomp", "madd", "ct_select", "small_mult", "small_mult_call", "affine_run",
            "affine_run_call", "affine_fwdbwd", "key_rows", "recode", "wellformed"]
GMAX = {GE_GROUP_KC: KC_GMAX, GE_GROUP_SIGN: SIGN_GMAX, GE_GROUP_SIGN2: 2 * SIGN_GMAX}
IN_WORDS = {op: 32 for op in range(GE_OP_COUNT)}
IN_WORDS.update({GE_DECODE: 8, GE_ADDSUB: 72, GE_ADDSUB_CALL: 72, GE_MADD: 64, GE_AFFINE_RUN: 64, GE_AFFINE_RUN_CALL: 64,
                 GE_AFFINE_FWDBWD: 64, GE_CT_SELECT: 200, GE_SMALL_MULT: 40, GE_SMALL_MULT_CALL: 40, GE_KEY_ROWS: 16,
                 GE_RECODE: 16, GE_WELLFORMED: 16})
IN_WORDS.update({op: 8 + 24 * g for op, g in GMAX.items()})
OUT_WORDS = {op: 32 for op in range(GE_OP_COUNT)}
OUT_WORDS.update({GE_DECODE: 40, GE_ENCODE: 8, GE_ENCODE_CALL: 8, GE_WELLFORMED: 8, GE_TO_PRECOMP: 24, GE_CT_SELECT: 24,
                  GE_AFFINE_RUN: 64 * 24 + 32, GE_AFFINE_RUN_CALL: 64 * 24 + 32, GE_AFFINE_FWDBWD: KR_SLICE * 24 + 32,
                  GE_KEY_ROWS: 8 + 2 * COMB_COLS * 24, GE_RECODE: 80})
OUT_WORDS.update({op: 8 * g for op, g in GMAX.items()})
RUN_LEN = {GE_AFFINE_RUN: 64, GE_AFFINE_RUN_CALL: 64, GE_AFFINE_FWDBWD: KR_SLICE}
# GE_RECODE kind -> (digit width, digits); kinds 16..22 are sc_recode_wide at w = kind
FIXED_RADIX = {0: (4, 64), 1: (8, 32), 2: (16, 16)}
RECODE_KINDS = [0, 1, 2] + list(range(16, 23))

DECODE_BRANCHES = {
    "decode.ok_pos": "v r^2 = u: the first root is right",
    "decode.sqrtm1": "v r^2 = -u only: the root is multiplied by sqrt(-1)",
    "decode.flip": "the root's parity differs from the sign bit: negated",
    "decode.reject": "u / v is not a square: no point",
    "decode.u0": "u = 0 (y = +-1): x = 0",
}


class Branches(collections.Counter):
    def hit(self, name, cond=True):
        if cond:
            self[name] += 1


NOBR = Branches()


# ----------------------------------------------------------------------------------------------- words
def words(v, n=8):
    return np.frombuffer(int(v).to_bytes(4 * n, "little"), dtype="<u4").astype(np.uint32)


def get(row, off, n=8):
    return int.from_bytes(np.ascontiguousarray(row[off:off + n], dtype="<u4").tobytes(), "little")


def put(row, off, v, n=8):
    row[off:off + n] = words(v, n)


def s32(v):
    return (int(v) ^ 0x80000000) - 0x80000000


# ----------------------------------------------------------------------------------------------- integer arithmetic
def inv(z):
    """z^-1 mod p, and 0 for z = 0 mod p (what z^(p-2), the device's inversion, gives)."""
    z %= P
    return pow(z, -1, P) if z else 0


def aff(ext):
    zi = inv(ext[2])
    return ext[0] * zi % P, ext[1] * zi % P


def add(a, b):
    return aff(GE._ext_add(GE._ext(a), GE._ext(b)))


def neg(a):
    return (-a[0]) % P, a[1]


def mul(k, a):
    return aff(GE._ext_mul(k, GE._ext(a)))


def precomp(a):
    x, y = a
    return (y + x) % P, (y - x) % P, 2 * D * x * y % P


IDENT = (0, 1)
B = GE.BASE


def decode(enc):
    return GE.decompress(int(enc).to_bytes(32, "little"))


def encode_int(pt):
    return int.from_bytes(GE._encode(GE._ext(pt)), "little")


# the formulas of afc_ge.cuh replayed mod p, on raw inputs (any 256-bit limbs, on the curve or not)
def _p1p1_to_p3(rX, rY, rZ, rT):
    return rX * rT % P, rY * rZ % P, rZ * rT % P, rX * rY % P


def r_dbl(X, Y, Z):
    xx, yy, b, a = X * X, Y * Y, 2 * Z * Z, (X + Y) ** 2
    rY, rZ = yy + xx, yy - xx
    return _p1p1_to_p3(a - rY, rY, rZ, b - rZ)


def r_cached(p3):
    X, Y, Z, T = p3
    return (Y + X) % P, (Y - X) % P, Z % P, T * D2 % P


def _finish(a, b, d, c, neg_):
    dpc, dmc = d + c, d - c
    rZ, rT = (dmc, dpc) if neg_ else (dpc, dmc)
    return _p1p1_to_p3(a - b, a + b, rZ, rT)


def r_addsub(p3, c, neg_):
    X, Y, Z, T = p3
    qa, qb = (c[1], c[0]) if neg_ else (c[0], c[1])
    return _finish((Y + X) * qa, (Y - X) * qb, 2 * Z * c[2], c[3] * T, neg_)


def r_madd(p3, e, neg_):
    X, Y, Z, T = p3
    qa, qb = (e[1], e[0]) if neg_ else (e[0], e[1])
    return _finish((Y + X) * qa, (Y - X) * qb, 2 * Z, e[2] * T, neg_)


def r_precomp(p3):
    zi = inv(p3[2])
    x, y = p3[0] * zi % P, p3[1] * zi % P
    return (y + x) % P, (y - x) % P, x * y % P * D2 % P


def r_encode(X, Y, Z):
    zi = inv(Z)
    x, y = X * zi % P, Y * zi % P
    return y | (x & 1) << 255


def r_small(p3, m):
    c = r_cached(p3)
    M, started = p3, False
    for bit in range(21, -1, -1):
        if started:
            M = r_dbl(*M[:3])
        if m >> bit & 1:
            if started:
                M = r_addsub(M, c, 0)
            else:
                M, started = p3, True
    return M


def r_affine(M, p3, ch, full):
    """ge_affine_run (full: M advances CH times) or ge_affine_run_fwd (CH - 1 times): entries and the final M."""
    c = r_cached(p3)
    recs = []
    for j in range(ch):
        recs.append(M)
        if full or j + 1 < ch:
            M = r_addsub(M, c, 0)
    return [r_precomp(r) for r in recs], M


def decode_replay(enc, br=NOBR):
    """ge_frombytes on integers, counting its branches: (x, y) or None."""
    sign = enc >> 255
    y = (enc & (2**255 - 1)) % P
    u, v = (y * y - 1) % P, (D * y * y + 1) % P
    v3 = v * v % P * v % P
    r = u * v3 % P * pow(u * v3 % P * v3 % P * v % P, (P - 5) // 8, P) % P
    chk = v * r % P * r % P
    ok_pos, ok_neg = chk == u, chk == (-u) % P
    br.hit("decode.u0", u == 0)
    br.hit("decode.ok_pos", ok_pos)
    if ok_neg and not ok_pos:
        br.hit("decode.sqrtm1")
        r = r * GE.SQRT_M1 % P
    if not (ok_pos or ok_neg):
        br.hit("decode.reject")
        return None
    if (r & 1) != sign:
        br.hit("decode.flip")
        r = (-r) % P
    return r, y


# ----------------------------------------------------------------------------------------------- recodings
def recode_geometry(kind):
    """(w, digits, offset C, wide) of a GE_RECODE kind, from the stated definitions."""
    if kind in FIXED_RADIX:
        w, n = FIXED_RADIX[kind]
        return w, n, sum(1 << (w * i + w - 1) for i in range(n)), False
    w = kind
    rows = (254 + w - 1) // w
    return w, rows, sum(1 << (w * i + w - 1) for i in range(rows - 1)), True


def top_max(w):
    """The largest top digit of sc_recode_wide over every s < 2^253, from integers: the top digit grows with s."""
    _, rows, c, _ = recode_geometry(w)
    return (2**253 - 1 + c) >> (w * (rows - 1))


def table_entries(w):
    _, rows, _, _ = recode_geometry(w)
    return (rows - 1) * (1 << (w - 1)) + (top_max(w) + 63) // 64 * 64


def recode_scalars(kind):
    """0, 1, L - 1, 2^252, 2^253 - 1 (and 2^254 - 1 for the fixed radixes), scalars whose digits are all -2^(w-1), all
    2^(w-1) - 1 or alternate between the two, scalars whose carry runs into the top digit, and random ones."""
    w, n, c, wide = recode_geometry(kind)
    bound = 2**253 if wide else 2**254
    out = [0, 1, L - 1, 2**252, 2**253 - 1] + ([] if wide else [2**254 - 1])
    lo, hi = -(1 << (w - 1)), (1 << (w - 1)) - 1
    top = 1 << (w * (n - 1))
    for pat in ([lo] * (n - 1), [hi] * (n - 1), [lo, hi] * n, [hi, lo] * n):
        low = sum(d << (w * i) for i, d in enumerate(pat[:n - 1]))
        for t in range(0, 4):
            s = low + t * top
            if 0 <= s < bound:
                out.append(s)
    for k in (1, 2, 3):           # s + C carries through every digit below the top
        for d in (-1, 0, 1):
            s = k * top - (c % top) + d
            if 0 <= s < bound:
                out.append(s)
            s = k * top - 1 + d
            if 0 <= s < bound:
                out.append(s)
    rng = random.Random(kind)
    out += [rng.randrange(bound) for _ in range(16)] + [rng.randrange(L) for _ in range(8)]
    return sorted(set(out))


# ----------------------------------------------------------------------------------------------- constructed cases
SCALES = 5


def proj(pt, kind, rng):
    """(X, Y, Z, T) raw limbs of an affine point: 0 Z = 1; 1 random Z; 2 random Z, every coordinate + p; 3 Z = 2^256 - 1
    (the value 37), the others + p; 4 Z = 1, every coordinate + p (so Y Z^-1 keeps the non-canonical limbs y + p)."""
    x, y = pt
    if kind in (0, 4):
        z, zraw = 1, 1 + (P if kind == 4 else 0)
    elif kind == 3:
        z, zraw = 37, M256
    else:
        z = rng.randrange(1, P)
        zraw = z + (P if kind == 2 else 0)
    co = [x * z % P, y * z % P, x * y % P * z % P]
    if kind in (2, 3, 4):
        co = [v + P for v in co]
    return co[0], co[1], zraw, co[2]


def put_p3(row, off, p3):
    for k, v in enumerate(p3):
        put(row, off + 8 * k, v)


def _row(op):
    return np.zeros(IN_WORDS[op], dtype=np.uint32)


@functools.lru_cache(maxsize=None)
def torsion():
    """The 8 points of order dividing 8, identity first."""
    return [decode(int.from_bytes(e, "little")) for e in GE.small_order_points()]


@functools.lru_cache(maxsize=None)
def group_points():
    """The identity and the 7 other torsion points, B, -B, B + T for each T != O, a random P and -P."""
    rng = random.Random(0x6E)
    T = torsion()
    R = mul(rng.randrange(1, L), B)
    return T + [B, neg(B)] + [add(B, t) for t in T[1:]] + [R, neg(R)]


def decode_cases(rng):
    encs = []
    for e in GE.small_order_points():
        y = int.from_bytes(e, "little") & (2**255 - 1)
        for s in (0, 1):
            encs.append(y | s << 255)
            if y + P < 2**255:
                encs.append((y + P) | s << 255)
    for y in list(range(19)) + [P - 1, P - 2]:
        for s in (0, 1):
            encs.append(y | s << 255)
            if y + P < 2**255:
                encs.append((y + P) | s << 255)
    for pt in group_points():
        encs.append(encode_int(pt))
    need = {"decode.reject": 64, "decode.sqrtm1": 64, "decode.ok_pos": 64}
    got = Branches()
    while any(got[k] < v for k, v in need.items()):
        enc = rng.getrandbits(256)
        br = Branches()
        decode_replay(enc, br)
        for k in need:
            if br[k] and got[k] < need[k]:
                got[k] += 1
                encs.append(enc)
                break
    out = []
    for enc in encs:
        row = _row(GE_DECODE)
        put(row, 0, enc)
        out.append((row, None))
    return out


def _pairs_p3(op, rng, pts, extra):
    out = []
    for i, a in enumerate(pts):
        for j, b in enumerate(pts):
            for ng in (0, 1):
                for e in extra:
                    row = _row(op)
                    put_p3(row, 0, proj(a, (i + j + ng) % SCALES, rng))
                    out.append((row, a, b, ng, e))
    return out


def point_cases(rng):
    pts = group_points()
    cases = collections.defaultdict(list)
    for op in (GE_DBL, GE_DBL_CALL, GE_TO_PRECOMP, GE_ENCODE, GE_ENCODE_CALL):
        for a in pts:
            for k in range(SCALES):
                row = _row(op)
                put_p3(row, 0, proj(a, k, rng))
                cases[op].append((row, add(a, a) if op in (GE_DBL, GE_DBL_CALL) else a))
    for op in (GE_ADDSUB, GE_ADDSUB_CALL):
        for row, a, b, ng, _ in _pairs_p3(op, rng, pts, (None,)):
            put_p3(row, 32, proj(b, rng.randrange(SCALES), rng))
            row[64] = ng
            cases[op].append((row, add(a, neg(b) if ng else b)))
    for row, a, b, ng, mode in _pairs_p3(GE_MADD, rng, pts, (0, 1)):
        e = precomp(b)
        if rng.random() < 0.5:
            e = tuple(v + P for v in e)          # weakly reduced entry limbs
        for k, v in enumerate(e):
            put(row, 32 + 8 * k, v)
        row[56], row[57] = ng, mode
        cases[GE_MADD].append((row, add(a, neg(b) if ng else b)))
    return cases


def group_cases(rng):
    """Groups at every G <= GMAX: the identity, x = 0 points (y = +-1), torsion points, non-canonical y limbs, random points,
    the padding members the kernels insert past n (X = 0, Y = Z = 1), and garbage past G."""
    T = torsion()
    pool = T + [B, neg(B)] + [mul(rng.randrange(1, L), B) for _ in range(6)]
    out = collections.defaultdict(list)
    for op, gmax in GMAX.items():
        for G in range(1, gmax + 1):
            for variant in range(3):
                row = _row(op)
                row[0] = G
                exp = []
                npad = 0 if variant == 0 else rng.randint(1, G)
                for g in range(gmax):
                    off = 8 + 24 * g
                    if g >= G:                              # not part of the group: garbage, Z = 0 included
                        row[off:off + 24] = np.array([rng.getrandbits(32) for _ in range(24)], dtype=np.uint32)
                        if rng.random() < 0.3:
                            row[off + 16:off + 24] = 0
                        continue
                    if g >= G - npad:
                        X, Y, Z = 0, 1, 1
                        exp.append(1)
                    else:
                        a = pool[rng.randrange(len(pool))] if variant != 2 else pool[g % len(pool)]
                        X, Y, Z, _ = proj(a, rng.randrange(SCALES), rng)
                        exp.append(encode_int(a))
                    for k, v in enumerate((X, Y, Z)):
                        put(row, off + 8 * k, v)
                out[op].append((row, exp))
    return out


def ct_select_cases(rng):
    out = []
    Q = mul(rng.randrange(1, L), B)
    rows = [[precomp(mul(j + 1, B)) for j in range(8)], [precomp(mul(j + 1, Q)) for j in range(8)],
            [tuple(v + P for v in precomp(mul(j + 1, Q))) for j in range(8)],
            [tuple(rng.getrandbits(256) for _ in range(3)) for _ in range(8)]]
    for entries in rows:
        for d in range(-8, 9):
            row = _row(GE_CT_SELECT)
            for j, e in enumerate(entries):
                for k, v in enumerate(e):
                    put(row, 24 * j + 8 * k, v)
            row[192] = d & 0xFFFFFFFF
            out.append((row, None))
    return out


def small_mult_cases(rng):
    out = collections.defaultdict(list)
    T = torsion()
    pts = [B, T[4], T[1], IDENT, add(B, T[6]), mul(rng.randrange(1, L), B)]
    ms = [1, 2, 3, 127, 128, 255, 2**21 - 1, 2**21, 2**21 + 1, 2**22 - 2, 2**22 - 1, 0x155555, 0x2AAAAA]
    ms += [rng.randrange(2**21, 2**22) for _ in range(4)]
    for op in (GE_SMALL_MULT, GE_SMALL_MULT_CALL):
        for i, a in enumerate(pts):
            for j, m in enumerate(ms):
                row = _row(op)
                put_p3(row, 0, proj(a, (i + j) % SCALES, rng))
                row[32] = m
                out[op].append((row, mul(m, a)))
    return out


def affine_cases(rng):
    out = collections.defaultdict(list)
    T = torsion()
    R = mul(rng.randrange(1, L), B)
    combos = [(B, B), (R, mul(33, R)), (R, IDENT), (add(B, T[5]), T[2]), (T[4], T[7]), (IDENT, IDENT), (B, neg(B)),
              (R, mul(rng.randrange(1, L), B))]
    for op, ch in RUN_LEN.items():
        for i, (p, m) in enumerate(combos):
            row = _row(op)
            put_p3(row, 0, proj(m, i % SCALES, rng))
            put_p3(row, 32, proj(p, (i + 2) % SCALES, rng))
            exp, cur = [], m
            for _ in range(ch):
                exp.append(cur)
                cur = add(cur, p)
            final = cur if op != GE_AFFINE_FWDBWD else exp[-1]
            out[op].append((row, (exp, final)))
    return out


def key_list(rng):
    """(name, encoding): the identity and every small-order point, their non-canonical encodings, mixed-order keys, one
    undecodable key and two honest keys."""
    keys = [("torsion%d" % i, int.from_bytes(e, "little")) for i, e in enumerate(GE.small_order_points())]
    keys += [("y=0+p", P), ("y=0+p,sign", P | 1 << 255), ("y=1+p", P + 1), ("y=1+p,sign", (P + 1) | 1 << 255),
             ("y=1,sign", 1 | 1 << 255), ("y=p-1,sign", (P - 1) | 1 << 255)]
    A = decode(int.from_bytes(GE.public_key(bytes(range(32))), "little"))
    T = torsion()
    keys += [("A+T%d" % i, encode_int(add(A, T[i]))) for i in (1, 2, 5)]
    while True:
        enc = rng.getrandbits(255)
        if decode(enc) is None:
            keys.append(("undecodable", enc))
            break
    keys += [("honest%d" % i, int.from_bytes(GE.public_key(bytes([i + 7]) * 32), "little")) for i in range(2)]
    return keys


@functools.lru_cache(maxsize=4096)
def key_row_expect(enc, row):
    """The 128 entries of row `row` of the table of key `enc`: (j+1) 256^row (-A) in precomputed form, one addition each."""
    A = decode(enc)
    base = GE._ext_mul(256**row, GE._ext(neg(A)))
    out, cur = [], base
    for _ in range(COMB_COLS):
        out.append(precomp(aff(cur)))
        cur = GE._ext_add(cur, base)
    return tuple(out)


def key_row_cases(rng):
    out = []
    for _, enc in key_list(rng):
        for r in (0, 1, 2, 31):
            for stages in (1, 2, 4):
                row = _row(GE_KEY_ROWS)
                put(row, 0, enc)
                row[8], row[9] = r, stages
                out.append((row, None))
    return out


def recode_cases():
    out = []
    for kind in RECODE_KINDS:
        for s in recode_scalars(kind):
            row = _row(GE_RECODE)
            put(row, 0, s)
            row[8] = kind
            out.append((row, None))
    return out


def wellformed_cases(rng):
    out = []
    for S in (L - 1, L, L + 1, 2**253 - 1, 2**256 - 1, 0, 2**252):
        for bits in range(8):
            s = (S & (2**253 - 1)) | bits << 253
            row = _row(GE_WELLFORMED)
            put(row, 0, rng.getrandbits(256))
            put(row, 8, s)
            out.append((row, None))
    return out


def all_cases(seed=0x6E25519):
    """{op: [(input row, expectation or None)]}."""
    rng = random.Random(seed)
    cases = collections.defaultdict(list)
    cases[GE_DECODE] = decode_cases(rng)
    for part in (point_cases(rng), group_cases(rng), small_mult_cases(rng), affine_cases(rng)):
        for op, items in part.items():
            cases[op] += items
    cases[GE_CT_SELECT] = ct_select_cases(rng)
    cases[GE_KEY_ROWS] = key_row_cases(rng)
    cases[GE_RECODE] = recode_cases()
    cases[GE_WELLFORMED] = wellformed_cases(rng)
    return cases


def pack(op, items):
    return np.ascontiguousarray(np.stack([r for r, _ in items]), dtype=np.uint32)


# ----------------------------------------------------------------------------------------------- checks
def _p3_err(y, off, want, exp):
    """A P3 output against the replayed formula (mod p) and, for constructed cases, the affine group element exp."""
    got = tuple(get(y, off + 8 * k) % P for k in range(4))
    if got != tuple(v % P for v in want):
        return "P3 %s != replay %s" % (tuple(map(hex, got)), tuple(map(hex, want)))
    if exp is not None:
        X, Y, Z, T = got
        if Z == 0 or (X * inv(Z) % P, Y * inv(Z) % P) != tuple(exp) or X * Y % P != Z * T % P:
            return "P3 %s is not the group element %s" % (tuple(map(hex, got)), tuple(map(hex, exp)))
    return None


def _entries_err(y, off, want, n):
    for j in range(n):
        got = tuple(get(y, off + 24 * j + 8 * k) % P for k in range(3))
        if got != tuple(v % P for v in want[j]):
            return "entry %d: %s != %s" % (j, tuple(map(hex, got)), tuple(map(hex, want[j])))
    return None


def _p3_in(x, off):
    return tuple(get(x, off + 8 * k) for k in range(4))


def check(op, x, y, exp=None):
    """None if output words y are right for input words x, else what is wrong.  exp: the constructed case's expectation."""
    if op == GE_DECODE:
        enc = get(x, 0)
        want = decode(enc)
        if int(y[32]) != (want is not None) or y[33:40].any():
            return "ok = %d, oracle %s" % (int(y[32]), want)
        if want is not None:
            X, Y, Z, T = (get(y, 8 * k) % P for k in range(4))
            if (X, Y, Z, T) != (want[0], want[1], 1, want[0] * want[1] % P):
                return "decoded %s, oracle %s" % ((hex(X), hex(Y), hex(Z), hex(T)), want)
        return None
    if op in (GE_ENCODE, GE_ENCODE_CALL):
        want = r_encode(*_p3_in(x, 0)[:3])
        if exp is not None and want != encode_int(exp):
            return "constructed point scaled wrong"
        return None if get(y, 0) == want else "encoding %#x != %#x" % (get(y, 0), want)
    if op in GMAX:
        G = int(x[0])
        for g in range(GMAX[op]):
            o = 8 + 24 * g
            want = r_encode(get(x, o), get(x, o + 8), get(x, o + 16)) if g < G else 0
            if g < G and exp is not None and want != exp[g]:
                return "constructed member %d scaled wrong" % g
            if get(y, 8 * g) != want:
                return "G = %d, member %d: %#x != %#x" % (G, g, get(y, 8 * g), want)
        return None
    if op in (GE_DBL, GE_DBL_CALL):
        return _p3_err(y, 0, r_dbl(*_p3_in(x, 0)[:3]), exp)
    if op in (GE_ADDSUB, GE_ADDSUB_CALL):
        return _p3_err(y, 0, r_addsub(_p3_in(x, 0), r_cached(_p3_in(x, 32)), int(x[64])), exp)
    if op == GE_TO_PRECOMP:
        want = r_precomp(_p3_in(x, 0))
        if exp is not None and want != precomp(exp):
            return "constructed point scaled wrong"
        return _entries_err(y, 0, [want], 1)
    if op == GE_MADD:
        e = tuple(get(x, 32 + 8 * k) for k in range(3))
        return _p3_err(y, 0, r_madd(_p3_in(x, 0), e, int(x[56])), exp)
    if op == GE_CT_SELECT:
        d = s32(x[192])
        got = tuple(get(y, 8 * k) for k in range(3))
        if d == 0:
            ok = got == (1, 1, 0)
        else:
            e = tuple(get(x, 24 * (abs(d) - 1) + 8 * k) for k in range(3))
            ok = got == e if d > 0 else (got[0], got[1]) == (e[1], e[0]) and got[2] % P == (-e[2]) % P
        return None if ok else "d = %d: %s" % (d, tuple(map(hex, got)))
    if op in (GE_SMALL_MULT, GE_SMALL_MULT_CALL):
        return _p3_err(y, 0, r_small(_p3_in(x, 0), int(x[32])), exp)
    if op in RUN_LEN:
        ch = RUN_LEN[op]
        want, final = r_affine(_p3_in(x, 0), _p3_in(x, 32), ch, op != GE_AFFINE_FWDBWD)
        if exp is not None:
            if [precomp(a) for a in exp[0]] != list(want):
                return "constructed run scaled wrong"
        err = _entries_err(y, 0, want, ch) or _p3_err(y, 24 * ch, final, None if exp is None else exp[1])
        return err
    if op == GE_KEY_ROWS:
        enc, r = get(x, 0), int(x[8])
        A = decode(enc)
        if (int(y[0]), int(y[1])) != ((A is not None),) * 2 or y[2:8].any():
            return "ok = %d, %d for a key that %s" % (int(y[0]), int(y[1]), "decodes" if A else "does not decode")
        if A is None:           # the staged build walks the neutral element; ge_build_key_row's table is never read
            return _entries_err(y, 8, [(1, 1, 0)] * COMB_COLS, COMB_COLS)
        want = key_row_expect(enc, r)
        e1 = _entries_err(y, 8, want, COMB_COLS)
        e2 = _entries_err(y, 8 + 24 * COMB_COLS, want, COMB_COLS)
        return ("staged build: " + e1) if e1 else ("ge_build_key_row: " + e2) if e2 else None
    if op == GE_RECODE:
        return recode_err(get(x, 0), int(x[8]), y)
    if op == GE_WELLFORMED:
        s = get(x, 8)
        want = int(s >> 253 == 0 and s < L)
        return None if (int(y[0]), y[1:].any()) == (want, False) else "S = %#x: %d" % (s, int(y[0]))
    raise ValueError(op)


def recode_err(s, kind, y):
    w, n, c, wide = recode_geometry(kind)
    t = get(y, 0)
    if t != (s + c) & M256:
        return "t = %#x, want s + C = %#x" % (t, (s + c) & M256)
    d = [s32(v) for v in y[8:8 + n]]
    if y[8 + n:72].any():
        return "words past the %d digits" % n
    if sum(v << (w * i) for i, v in enumerate(d)) != s:
        return "digits %s do not sum to s = %#x" % (d, s)
    lo, hi = -(1 << (w - 1)), (1 << (w - 1)) - 1
    body = d[:-1] if wide else d
    if any(not lo <= v <= hi for v in body):
        return "digit out of [%d, %d]: %s" % (lo, hi, d)
    if wide:
        if not 0 <= d[-1] <= top_max(w):
            return "top digit %d outside [0, %d]" % (d[-1], top_max(w))
        if (int(y[72]), get(y, 73, 2)) != (top_max(w), table_entries(w)):
            return "base_table_top_max / entries = %d / %d, want %d / %d" % (int(y[72]), get(y, 73, 2), top_max(w),
                                                                              table_entries(w))
    elif y[72:].any():
        return "table geometry words set for a fixed radix"
    return None


def mismatches(op, x, y, exps=None):
    bad = []
    for i in range(len(x)):
        err = check(op, x[i], y[i], None if exps is None else exps[i])
        if err:
            bad.append((i, err))
    return bad


def describe(op, bad, n, x):
    i, err = bad[0]
    return "%s: %d of %d items wrong; first (item %d, input %s...): %s" % (
        OP_NAMES[op], len(bad), n, i, " ".join("%08x" % v for v in x[i][:16]), err)


# ----------------------------------------------------------------------------------------------- the harness libraries
def check_widths(lib):
    """Refuse a harness library built with another numbering or item layout."""
    assert lib.ge_op_count() == GE_OP_COUNT
    for op in range(GE_OP_COUNT):
        assert (lib.ge_words(op, 0), lib.ge_words(op, 1)) == (IN_WORDS[op], OUT_WORDS[op]), OP_NAMES[op]


def build_host_lib(tmp_dir):
    """tests/devsim/ge_host.cpp (the portable twins) compiled into tmp_dir and loaded."""
    out = os.path.join(tmp_dir, "libafc_ge_host.so")
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "devsim", "ge_host.cpp")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out, src])
    lib = ctypes.CDLL(out)
    lib.ge_run.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64]
    check_widths(lib)
    return lib


def run(lib, op, x):
    """Output words of op over input rows x through a harness library's ge_run."""
    x = np.ascontiguousarray(x, dtype=np.uint32)
    y = np.zeros((len(x), OUT_WORDS[op]), dtype=np.uint32)
    assert lib.ge_run(op, x.ctypes.data, y.ctypes.data, len(x)) == 0, OP_NAMES[op]
    return y


# ----------------------------------------------------------------------------------------------- device generator
def shape(op, w):
    """tests/devsim/ge.cu ge_shape: random words into the operation's domain (in place)."""
    if op in GMAX:
        w[:, 0] = 1 + w[:, 0] % GMAX[op]
    elif op in (GE_ADDSUB, GE_ADDSUB_CALL):
        w[:, 64] &= 1
    elif op == GE_MADD:
        w[:, 56] &= 1
        w[:, 57] &= 1
    elif op == GE_CT_SELECT:
        w[:, 192] = ((w[:, 192] % 17).astype(np.int64) - 8).astype(np.uint32)
    elif op in (GE_SMALL_MULT, GE_SMALL_MULT_CALL):
        w[:, 32] = 1 + w[:, 32] % (2**22 - 1)
    elif op == GE_KEY_ROWS:
        w[:, 8] %= COMB_ROWS
        w[:, 9] = np.left_shift(1, w[:, 9] % 3).astype(np.uint32)
    elif op == GE_RECODE:
        k = w[:, 8] % 10
        w[:, 8] = np.where(k < 3, k, k + 13)
        w[:, 7] &= np.where(k < 3, 0x3FFFFFFF, 0x1FFFFFFF).astype(np.uint32)
    return w


def device_items(op, seed, indices):
    """The input words tests/devsim/ge.cu generates for items `indices` (gen_word, then ge_shape)."""
    n = IN_WORDS[op]
    i = np.asarray(indices, dtype=np.uint64)[:, None]
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + i * np.uint64(1024) + np.arange(n, dtype=np.uint64)[None, :]
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    sel = z >> np.uint64(60)
    w = (z & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    w[sel == 0] = 0
    w[(sel == 1) | (sel == 2)] = 0xFFFFFFFF
    return np.ascontiguousarray(shape(op, w))
