"""SHA-512 of prefix || message (afc_sha.cuh, sha512_prefixed), CPU build of the kernel code, against hashlib: around every
length at which the last block of a 16-byte-aligned message changes shape (the 0x80 byte at the end of a word, the length
spilling into a block of its own at 112 tail bytes, tails of 0 and 127 bytes), for both prefix sizes, aligned and unaligned."""
import ctypes as C
import hashlib

import numpy as np


def _placed(raw, al):
    """raw at byte offset al of a 16-byte-aligned buffer whose other bytes are 0xa5, so that bytes read past the end and not
    masked off change the digest."""
    base = np.full(len(raw) + 64, 0xA5, dtype=np.uint8)
    a0 = (-base.ctypes.data) % 16
    base[a0 + al:a0 + al + len(raw)] = np.frombuffer(raw, dtype=np.uint8)
    return base, C.cast(base.ctypes.data + a0 + al, C.POINTER(C.c_uint8))


def _lengths(m0):
    """Message lengths whose bytes after block 0 (m0 of them share it with the prefix) end at each tail shape."""
    tails = (0, 1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 110, 111, 112, 113, 119, 120, 127)
    return sorted({m0 + 128 * full + t for full in (0, 1, 3, 4) for t in tails} | set(range(0, m0 + 1)) |
                  {511, 512, 513, 575, 576, 577})


def test_sha512_prefixed_lean_tail_and_general_path(hostsim):
    rng = np.random.default_rng(0x5A12)
    for fn, plen in ((hostsim.hs_sha512_pre64, 64), (hostsim.hs_sha512_pre32, 32)):
        pre = rng.integers(0, 256, plen, dtype=np.uint8).tobytes()
        for n in _lengths(128 - plen):
            for al in (0, 4, 5, 13):
                m = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
                keep, p = _placed(m, al)
                o = (C.c_uint8 * 64)()
                fn(pre, p, C.c_uint64(n), o)
                assert bytes(o) == hashlib.sha512(pre + m).digest(), (plen, n, al)
