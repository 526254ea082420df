"""The table-driven verify through its radix-2^w fixed-base table, at every window AFC_VERIFY_BASE_WINDOW accepts (16 is the
radix-65536 table that also serves when a wider one cannot be allocated), bit for bit against the oracle.

A key at the identity point makes [k](-A) vanish, so the signature (enc([S]B), S) is valid for every S < L and every message (Go
accepts small-order keys): that puts chosen scalars S — every digit at its extreme, carries into the top row, a zero digit in each
row — through the fixed-base half of the kernel.  The Go edge set and honest random signatures ride in the same batches, through
the transparent issuer-key cache and through an explicit key set."""
import numpy as np
import pytest

from conftest import golden
from oracle import c_oracle as CO, go_ed25519 as G
from wide_base_cases import WINDOWS, scalars

pytestmark = pytest.mark.gpu

IDENTITY = (1).to_bytes(32, "little")


def _batch(w, ctx):
    pks, sigs, msgs = [], [], []
    for name, s in scalars(w).items():
        r = G._encode(G._ext_mul(s, G._BASE_EXT))
        sb = s.to_bytes(32, "little")
        for m, sig in ((name.encode(), r + sb),                                   # valid
                       (b"R" + name.encode(), bytes([r[0] ^ 1]) + r[1:] + sb),    # R off by one bit
                       (b"S" + name.encode(), r + ((s + 1) % G.L).to_bytes(32, "little"))):
            pks.append(IDENTITY); sigs.append(sig); msgs.append(m)
    pks, sigs, msgs = pks * 2, sigs * 2, msgs * 2                 # >= 48 credentials: the identity key gets a table
    for e in golden("ed25519_edge.json") * 60:
        pks.append(bytes.fromhex(e["pk"])); sigs.append(bytes.fromhex(e["sig"])); msgs.append(bytes.fromhex(e["msg"]))
    rng = np.random.default_rng(0xAF22 + w)
    seeds = rng.integers(0, 256, (2, 32), dtype=np.uint8)
    kp = ctx.pubkeys(seeds)
    for i in range(160):
        m = rng.integers(0, 256, int(rng.integers(0, 700)), dtype=np.uint8).tobytes()
        pks.append(bytes(kp[i % 2])); msgs.append(m)
        sigs.append(G.sign(bytes(seeds[i % 2]), m))
    from agentfield_b200 import pack
    buf, off = pack(msgs)
    P = np.frombuffer(b"".join(pks), dtype=np.uint8).reshape(-1, 32).copy()
    S = np.frombuffer(b"".join(sigs), dtype=np.uint8).reshape(-1, 64).copy()
    first = 6 * len(scalars(w))
    S[first + 5::13, 40] ^= 0x20                                  # corruption in S of the edge and random signatures
    return pks, P, S, buf, off


@pytest.mark.parametrize("w", WINDOWS)
def test_wide_base_table_verify_matches_oracle(w, monkeypatch):
    import agentfield_b200 as afb
    from agentfield_b200 import KeySet
    monkeypatch.setenv("AFC_VERIFY_BASE_WINDOW", str(w))
    ctx = afb.Context(0)
    try:
        pks, P, S, buf, off = _batch(w, ctx)
        exp = CO.ed25519_verify_batch(P, S, buf, off, 8)
        n_named = 3 * len(scalars(w))
        assert exp[:n_named:3].all() and not exp[1:n_named:3].any() and not exp[2:n_named:3].any()
        got = ctx.verify_packed(P, S, buf, off)
        st = ctx.keycache_stats()
        assert st["last_cold"] == 0 and st["last_hot"] == len(pks)            # every credential went through a table
        assert st["base_window"] == w
        assert (st["base_table_bytes"] > 0) == (w != 16)
        assert (got == exp).all(), np.nonzero(got != exp)[0][:20]
        uniq = sorted(set(pks))
        ks = KeySet(uniq, ctx)
        ki = np.array([uniq.index(p) for p in pks], dtype=np.uint32)
        assert (ks.verify_packed(ki, S, buf, off) == exp).all()
        ks.close()
    finally:
        ctx.close()


def test_verify_window_knob_default_and_out_of_range(monkeypatch):
    """An out-of-range AFC_VERIFY_BASE_WINDOW keeps the compiled default; before the first table-driven verify nothing is allocated."""
    import agentfield_b200 as afb
    monkeypatch.setenv("AFC_VERIFY_BASE_WINDOW", "23")
    ctx = afb.Context(0)
    try:
        st = ctx.keycache_stats()
        assert 16 <= st["base_window"] <= 22 and st["base_table_bytes"] == 0
    finally:
        ctx.close()
