"""Host-side mirror of the Go `pkg/crypto` interfaces this build adds to the reference (SURVEY.md §8b):

    type Signer   interface{ SignBatch(seeds [][32]byte, msgs [][]byte) ([][64]byte, error) }
    type Verifier interface{ VerifyBatch(pks [][32]byte, msgs [][]byte, sigs [][64]byte) ([]bool, error) }
    type MAC      interface{ HMACSHA256Batch(keys, msgs [][]byte) ([][32]byte, error) }
    type Hasher   interface{ SHA256Batch(msgs [][]byte) ([][32]byte, error) }

Same names (snake_cased), argument meaning and error behaviour; all arithmetic runs in
libafcrypto.so's sm_90a kernels through the C ABI (agentfield_b200/_abi.py).  The Go source of the
real adapter is under go/; this module is what the parity tests and bench.py drive because the image
has no Go toolchain.

Error behaviour mirrored from Go:
  * ed25519.Verify panics when len(publicKey) != 32  -> ValueError here (before anything is packed);
  * len(sig) != 64 is simply "false"                  -> that item is reported False;
  * ed25519.NewKeyFromSeed panics when len(seed) != 32 -> ValueError.
"""
import ctypes as C

import numpy as np

from . import _abi


def pack(msgs):
    """[bytes] -> (uint8 buffer, uint64 offsets[n+1]) — the packed layout of include/afcrypto.h."""
    n = len(msgs)
    off = np.zeros(n + 1, dtype=np.uint64)
    if n:
        off[1:] = np.cumsum(np.fromiter((len(m) for m in msgs), dtype=np.uint64, count=n))
    buf = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy() if n and off[-1] else np.zeros(1, dtype=np.uint8)
    return buf, off


def pack32(keys):
    n = len(keys)
    off = np.zeros(n + 1, dtype=np.uint32)
    if n:
        off[1:] = np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=n)).astype(np.uint32)
    buf = np.frombuffer(b"".join(keys), dtype=np.uint8).copy() if n and off[-1] else np.zeros(1, dtype=np.uint8)
    return buf, off


class Context:
    """One afc_ctx per GPU (afc_init / afc_destroy)."""

    def __init__(self, device=0):
        self._lib = _abi.load()
        h = C.c_void_p()
        _abi.check(self._lib.afc_init(int(device), C.byref(h)))
        self.handle = h
        self.device = int(device)

    def close(self):
        if getattr(self, "handle", None):
            self._lib.afc_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- facts
    def device_info(self):
        sm, khz, mem = C.c_int(), C.c_int(), C.c_uint64()
        _abi.check(self._lib.afc_device_info(self.handle, C.byref(sm), C.byref(khz), C.byref(mem)))
        return {"sm_count": sm.value, "clock_khz": khz.value, "mem_bytes": mem.value}

    def numa_info(self):
        node, cpus = C.c_int(), C.c_int()
        _abi.check(self._lib.afc_numa_info(self.handle, C.byref(node), C.byref(cpus)))
        return {"numa_node": node.value, "local_cpus": cpus.value}

    def launch_count(self):
        return int(self._lib.afc_launch_count(self.handle))

    def selftest(self, iters=2000):
        return _abi.check(self._lib.afc_selftest(self.handle, iters), self.handle)

    def microbench(self, which, iters):
        ops, ms = C.c_double(), C.c_double()
        _abi.check(self._lib.afc_microbench(self.handle, which, iters, C.byref(ops), C.byref(ms)), self.handle)
        return ops.value, ms.value

    def sign_configure(self, constant_time=True):
        """Constant-time fixed-base multiplication for secret scalars (default) or the fast variable-time path."""
        _abi.check(self._lib.afc_sign_configure(self.handle, 1 if constant_time else 0))

    def sign_mode(self):
        return "constant-time" if self._lib.afc_sign_mode(self.handle) == 1 else "fast"

    def keycache_configure(self, max_keys):
        """Capacity of the transparent issuer-key cache behind verify (0 disables it: always the generic kernel)."""
        _abi.check(self._lib.afc_keycache_configure(self.handle, int(max_keys)), self.handle)

    def keycache_clear(self, stream=None):
        """Forget every cached table (stream-ordered; device memory is kept)."""
        _abi.check(self._lib.afc_keycache_clear(self.handle, self._stream(stream)), self.handle)

    def keycache_info(self):
        mk, ck, md = C.c_uint32(), C.c_uint32(), C.c_uint32()
        _abi.check(self._lib.afc_keycache_info(self.handle, C.byref(mk), C.byref(ck), C.byref(md)), self.handle)
        return {"max_keys": mk.value, "cached_keys": ck.value, "last_mode": md.value}

    def keycache_stats(self):
        """How the last verify call was split (hot = through per-key tables, cold = generic kernel) and the running totals."""
        st = _abi.KeycacheStats()
        _abi.check(self._lib.afc_keycache_stats(self.handle, C.byref(st)), self.handle)
        return {k: getattr(st, k) for k, _ in st._fields_}

    def profile_begin(self, max_launches=4096):
        _abi.check(self._lib.afc_profile_begin(self.handle, max_launches), self.handle)

    def profile_end(self):
        """-> {kernel name: {"count", "total_ms", "avg_ms", "min_ms", "max_ms"}} (device-synchronising)."""
        arr = (_abi.ProfileEntry * 64)()
        n = _abi.check(self._lib.afc_profile_end(self.handle, C.cast(arr, C.c_void_p), 64), self.handle)
        return {arr[i].name.decode(): {"count": arr[i].count, "total_ms": arr[i].total_ms, "avg_ms": arr[i].total_ms / max(arr[i].count, 1),
                                       "min_ms": arr[i].min_ms, "max_ms": arr[i].max_ms} for i in range(n)}

    # ---- packed host-buffer calls (numpy arrays, any of them may be pinned)
    def sha256_packed(self, buf, off):
        n = len(off) - 1
        out = np.empty((n, 32), dtype=np.uint8)
        _abi.check(self._lib.afc_sha256_batch(self.handle, _abi.ptr(buf), _abi.ptr(off), n, _abi.ptr(out)), self.handle)
        return out

    def hmac_sha256_packed(self, keys, koff, buf, off):
        n = len(off) - 1
        out = np.empty((n, 32), dtype=np.uint8)
        _abi.check(self._lib.afc_hmac_sha256_batch(self.handle, _abi.ptr(keys), _abi.ptr(koff), _abi.ptr(buf), _abi.ptr(off), n,
                                                   _abi.ptr(out)), self.handle)
        return out

    def webhook_sign_packed(self, cols, col_off, duration_ms, flags, results, result_off, secrets, secret_off):
        """afc_webhook_sign_batch over packed inputs (include/afcrypto.h) -> (bodies, body_off, headers n x 71, status)."""
        n = len(result_off) - 1
        cap = int(self._lib.afc_webhook_bound(_abi.ptr(col_off), _abi.ptr(result_off), n))
        bodies = np.empty(max(cap, 1), dtype=np.uint8)
        body_off = np.zeros(n + 1, dtype=np.uint64)
        headers = np.zeros((n, _abi.WEBHOOK_HEADER_CHARS), dtype=np.uint8)
        status = np.zeros(n, dtype=np.uint8)
        _abi.check(self._lib.afc_webhook_sign_batch(self.handle, _abi.ptr(cols), _abi.ptr(col_off), _abi.ptr(duration_ms), _abi.ptr(flags),
                                                    _abi.ptr(results), _abi.ptr(result_off), _abi.ptr(secrets), _abi.ptr(secret_off), n,
                                                    _abi.ptr(bodies), cap, _abi.ptr(body_off), _abi.ptr(headers), _abi.ptr(status)), self.handle)
        return bodies[:int(body_off[-1])], body_off, headers, status

    def verify_packed(self, pks, sigs, buf, off, out=None):
        n = len(off) - 1
        if out is None:
            out = np.empty(n, dtype=np.uint8)
        _abi.check(self._lib.afc_ed25519_verify_batch(self.handle, _abi.ptr(pks), _abi.ptr(sigs), _abi.ptr(buf), _abi.ptr(off), n,
                                                      _abi.ptr(out)), self.handle)
        return out

    def sign_packed(self, seeds, buf, off):
        n = len(off) - 1
        out = np.empty((n, 64), dtype=np.uint8)
        _abi.check(self._lib.afc_ed25519_sign_batch(self.handle, _abi.ptr(seeds), _abi.ptr(buf), _abi.ptr(off), n, _abi.ptr(out)),
                   self.handle)
        return out

    def pubkeys(self, seeds):
        seeds = np.ascontiguousarray(seeds, dtype=np.uint8).reshape(-1, 32)
        out = np.empty((seeds.shape[0], 32), dtype=np.uint8)
        _abi.check(self._lib.afc_ed25519_pubkey_batch(self.handle, _abi.ptr(seeds), seeds.shape[0], _abi.ptr(out)), self.handle)
        return out

    def expand(self, seeds):
        seeds = np.ascontiguousarray(seeds, dtype=np.uint8).reshape(-1, 32)
        out = np.empty((seeds.shape[0], 96), dtype=np.uint8)
        _abi.check(self._lib.afc_ed25519_expand_batch(self.handle, _abi.ptr(seeds), seeds.shape[0], _abi.ptr(out)), self.handle)
        return out

    def sign_expanded_packed(self, expanded96, key_index, buf, off):
        n = len(off) - 1
        expanded96 = np.ascontiguousarray(expanded96, dtype=np.uint8).reshape(-1, 96)
        ki = None if key_index is None else np.ascontiguousarray(key_index, dtype=np.uint32)
        out = np.empty((n, 64), dtype=np.uint8)
        _abi.check(self._lib.afc_ed25519_sign_expanded_batch(self.handle, _abi.ptr(expanded96), _abi.ptr(ki), expanded96.shape[0],
                                                             _abi.ptr(buf), _abi.ptr(off), n, _abi.ptr(out)), self.handle)
        return out

    # ---- device-pointer calls (torch tensors on this ctx's GPU; `stream` = torch.cuda.Stream or None)
    @staticmethod
    def _stream(stream):
        if stream is None:
            import torch
            return torch.cuda.current_stream().cuda_stream
        return stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)

    def sha256_dev(self, d_msgs, d_off, n, d_out, stream=None):
        _abi.check(self._lib.afc_sha256_batch_dev(self.handle, _abi.ptr(d_msgs), _abi.ptr(d_off), n, _abi.ptr(d_out), self._stream(stream)),
                   self.handle)

    def hmac_sha256_dev(self, d_keys, d_koff, d_msgs, d_off, n, d_out, stream=None):
        _abi.check(self._lib.afc_hmac_sha256_batch_dev(self.handle, _abi.ptr(d_keys), _abi.ptr(d_koff), _abi.ptr(d_msgs), _abi.ptr(d_off), n,
                                                       _abi.ptr(d_out), self._stream(stream)), self.handle)

    def webhook_sign_dev(self, d_cols, d_col_off, d_duration_ms, d_flags, d_results, d_result_off, d_secrets, d_secret_off, n, d_bodies, bodies_cap,
                         d_body_off, d_headers, d_status, stream=None):
        _abi.check(self._lib.afc_webhook_sign_batch_dev(self.handle, _abi.ptr(d_cols), _abi.ptr(d_col_off), _abi.ptr(d_duration_ms), _abi.ptr(d_flags),
                                                        _abi.ptr(d_results), _abi.ptr(d_result_off), _abi.ptr(d_secrets), _abi.ptr(d_secret_off), n,
                                                        _abi.ptr(d_bodies), int(bodies_cap), _abi.ptr(d_body_off), _abi.ptr(d_headers),
                                                        _abi.ptr(d_status), self._stream(stream)), self.handle)

    def verify_dev(self, d_pks, d_sigs, d_msgs, d_off, n, d_ok, stream=None):
        _abi.check(self._lib.afc_ed25519_verify_batch_dev(self.handle, _abi.ptr(d_pks), _abi.ptr(d_sigs), _abi.ptr(d_msgs), _abi.ptr(d_off), n,
                                                          _abi.ptr(d_ok), self._stream(stream)), self.handle)

    def sign_dev(self, d_seeds, d_msgs, d_off, n, d_sigs, stream=None):
        _abi.check(self._lib.afc_ed25519_sign_batch_dev(self.handle, _abi.ptr(d_seeds), _abi.ptr(d_msgs), _abi.ptr(d_off), n, _abi.ptr(d_sigs),
                                                        self._stream(stream)), self.handle)

    def expand_dev(self, d_seeds, n, d_expanded96, stream=None):
        _abi.check(self._lib.afc_ed25519_expand_batch_dev(self.handle, _abi.ptr(d_seeds), n, _abi.ptr(d_expanded96), self._stream(stream)),
                   self.handle)

    def sign_expanded_dev(self, d_expanded96, d_key_index, d_msgs, d_off, n, d_sigs, stream=None):
        _abi.check(self._lib.afc_ed25519_sign_expanded_batch_dev(self.handle, _abi.ptr(d_expanded96), _abi.ptr(d_key_index), _abi.ptr(d_msgs),
                                                                 _abi.ptr(d_off), n, _abi.ptr(d_sigs), self._stream(stream)), self.handle)

    def b64url_encode_dev(self, d_in, item_bytes, n, d_out, stream=None):
        _abi.check(self._lib.afc_b64url_encode_fixed_dev(self.handle, _abi.ptr(d_in), item_bytes, n, _abi.ptr(d_out), self._stream(stream)), self.handle)

    def hex_encode_dev(self, d_in, item_bytes, n, d_out, stream=None):
        _abi.check(self._lib.afc_hex_encode_fixed_dev(self.handle, _abi.ptr(d_in), item_bytes, n, _abi.ptr(d_out), self._stream(stream)), self.handle)

    def merkle_leaf_hashes_dev(self, d_leaves, d_off, n, d_out, stream=None):
        _abi.check(self._lib.afc_merkle_leaf_hashes_dev(self.handle, _abi.ptr(d_leaves), _abi.ptr(d_off), n, _abi.ptr(d_out),
                                                        self._stream(stream)), self.handle)


_default_ctx = {}


def default_context(device=0):
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


class Hasher:
    """SHA256Batch — hashData (vc_service.go:508-515), payload digests (payload_store.go:69-94)."""

    def __init__(self, ctx=None):
        self.ctx = ctx or default_context()

    def sha256_batch(self, msgs):
        buf, off = pack(msgs)
        return [bytes(r) for r in self.ctx.sha256_packed(buf, off)]


class PayloadHasher:
    """Streaming SHA-256 over many concurrent payload uploads: FilePayloadStore.SaveFromReader (internal/services/payload_store.go:45-97)
    hashes each request / response payload while it streams to disk in 32 KiB chunks; here n streams advance together, one GPU
    batch per round of chunks.  States are 108 bytes in Go's crypto/sha256 MarshalBinary layout (include/afcrypto.h)."""

    def __init__(self, n_streams, ctx=None):
        self.ctx = ctx or default_context()
        self._lib = _abi.load()
        self.states = np.zeros((n_streams, _abi.SHA256_STATE_BYTES), dtype=np.uint8)
        _abi.check(self._lib.afc_sha256_stream_init(_abi.ptr(self.states), n_streams))

    def update(self, chunks, final=None):
        """chunks[i] (bytes, b"" for an idle stream) into stream i.  final: None, or a list of booleans — where set, the chunk may be
        ragged and that stream's digest is returned (None elsewhere).  A non-final chunk must be a multiple of 64 bytes: ValueError."""
        n = self.states.shape[0]
        if len(chunks) != n:
            raise ValueError("one chunk per stream")
        fl = np.zeros(n, dtype=np.uint8) if final is None else np.array([1 if f else 0 for f in final], dtype=np.uint8)
        for c, f in zip(chunks, fl):
            if not f and len(c) % 64:
                raise ValueError("only a stream's last chunk may have a length that is not a multiple of 64")
        buf, off = pack([bytes(c) for c in chunks])
        out = np.zeros((n, 32), dtype=np.uint8)
        _abi.check(self._lib.afc_sha256_update_batch(self.ctx.handle, _abi.ptr(self.states), _abi.ptr(buf), _abi.ptr(off), n,
                                                     _abi.ptr(fl) if final is not None else None, _abi.ptr(out)), self.ctx.handle)
        return [bytes(out[i]) if fl[i] else None for i in range(n)]


class MAC:
    """HMACSHA256Batch — generateWebhookSignature (webhook_dispatcher.go:470-474)."""

    def __init__(self, ctx=None):
        self.ctx = ctx or default_context()

    def hmac_sha256_batch(self, keys, msgs):
        if len(keys) != len(msgs):
            raise ValueError("keys and msgs must have the same length")
        kb, ko = pack32(keys)
        buf, off = pack(msgs)
        return [bytes(r) for r in self.ctx.hmac_sha256_packed(kb, ko, buf, off)]


class Signer:
    """SignBatch — ed25519.NewKeyFromSeed + ed25519.Sign (vc_service.go:460-463)."""

    def __init__(self, ctx=None):
        self.ctx = ctx or default_context()

    def sign_batch(self, seeds, msgs):
        if len(seeds) != len(msgs):
            raise ValueError("seeds and msgs must have the same length")
        for s in seeds:
            if len(s) != 32:
                raise ValueError("ed25519: bad seed length: %d" % len(s))      # Go panics
        sd = np.frombuffer(b"".join(seeds), dtype=np.uint8).reshape(-1, 32).copy() if seeds else np.zeros((0, 32), np.uint8)
        buf, off = pack(msgs)
        return [bytes(r) for r in self.ctx.sign_packed(sd, buf, off)]

    def public_keys(self, seeds):
        for s in seeds:
            if len(s) != 32:
                raise ValueError("ed25519: bad seed length: %d" % len(s))
        sd = np.frombuffer(b"".join(seeds), dtype=np.uint8).reshape(-1, 32).copy() if seeds else np.zeros((0, 32), np.uint8)
        return [bytes(r) for r in self.ctx.pubkeys(sd)]


class Verifier:
    """VerifyBatch — ed25519.Verify (vc_service.go:504,1624; cli/vc_verification_enhanced.go:453)."""

    def __init__(self, ctx=None):
        self.ctx = ctx or default_context()

    def verify_batch(self, pks, msgs, sigs):
        if not (len(pks) == len(msgs) == len(sigs)):
            raise ValueError("pks, msgs and sigs must have the same length")
        for p in pks:
            if len(p) != 32:
                raise ValueError("ed25519: bad public key length: %d" % len(p))   # Go panics
        n = len(pks)
        if n == 0:
            return []
        bad_len = [len(s) != 64 for s in sigs]                                      # Go: plain false
        sg = np.zeros((n, 64), dtype=np.uint8)
        for i, s in enumerate(sigs):
            if not bad_len[i]:
                sg[i] = np.frombuffer(s, dtype=np.uint8)
        pk = np.frombuffer(b"".join(pks), dtype=np.uint8).reshape(-1, 32).copy()
        buf, off = pack(msgs)
        ok = self.ctx.verify_packed(pk, sg, buf, off)
        return [bool(o) and not b for o, b in zip(ok, bad_len)]
