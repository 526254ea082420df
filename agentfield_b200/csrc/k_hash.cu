// SHA-256 / HMAC-SHA256 / RFC 6962 Merkle kernels for sm_90a.
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_sha256_batch       sha256.Sum256 in VCService.hashData        internal/services/vc_service.go:508-515
//                        payload digest                              internal/services/payload_store.go:69-94
//                        seed derivation hash                        internal/services/did_service.go:515-521
//   k_hmac_sha256_batch  generateWebhookSignature                    internal/services/webhook_dispatcher.go:470-474
//   k_merkle_*           NEW (RFC 6962 §2.1); reference stub         internal/cli/vc_verification_enhanced.go:531-534
//
// Shape: one message per thread; every lane runs the identical fully-unrolled compression (SHF funnel
// rotates, LOP3 Ch/Maj, round constants as constant-bank immediates).  These kernels are integer-ALU
// bound (~1.5k ALU ops per 64-byte block => ~20 ops/byte), an order of magnitude above the HBM
// roofline's ops/byte; see DESIGN.md §kernels.
#include "afc_launch.h"
#include "afc_sha.cuh"
#include "afc_json.cuh"

namespace afc {

static constexpr int HASH_THREADS = 128;

__global__ void __launch_bounds__(HASH_THREADS)
k_sha256_batch(const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ off, uint32_t n, uint8_t* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t o0 = off[i], o1 = off[i + 1];
    uint32_t st[8];
    sha256_msg(st, msgs + o0, o1 - o0);
    store_digest256(out + 32ull * i, st);
}

// H2 streaming (FilePayloadStore.SaveFromReader, internal/services/payload_store.go:45-97): stream i absorbs chunk i into its
// 108-byte state; where final[i] is set the chunk may be ragged, the stream is padded and out32[i] receives the digest (the state
// is left as it was after the last whole block: a finished stream is not resumed).  status[i] = 0 for a malformed state.
__global__ void __launch_bounds__(HASH_THREADS)
k_sha256_update(uint8_t* __restrict__ states, const uint8_t* __restrict__ chunks, const uint64_t* __restrict__ off, uint32_t n,
                const uint8_t* __restrict__ final_flags, uint8_t* __restrict__ out32, uint8_t* __restrict__ status) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t* s = states + (size_t)SHA256_STATE_BYTES * i;
    uint32_t st[8];
    uint64_t prior;
    const int ok = sha256_state_load(st, &prior, s);
    const uint64_t o0 = off[i], len = off[i + 1] - o0;
    const bool fin = final_flags && final_flags[i];
    if (!ok || (!fin && (len & 63))) { if (status) status[i] = 0; return; }
    if (status) status[i] = 1;
    if (!fin) {
        sha256_absorb_blocks(st, chunks + o0, len);
        sha256_state_store(s, st, prior + len);
    } else {
        sha256_finish_stream(st, chunks + o0, len, prior);
        for (int w = 0; w < 8; w++) store_be32(out32 + 32ull * i + 4 * w, st[w]);
    }
}

__global__ void __launch_bounds__(HASH_THREADS)
k_hmac_sha256_batch(const uint8_t* __restrict__ keys, const uint32_t* __restrict__ koff, const uint8_t* __restrict__ msgs,
                    const uint64_t* __restrict__ off, uint32_t n, uint8_t* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t k0 = koff[i], k1 = koff[i + 1];
    uint64_t o0 = off[i], o1 = off[i + 1];
    uint32_t st[8];
    hmac_sha256_msg(st, keys + k0, k1 - k0, msgs + o0, o1 - o0);
    store_digest256(out + 32ull * i, st);
}

__global__ void __launch_bounds__(HASH_THREADS)
k_merkle_leaf(const uint8_t* __restrict__ leaves, const uint64_t* __restrict__ off, uint32_t n, uint8_t* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t o0 = off[i], o1 = off[i + 1];
    uint32_t st[8];
    sha256_merkle_leaf(st, leaves + o0, o1 - o0);
    store_digest256(out + 32ull * i, st);
}

__device__ __forceinline__ void load_node(uint32_t w[8], const uint8_t* p) {
    const uint4* q = (const uint4*)p;       // node arrays are 32-byte records in 16B-aligned buffers
    uint4 a = q[0], b = q[1];
    w[0] = bswap32(a.x); w[1] = bswap32(a.y); w[2] = bswap32(a.z); w[3] = bswap32(a.w);
    w[4] = bswap32(b.x); w[5] = bswap32(b.y); w[6] = bswap32(b.z); w[7] = bswap32(b.w);
}

// One level of the RFC 6962 tree over an index range (see afc_launch.h for the meaning of the flags).
__global__ void __launch_bounds__(HASH_THREADS)
k_merkle_level(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint64_t npairs, int left_merge, int right_orphan,
               uint8_t* frontier, int h) {
    uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t first = left_merge ? 1 : 0;
    if (p < npairs) {
        uint32_t l[8], r[8], o[8];
        load_node(l, in + 32 * (first + 2 * p));
        load_node(r, in + 32 * (first + 2 * p + 1));
        sha256_merkle_node(o, l, r);
        store_digest256(out + 32 * (first + p), o);
    } else if (p == npairs) {
        if (left_merge) {
            uint32_t l[8], r[8], o[8];
            load_node(l, frontier + 32 * h);
            load_node(r, in);
            sha256_merkle_node(o, l, r);
            store_digest256(out, o);
        }
        if (right_orphan) {
            const uint4* src = (const uint4*)(in + 32 * (first + 2 * npairs));
            uint4 a = src[0], b = src[1];
            uint4* dst = (uint4*)(frontier + 32 * h);
            dst[0] = a; dst[1] = b;
        }
    }
}

__global__ void k_merkle_root(const uint8_t* __restrict__ frontier, uint64_t size, uint8_t* __restrict__ out) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    uint32_t acc[8];
    if (size == 0) {
        sha256_msg(acc, (const uint8_t*)0, 0);
    } else {
        int h = 0;
        while (!((size >> h) & 1)) h++;
        load_node(acc, frontier + 32 * h);
        for (h = h + 1; h < 64; h++) {
            if ((size >> h) & 1) {
                uint32_t l[8], o[8];
                load_node(l, frontier + 32 * h);
                sha256_merkle_node(o, l, acc);
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] = o[i];
            }
        }
    }
    store_digest256(out, acc);
}



// ---- materialised tree for audit proofs (SURVEY.md §8f N4): every level kept, unpaired last node promoted unchanged
__global__ void __launch_bounds__(HASH_THREADS)
k_merkle_level_promote(const uint8_t* __restrict__ in, uint64_t n_in, uint8_t* __restrict__ out) {
    uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t npairs = n_in >> 1;
    if (p < npairs) {
        uint32_t l[8], r[8], o[8];
        load_node(l, in + 64 * p);
        load_node(r, in + 64 * p + 32);
        sha256_merkle_node(o, l, r);
        store_digest256(out + 32 * p, o);
    } else if (p == npairs && (n_in & 1)) {
        const uint4* src = (const uint4*)(in + 32 * (n_in - 1));
        uint4 a = src[0], b = src[1];
        uint4* dst = (uint4*)(out + 32 * npairs);
        dst[0] = a; dst[1] = b;
    }
}

// RFC 6962 §2.1.1 audit paths for many leaves at once: one thread per requested index walks the stored levels.
// levels[h] = device pointer to level h (32-byte nodes), sizes[h] = node count; out: m x depth x 32, lens: m.
__global__ void __launch_bounds__(HASH_THREADS)
k_merkle_gather_proofs(const uint8_t* const* __restrict__ levels, const uint64_t* __restrict__ sizes, int n_levels,
                       const uint64_t* __restrict__ indices, uint32_t m, uint8_t* __restrict__ out, uint32_t* __restrict__ lens) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    uint64_t idx = indices[t];
    uint8_t* o = out + (size_t)t * (n_levels > 1 ? n_levels - 1 : 1) * 32;
    uint32_t k = 0;
    if (idx < sizes[0]) {
        for (int h = 0; h + 1 < n_levels; h++) {
            uint64_t sib = idx ^ 1;
            if (sib < sizes[h]) {
                const uint4* src = (const uint4*)(levels[h] + 32 * sib);
                uint4 a = src[0], b = src[1];
                uint4* dst = (uint4*)(o + 32 * k);
                dst[0] = a; dst[1] = b;
                k++;
            }
            idx >>= 1;
        }
    }
    lens[t] = k;
}

// RFC 9162 §2.1.3.2 inclusion verification, one proof per thread.  leaf_hashes: m x 32; proofs packed, proof_off[m+1] in
// units of 32-byte nodes; ok[i] = 1 iff the path leads to `root` for (indices[i], tree_size).
__global__ void __launch_bounds__(HASH_THREADS)
k_merkle_verify_inclusion(const uint8_t* __restrict__ leaf_hashes, const uint64_t* __restrict__ indices, uint64_t tree_size,
                          const uint8_t* __restrict__ proofs, const uint32_t* __restrict__ proof_off, const uint8_t* __restrict__ root,
                          uint32_t m, uint8_t* __restrict__ ok) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    uint64_t fn = indices[t], sn = tree_size - 1;
    uint32_t good = (tree_size != 0) && (fn < tree_size);
    uint32_t r[8], want[8];
    load_node(r, leaf_hashes + 32ull * t);
    load_node(want, root);
    if (good) {
        for (uint32_t k = proof_off[t]; k < proof_off[t + 1]; k++) {
            if (sn == 0) { good = 0; break; }
            uint32_t p[8], o[8];
            load_node(p, proofs + 32ull * k);
            if ((fn & 1) || fn == sn) {
                sha256_merkle_node(o, p, r);
                if (!(fn & 1)) { while (fn && !(fn & 1)) { fn >>= 1; sn >>= 1; } }
            } else {
                sha256_merkle_node(o, r, p);
            }
#pragma unroll
            for (int i = 0; i < 8; i++) r[i] = o[i];
            fn >>= 1; sn >>= 1;
        }
    }
    uint32_t diff = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) diff |= r[i] ^ want[i];
    ok[t] = (uint8_t)(good && sn == 0 && diff == 0);
}

// RFC 9162 §2.1.4.2 consistency verification, one proof per thread: the tree of second_size leaves with root second_root
// extends the tree of first_sizes[t] leaves with root first_roots[t].  Proofs packed as for inclusion.
__global__ void __launch_bounds__(HASH_THREADS)
k_merkle_verify_consistency(const uint64_t* __restrict__ first_sizes, const uint8_t* __restrict__ first_roots, uint64_t second_size,
                            const uint8_t* __restrict__ second_root, const uint8_t* __restrict__ proofs,
                            const uint32_t* __restrict__ proof_off, uint32_t m, uint8_t* __restrict__ ok) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    const uint64_t first = first_sizes[t];
    uint32_t k = proof_off[t];
    const uint32_t k1 = proof_off[t + 1];
    uint32_t good = first > 0 && first <= second_size;
    uint32_t fw[8], sw[8], fr[8], sr[8];
    load_node(fw, first_roots + 32ull * t);
    load_node(sw, second_root);
    uint32_t same = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) same |= fw[i] ^ sw[i];
    if (!good || first == second_size) { ok[t] = (uint8_t)(good && k == k1 && same == 0); return; }
    if ((first & (first - 1)) == 0) {
#pragma unroll
        for (int i = 0; i < 8; i++) fr[i] = fw[i];               // a power of two: the old root itself starts the path
    } else if (k < k1) {
        load_node(fr, proofs + 32ull * k); k++;
    } else { ok[t] = 0; return; }
#pragma unroll
    for (int i = 0; i < 8; i++) sr[i] = fr[i];
    uint64_t fn = first - 1, sn = second_size - 1;
    while (fn & 1) { fn >>= 1; sn >>= 1; }
    for (; k < k1; k++) {
        if (sn == 0) { good = 0; break; }
        uint32_t c[8], o[8];
        load_node(c, proofs + 32ull * k);
        if ((fn & 1) || fn == sn) {
            sha256_merkle_node(o, c, fr);
#pragma unroll
            for (int i = 0; i < 8; i++) fr[i] = o[i];
            sha256_merkle_node(o, c, sr);
            while (fn && !(fn & 1)) { fn >>= 1; sn >>= 1; }
        } else {
            sha256_merkle_node(o, sr, c);
        }
#pragma unroll
        for (int i = 0; i < 8; i++) sr[i] = o[i];
        fn >>= 1; sn >>= 1;
    }
    uint32_t diff = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) diff |= (fr[i] ^ fw[i]) | (sr[i] ^ sw[i]);
    ok[t] = (uint8_t)(good && sn == 0 && diff == 0);
}

// ---- canonical form (SURVEY.md §8f N3): n documents assembled from one template and n x F values (afc_json.cuh) ----------
// Pass 1 writes every document's length to len_out[i] (= d_out_off + 1), an inclusive scan turns them into offsets, pass 2
// writes the bytes.  One document per thread; aligned 32-bit reads, 32-byte writes, four plain bytes at a time.
// Tried and dropped: 4-byte writes, 16-byte writes and one WARP per document with one byte per lane (a 32-byte value costs a
// whole ballot + scan round, 47 pieces per document).
__global__ void __launch_bounds__(HASH_THREADS)
k_json_sizes(const uint8_t* __restrict__ segs, const uint32_t* __restrict__ seg_off, const uint8_t* __restrict__ kinds, uint32_t F,
             const uint8_t* __restrict__ fields, const uint64_t* __restrict__ field_off, uint32_t n, uint64_t* __restrict__ len_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ByteCounter c; c.init();
    json_fill_one(c, segs, seg_off, kinds, F, fields, field_off + (uint64_t)i * F);
    len_out[i] = c.n;
}
__global__ void __launch_bounds__(HASH_THREADS)
k_json_fill(const uint8_t* __restrict__ segs, const uint32_t* __restrict__ seg_off, const uint8_t* __restrict__ kinds, uint32_t F,
            const uint8_t* __restrict__ fields, const uint64_t* __restrict__ field_off, uint32_t n, const uint64_t* __restrict__ out_off,
            uint8_t* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ByteWriter w; w.init(out + out_off[i]);
    json_fill_one(w, segs, seg_off, kinds, F, fields, field_off + (uint64_t)i * F);
    w.finish();
}
__global__ void k_set_u64(uint64_t* p, uint64_t v) { *p = v; }
// In-place inclusive scan of n 64-bit values: per-block scan (1024 values per 256-thread block) + block totals, an exclusive
// scan of the totals by one block, and a final add.
constexpr int SCAN_THREADS = 256, SCAN_PER_THREAD = 4, SCAN_TILE = SCAN_THREADS * SCAN_PER_THREAD;
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_tiles(uint64_t* __restrict__ v, uint64_t n, uint64_t* __restrict__ tile_sums) {
    __shared__ uint64_t warp_tot[SCAN_THREADS / 32];
    const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_PER_THREAD;
    uint64_t x[SCAN_PER_THREAD], run = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) { x[k] = (base + k < n) ? v[base + k] : 0; run += x[k]; x[k] = run; }
    uint64_t incl = run;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (unsigned)d) incl += y; }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    uint64_t before = 0;
    for (unsigned w = 0; w < warp; w++) before += warp_tot[w];
    const uint64_t excl = before + incl - run;
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) if (base + k < n) v[base + k] = x[k] + excl;
    if (threadIdx.x == SCAN_THREADS - 1) tile_sums[blockIdx.x] = before + incl;
}
__global__ void __launch_bounds__(1024)
k_scan_tile_sums(uint64_t* __restrict__ tile_sums, uint64_t n_tiles) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint64_t b = 0; b < n_tiles; b += 1024) {
        const uint64_t i = b + threadIdx.x;
        const uint64_t x = i < n_tiles ? tile_sums[i] : 0;
        uint64_t incl = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (unsigned)d) incl += y; }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        uint64_t before = carry;
        for (unsigned w = 0; w < warp; w++) before += warp_tot[w];
        if (i < n_tiles) tile_sums[i] = before + incl - x;             // exclusive
        __syncthreads();
        if (threadIdx.x == 1023) carry = before + incl;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_add(uint64_t* __restrict__ v, uint64_t n, const uint64_t* __restrict__ tile_sums) {
    const uint64_t add = tile_sums[blockIdx.x];
    const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_PER_THREAD;
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) if (base + k < n) v[base + k] += add;
}
// The ends a _dev call needs before it can size anything (offset_ends): one thread, since an indirect span's indices are device words
__global__ void k_offset_ends(const launch::OffsetSpans S, uint32_t n, uint64_t* __restrict__ out) { offset_ends(S.s, S.k, n, out); }

// ---- text codecs either side of the kernels (SURVEY.md §8f N3): base64url without padding for signatures / digests
// (base64.RawURLEncoding in vc_service.go:465,514) and lowercase hex for the webhook header (hex.EncodeToString,
// webhook_dispatcher.go:473).  Fixed-size records; one thread per 3-byte group / per byte pair.
__global__ void __launch_bounds__(256)
k_b64url_encode(const uint8_t* __restrict__ in, uint32_t item, uint32_t n, uint8_t* __restrict__ out) {
    const uint32_t groups = (item + 2) / 3, out_item = (item * 4 + 2) / 3;
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n * groups) return;
    uint32_t rec = (uint32_t)(t / groups), g = (uint32_t)(t % groups);
    const uint8_t* p = in + (uint64_t)rec * item + 3 * g;
    uint32_t rem = item - 3 * g;
    uint32_t v = (uint32_t)p[0] << 16;
    if (rem > 1) v |= (uint32_t)p[1] << 8;
    if (rem > 2) v |= p[2];
    uint8_t* o = out + (uint64_t)rec * out_item + 4 * g;
    uint32_t nch = rem >= 3 ? 4 : rem + 1;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        if (k < nch) {
            uint32_t x = (v >> (18 - 6 * k)) & 63u;
            o[k] = (uint8_t)(x < 26 ? 'A' + x : x < 52 ? 'a' + (x - 26) : x < 62 ? '0' + (x - 52) : (x == 62 ? '-' : '_'));
        }
    }
}
__global__ void __launch_bounds__(256)
k_hex_encode(const uint8_t* __restrict__ in, uint64_t total, uint8_t* __restrict__ out) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    uint32_t b = in[t], hi = b >> 4, lo = b & 15;
    out[2 * t] = (uint8_t)(hi < 10 ? '0' + hi : 'a' + (hi - 10));
    out[2 * t + 1] = (uint8_t)(lo < 10 ? '0' + lo : 'a' + (lo - 10));
}

// register-only throughput probes: which = 3 SHA-256 compress, 4 SHA-512 compress
__global__ void k_microbench_hash(int which, uint32_t iters, uint32_t* sink) {
    uint32_t seed = blockIdx.x * blockDim.x + threadIdx.x;
    if (which == 3) {
        uint32_t st[8], w[16];
#pragma unroll
        for (int i = 0; i < 8; i++) st[i] = seed + i;
        for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = st[i & 7] ^ (it + i);
            sha256_compress(st, w);
        }
        if (st[0] == 0x12345678u) sink[0] = st[1];
    } else {
        sha512_st x;
        sha512_blk b;
#pragma unroll
        for (int i = 0; i < 8; i++) x.st[i] = seed + i;
        for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
            for (int i = 0; i < 16; i++) b.w[i] = x.st[i & 7] ^ (it + i);
            x = sha512_compress_regs(x, b);
        }
        if (x.st[0] == 0x12345678u) sink[0] = (uint32_t)x.st[1];
    }
}

namespace launch {

static inline uint32_t blocks_for(uint64_t n, int t) { return (uint32_t)((n + t - 1) / t); }

cudaError_t sha256_batch(const uint8_t* msgs, const uint64_t* off, uint32_t n, uint8_t* out32, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_sha256_batch", s, k_sha256_batch<<<blocks_for(n, HASH_THREADS), HASH_THREADS, 0, s>>>(msgs, off, n, out32));
    return cudaGetLastError();
}
cudaError_t sha256_update(uint8_t* states, const uint8_t* chunks, const uint64_t* off, uint32_t n, const uint8_t* final_flags, uint8_t* out32,
                          uint8_t* status, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_sha256_update", s, k_sha256_update<<<blocks_for(n, HASH_THREADS), HASH_THREADS, 0, s>>>(states, chunks, off, n, final_flags, out32, status));
    return cudaGetLastError();
}
cudaError_t hmac_sha256_batch(const uint8_t* keys, const uint32_t* koff, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                              uint8_t* out32, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_hmac_sha256_batch", s, k_hmac_sha256_batch<<<blocks_for(n, HASH_THREADS), HASH_THREADS, 0, s>>>(keys, koff, msgs, off, n, out32));
    return cudaGetLastError();
}
cudaError_t merkle_leaf_hashes(const uint8_t* leaves, const uint64_t* off, uint32_t n, uint8_t* out32, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_merkle_leaf", s, k_merkle_leaf<<<blocks_for(n, HASH_THREADS), HASH_THREADS, 0, s>>>(leaves, off, n, out32));
    return cudaGetLastError();
}
cudaError_t merkle_level(const uint8_t* in, uint8_t* out, uint64_t npairs, int left_merge, int right_orphan,
                         uint8_t* frontier, int h, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_merkle_level", s, k_merkle_level<<<blocks_for(npairs + 1, HASH_THREADS), HASH_THREADS, 0, s>>>(in, out, npairs, left_merge, right_orphan, frontier, h));
    return cudaGetLastError();
}
cudaError_t merkle_root(const uint8_t* frontier, uint64_t size, uint8_t* out32, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_merkle_root", s, k_merkle_root<<<1, 32, 0, s>>>(frontier, size, out32));
    return cudaGetLastError();
}
cudaError_t merkle_level_promote(const uint8_t* in, uint64_t n_in, uint8_t* out, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_merkle_level_promote", s, k_merkle_level_promote<<<blocks_for((n_in >> 1) + 1, HASH_THREADS), HASH_THREADS, 0, s>>>(in, n_in, out));
    return cudaGetLastError();
}
cudaError_t merkle_gather_proofs(const uint8_t* const* levels, const uint64_t* sizes, int n_levels, const uint64_t* indices, uint32_t m,
                                 uint8_t* out, uint32_t* lens, cudaStream_t s, LaunchLog* lg) {
    if (m == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_merkle_gather_proofs", s, k_merkle_gather_proofs<<<blocks_for(m, HASH_THREADS), HASH_THREADS, 0, s>>>(levels, sizes, n_levels, indices, m, out, lens));
    return cudaGetLastError();
}
cudaError_t merkle_verify_inclusion(const uint8_t* leaf_hashes, const uint64_t* indices, uint64_t tree_size, const uint8_t* proofs,
                                    const uint32_t* proof_off, const uint8_t* root, uint32_t m, uint8_t* ok, cudaStream_t s, LaunchLog* lg) {
    if (m == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_merkle_verify_inclusion", s, k_merkle_verify_inclusion<<<blocks_for(m, HASH_THREADS), HASH_THREADS, 0, s>>>(leaf_hashes, indices, tree_size, proofs, proof_off, root, m, ok));
    return cudaGetLastError();
}
cudaError_t merkle_verify_consistency(const uint64_t* first_sizes, const uint8_t* first_roots, uint64_t second_size, const uint8_t* second_root,
                                      const uint8_t* proofs, const uint32_t* proof_off, uint32_t m, uint8_t* ok, cudaStream_t s, LaunchLog* lg) {
    if (m == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_merkle_verify_consistency", s, k_merkle_verify_consistency<<<blocks_for(m, HASH_THREADS), HASH_THREADS, 0, s>>>(first_sizes, first_roots, second_size, second_root, proofs, proof_off, m, ok));
    return cudaGetLastError();
}
size_t json_scan_scratch_bytes(uint32_t n) { return (((size_t)n + SCAN_TILE - 1) / SCAN_TILE + 1) * 8; }
cudaError_t json_fill_sizes(const uint8_t* segs, const uint32_t* seg_off, const uint8_t* kinds, uint32_t F, const uint8_t* fields,
                            const uint64_t* field_off, uint32_t n, uint64_t* out_off, uint64_t* scan_scratch, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) { k_set_u64<<<1, 1, 0, s>>>(out_off, 0); return cudaGetLastError(); }
    AFC_LAUNCH(lg, "k_json_sizes", s, k_json_sizes<<<blocks_for(n, HASH_THREADS), HASH_THREADS, 0, s>>>(segs, seg_off, kinds, F, fields, field_off, n, out_off + 1));
    return offsets_from_lengths(out_off, n, scan_scratch, s, lg);
}
cudaError_t offsets_from_lengths(uint64_t* out_off, uint32_t n, uint64_t* scan_scratch, cudaStream_t s, LaunchLog* lg) {
    k_set_u64<<<1, 1, 0, s>>>(out_off, 0);          // (a kernel, not cudaMemsetAsync: see k_fill_u32 in k_ed25519.cu)
    if (n == 0) return cudaGetLastError();
    const uint32_t tiles = blocks_for(n, SCAN_TILE);
    AFC_LAUNCH(lg, "k_scan_tiles", s, k_scan_tiles<<<tiles, SCAN_THREADS, 0, s>>>(out_off + 1, n, scan_scratch));
    AFC_LAUNCH(lg, "k_scan_tile_sums", s, k_scan_tile_sums<<<1, 1024, 0, s>>>(scan_scratch, tiles));
    AFC_LAUNCH(lg, "k_scan_add", s, k_scan_add<<<tiles, SCAN_THREADS, 0, s>>>(out_off + 1, n, scan_scratch));
    return cudaGetLastError();
}
cudaError_t offset_ends(const OffsetSpans& S, uint32_t n, uint64_t* out, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_offset_ends", s, k_offset_ends<<<1, 1, 0, s>>>(S, n, out));
    return cudaGetLastError();
}
cudaError_t json_fill(const uint8_t* segs, const uint32_t* seg_off, const uint8_t* kinds, uint32_t F, const uint8_t* fields,
                      const uint64_t* field_off, uint32_t n, const uint64_t* out_off, uint8_t* out, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_json_fill", s, k_json_fill<<<blocks_for(n, HASH_THREADS), HASH_THREADS, 0, s>>>(segs, seg_off, kinds, F, fields, field_off, n, out_off, out));
    return cudaGetLastError();
}
cudaError_t b64url_encode(const uint8_t* in, uint32_t item, uint32_t n, uint8_t* out, cudaStream_t s, LaunchLog* lg) {
    if (n == 0 || item == 0) return cudaSuccess;
    uint64_t threads = (uint64_t)n * ((item + 2) / 3);
    AFC_LAUNCH(lg, "k_b64url_encode", s, k_b64url_encode<<<blocks_for(threads, 256), 256, 0, s>>>(in, item, n, out));
    return cudaGetLastError();
}
cudaError_t hex_encode(const uint8_t* in, uint64_t total, uint8_t* out, cudaStream_t s, LaunchLog* lg) {
    if (total == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_hex_encode", s, k_hex_encode<<<blocks_for(total, 256), 256, 0, s>>>(in, total, out));
    return cudaGetLastError();
}
cudaError_t microbench_hash(int which, uint32_t iters, uint32_t blocks, uint32_t threads, uint32_t* sink, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_microbench_hash", s, k_microbench_hash<<<blocks, threads, 0, s>>>(which, iters, sink));
    return cudaGetLastError();
}

}  // namespace launch
}  // namespace afc
