// tests/devsim — TEST-ONLY sm_90a build of ge_ops.cuh (no torch, no libafcrypto.so).
//
// ge_run:  one thread per item, the routine as the product kernels inline it; copies in, launches, synchronises, copies out
//          and returns the CUDA error (cudaErrorInvalidValue for an unknown operation or an item outside its domain).
// ge_bulk: n items generated on the device from (seed, index) by gen_word (devsim.cu's generator) and shaped into the
//          operation's domain by ge_shape, each run through the product form and the portable twin (every field
//          multiplication through fe_mul_c / fe_sq_c).  It counts the items where the two differ and keeps the product form's
//          output of every stride-th item, which the tests regenerate and compare with Python integers.  Items go through in
//          chunks, so that the outputs and scratch of one chunk stay within a fixed amount of device memory.
#include "ge_ops.cuh"

namespace gesim {

__host__ __device__ inline uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t gen_word(uint64_t seed, uint64_t i, int w) {
    const uint64_t z = mix64(seed + i * 1024u + (uint64_t)w);
    const uint32_t sel = (uint32_t)(z >> 60);
    return sel == 0 ? 0u : sel <= 2 ? 0xffffffffu : (uint32_t)z;
}

// Random words into the operation's domain (tests/ge_cases.py shape() is the same map).
template <int OP>
__device__ void ge_shape(uint32_t* x) {
    if constexpr (OP == GE_GROUP_KC) x[0] = 1 + x[0] % KC_GMAX;
    if constexpr (OP == GE_GROUP_SIGN) x[0] = 1 + x[0] % SIGN_GMAX;
    if constexpr (OP == GE_GROUP_SIGN2) x[0] = 1 + x[0] % (2 * SIGN_GMAX);
    if constexpr (OP == GE_ADDSUB || OP == GE_ADDSUB_CALL) x[64] &= 1u;
    if constexpr (OP == GE_MADD) { x[56] &= 1u; x[57] &= 1u; }
    if constexpr (OP == GE_CT_SELECT) x[192] = (uint32_t)((int)(x[192] % 17u) - 8);
    if constexpr (OP == GE_SMALL_MULT || OP == GE_SMALL_MULT_CALL) x[32] = 1u + x[32] % ((1u << 22) - 1u);
    if constexpr (OP == GE_KEY_ROWS) {
        x[8] %= COMB_ROWS;
        x[9] = 1u << (x[9] % 3u);
    }
    if constexpr (OP == GE_RECODE) {
        const uint32_t k = x[8] % 10u;                 // 0, 1, 2: the fixed radixes (s < 2^254); 16..22: the wide form (s < 2^253)
        x[8] = k < 3 ? k : k + 13u;
        x[7] &= k < 3 ? 0x3fffffffu : 0x1fffffffu;
    }
}

template <int OP>
__global__ void k_ge_run(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint32_t* scratch, int n,
                         unsigned* __restrict__ refused) {
    constexpr int IN = ge_in_words(OP), OUT = ge_out_words(OP), SCR = ge_scratch_words(OP);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (run_op<OP, false>(in + (size_t)i * IN, out + (size_t)i * OUT, scratch + (size_t)i * SCR)) atomicAdd(refused, 1u);
}

template <int OP>
__global__ void k_ge_gen(uint64_t seed, uint64_t base, uint32_t cnt, uint32_t* __restrict__ in) {
    constexpr int IN = ge_in_words(OP);
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= cnt) return;
    uint32_t* x = in + (size_t)k * IN;
    for (int w = 0; w < IN; w++) x[w] = gen_word(seed, base + k, w);
    ge_shape<OP>(x);
}

// one thread per item of the chunk; y and z are the thread's slices of `outs` (product form, portable twin)
template <int OP>
__global__ void k_ge_bulk(uint64_t base, uint32_t cnt, uint64_t stride, const uint32_t* __restrict__ in, uint32_t* outs,
                          uint32_t* scratch, uint32_t* __restrict__ samples, unsigned long long* __restrict__ stats) {
    constexpr int IN = ge_in_words(OP), OUT = ge_out_words(OP), SCR = ge_scratch_words(OP);
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= cnt) return;
    const uint64_t i = base + k;
    uint32_t* y = outs + (size_t)k * 2 * OUT;
    uint32_t* z = y + OUT;
    uint32_t* s = scratch + (size_t)k * SCR;
    int r = run_op<OP, false>(in + (size_t)k * IN, y, s);
    r |= run_op<OP, true>(in + (size_t)k * IN, z, s);
    uint32_t d = (uint32_t)r;
    for (int w = 0; w < OUT; w++) d |= y[w] ^ z[w];
    if (d) {
        atomicAdd(&stats[0], 1ull);
        atomicMin(&stats[1], (unsigned long long)i);
    }
    if (i % stride == 0)
        for (int w = 0; w < OUT; w++) samples[(i / stride) * OUT + w] = y[w];
}

constexpr size_t BULK_BYTES = (size_t)256 << 20;       // outputs + scratch of one chunk

#define GE_TRY(x) do { e = (x); if (e != cudaSuccess) goto done; } while (0)

template <int OP>
static cudaError_t run(const uint32_t* in, uint32_t* out, uint64_t n) {
    constexpr int IN = ge_in_words(OP), OUT = ge_out_words(OP), SCR = ge_scratch_words(OP);
    uint32_t *din = nullptr, *dout = nullptr, *dscr = nullptr;
    unsigned* dref = nullptr;
    unsigned refused = 0;
    cudaError_t e = cudaSuccess;
    if (n > (1u << 30)) return cudaErrorInvalidValue;
    GE_TRY(cudaMalloc(&din, n * IN * sizeof(uint32_t)));
    GE_TRY(cudaMalloc(&dout, n * OUT * sizeof(uint32_t)));
    if (SCR) GE_TRY(cudaMalloc(&dscr, n * SCR * sizeof(uint32_t)));
    GE_TRY(cudaMalloc(&dref, sizeof(unsigned)));
    GE_TRY(cudaMemset(dref, 0, sizeof(unsigned)));
    GE_TRY(cudaMemcpy(din, in, n * IN * sizeof(uint32_t), cudaMemcpyHostToDevice));
    k_ge_run<OP><<<(unsigned)((n + 127) / 128), 128>>>(din, dout, dscr, (int)n, dref);
    GE_TRY(cudaGetLastError());
    GE_TRY(cudaDeviceSynchronize());
    GE_TRY(cudaMemcpy(out, dout, n * OUT * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    GE_TRY(cudaMemcpy(&refused, dref, sizeof(unsigned), cudaMemcpyDeviceToHost));
    if (refused) e = cudaErrorInvalidValue;
done:
    cudaFree(din);
    cudaFree(dout);
    cudaFree(dscr);
    cudaFree(dref);
    return e;
}

template <int OP>
static cudaError_t bulk(uint64_t seed, uint64_t n, uint64_t stride, uint32_t* samples, unsigned long long* stats) {
    constexpr int IN = ge_in_words(OP), OUT = ge_out_words(OP), SCR = ge_scratch_words(OP);
    const uint64_t per_item = (uint64_t)(IN + 2 * OUT + SCR) * sizeof(uint32_t);
    uint64_t chunk = BULK_BYTES / per_item;
    if (chunk > (1u << 20)) chunk = 1u << 20;
    if (chunk > n) chunk = n;
    const uint64_t ns = (n + stride - 1) / stride;
    uint32_t *din = nullptr, *douts = nullptr, *dscr = nullptr, *dsam = nullptr;
    unsigned long long* dstats = nullptr;
    const unsigned long long init[2] = {0ull, ~0ull};
    cudaError_t e = cudaSuccess;
    GE_TRY(cudaMalloc(&din, (chunk ? chunk : 1) * IN * sizeof(uint32_t)));
    GE_TRY(cudaMalloc(&douts, (chunk ? chunk : 1) * 2 * OUT * sizeof(uint32_t)));
    if (SCR) GE_TRY(cudaMalloc(&dscr, (chunk ? chunk : 1) * SCR * sizeof(uint32_t)));
    GE_TRY(cudaMalloc(&dsam, (ns ? ns : 1) * OUT * sizeof(uint32_t)));
    GE_TRY(cudaMalloc(&dstats, sizeof(init)));
    GE_TRY(cudaMemcpy(dstats, init, sizeof(init), cudaMemcpyHostToDevice));
    for (uint64_t b = 0; b < n; b += chunk) {
        const uint32_t cnt = (uint32_t)(n - b < chunk ? n - b : chunk);
        k_ge_gen<OP><<<(cnt + 127) / 128, 128>>>(seed, b, cnt, din);
        k_ge_bulk<OP><<<(cnt + 127) / 128, 128>>>(b, cnt, stride, din, douts, dscr, dsam, dstats);
        GE_TRY(cudaGetLastError());
    }
    GE_TRY(cudaDeviceSynchronize());
    GE_TRY(cudaMemcpy(samples, dsam, ns * OUT * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    GE_TRY(cudaMemcpy(stats, dstats, sizeof(init), cudaMemcpyDeviceToHost));
done:
    cudaFree(din);
    cudaFree(douts);
    cudaFree(dscr);
    cudaFree(dsam);
    cudaFree(dstats);
    return e;
}

#define GE_OPS(X)                                                                                                        \
    X(GE_DECODE) X(GE_ENCODE) X(GE_ENCODE_CALL) X(GE_GROUP_KC) X(GE_GROUP_SIGN) X(GE_GROUP_SIGN2) X(GE_DBL) X(GE_DBL_CALL) \
    X(GE_ADDSUB) X(GE_ADDSUB_CALL) X(GE_TO_PRECOMP) X(GE_MADD) X(GE_CT_SELECT) X(GE_SMALL_MULT) X(GE_SMALL_MULT_CALL)      \
    X(GE_AFFINE_RUN) X(GE_AFFINE_RUN_CALL) X(GE_AFFINE_FWDBWD) X(GE_KEY_ROWS) X(GE_RECODE) X(GE_WELLFORMED)
static_assert(GE_OP_COUNT == 21, "GE_OPS lists every operation");

}  // namespace gesim

using namespace gesim;

extern "C" {

// out[n][ge_out_words(op)] = OP(in[n][ge_in_words(op)]) on the device
int ge_run(int op, const uint32_t* in, uint32_t* out, uint64_t n) {
    if (n == 0) return op >= 0 && op < GE_OP_COUNT ? 0 : (int)cudaErrorInvalidValue;
    switch (op) {
#define GE_CASE(OPC) case OPC: return (int)run<OPC>(in, out, n);
        GE_OPS(GE_CASE)
#undef GE_CASE
    default: return (int)cudaErrorInvalidValue;
    }
}

// stats[0] = items where the product form and the portable twin differ, stats[1] = the first such index (~0 if none);
// samples[(n + stride - 1) / stride][ge_out_words(op)] = the product form's output of items 0, stride, 2 stride, ...
int ge_bulk(int op, uint64_t seed, uint64_t n, uint64_t stride, uint32_t* samples, unsigned long long* stats) {
    if (stride == 0) return (int)cudaErrorInvalidValue;
    switch (op) {
#define GE_CASE(OPC) case OPC: return (int)bulk<OPC>(seed, n, stride, samples, stats);
        GE_OPS(GE_CASE)
#undef GE_CASE
    default: return (int)cudaErrorInvalidValue;
    }
}

// the numbering and widths this library was built with, so the tests can refuse a stale build
int ge_op_count(void) { return GE_OP_COUNT; }
int ge_words(int op, int which) { return which == 0 ? ge_in_words(op) : which == 1 ? ge_out_words(op) : ge_scratch_words(op); }

}  // extern "C"
