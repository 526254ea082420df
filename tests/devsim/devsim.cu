// tests/devsim — TEST-ONLY sm_90a build of devsim_ops.cuh (no torch, no libafcrypto.so).
//
// devsim_run:  one thread per item, the routine as the product kernels inline it; copies in, launches, synchronises, copies
//              out and returns the CUDA error (cudaErrorInvalidValue for an operation this build lacks).
// devsim_bulk: n items generated on the device from (seed, index) — each word is 0 with probability 1/16, all ones with
//              probability 1/8, else random — each run through the product form and the portable twin.  It counts the items
//              where the two differ and keeps the product form's output of every stride-th item, which the tests
//              regenerate and compare with Python integers.
#include "devsim_ops.cuh"

namespace devsim {

__host__ __device__ inline uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t gen_word(uint64_t seed, uint64_t i, int w) {
    const uint64_t z = mix64(seed + i * 32u + (uint64_t)w);
    const uint32_t sel = (uint32_t)(z >> 60);
    return sel == 0 ? 0u : sel <= 2 ? 0xffffffffu : (uint32_t)z;
}

template <int OP>
__global__ void k_devsim(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[32], y[16];
#pragma unroll
    for (int w = 0; w < 32; w++) x[w] = in[(size_t)i * 32 + w];
    run_op<OP, false>(x, y);
#pragma unroll
    for (int w = 0; w < 16; w++) out[(size_t)i * 16 + w] = y[w];
}

template <int OP>
__global__ void k_devsim_bulk(uint64_t seed, uint64_t n, uint64_t stride, uint32_t* __restrict__ samples,
                              unsigned long long* __restrict__ stats) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t x[32], y[16], z[16];
#pragma unroll
        for (int w = 0; w < 32; w++) x[w] = gen_word(seed, i, w);
        run_op<OP, false>(x, y);
        run_op<OP, true>(x, z);
        uint32_t d = 0;
#pragma unroll
        for (int w = 0; w < 16; w++) d |= y[w] ^ z[w];
        if (d) {
            atomicAdd(&stats[0], 1ull);
            atomicMin(&stats[1], (unsigned long long)i);
        }
        if (i % stride == 0) {
#pragma unroll
            for (int w = 0; w < 16; w++) samples[(i / stride) * 16 + w] = y[w];
        }
    }
}

template <int OP>
static cudaError_t launch(int bulk, const uint32_t* in, uint32_t* out, uint64_t n, uint64_t seed, uint64_t stride,
                          unsigned long long* stats) {
    if (!bulk) {
        k_devsim<OP><<<(unsigned)((n + 127) / 128), 128>>>(in, out, (int)n);
    } else {
        k_devsim_bulk<OP><<<132 * 16, 256>>>(seed, n, stride, out, stats);
    }
    return cudaGetLastError();
}

static cudaError_t dispatch(int op, int bulk, const uint32_t* in, uint32_t* out, uint64_t n, uint64_t seed, uint64_t stride,
                            unsigned long long* stats) {
    switch (op) {
#define DEVSIM_CASE(OPC) case OPC: return launch<OPC>(bulk, in, out, n, seed, stride, stats);
        DEVSIM_CASE(OP_MUL_WIDE) DEVSIM_CASE(OP_SQ_WIDE) DEVSIM_CASE(OP_MUL_WIDE_KARA) DEVSIM_CASE(OP_FOLD16)
        DEVSIM_CASE(OP_MUL) DEVSIM_CASE(OP_SQ) DEVSIM_CASE(OP_MUL_CALL) DEVSIM_CASE(OP_SQ_CALL) DEVSIM_CASE(OP_ADD)
        DEVSIM_CASE(OP_SUB) DEVSIM_CASE(OP_ADDSUB) DEVSIM_CASE(OP_TOWORDS) DEVSIM_CASE(OP_INVERT) DEVSIM_CASE(OP_POW22523)
        DEVSIM_CASE(OP_SC_REDUCE512) DEVSIM_CASE(OP_SC_REDUCE256) DEVSIM_CASE(OP_SC_MULADD)
#undef DEVSIM_CASE
    default: return cudaErrorInvalidValue;
    }
}

}  // namespace devsim

using namespace devsim;

#define DEVSIM_TRY(x) do { e = (x); if (e != cudaSuccess) goto done; } while (0)

extern "C" {

// out[n][16] = OP(in[n][32]) on the device
int devsim_run(int op, const uint32_t* in, uint32_t* out, uint64_t n) {
    if (op < 0 || op >= OP_COUNT) return (int)cudaErrorInvalidValue;
    if (n == 0) return 0;
    uint32_t *din = nullptr, *dout = nullptr;
    cudaError_t e = cudaSuccess;
    DEVSIM_TRY(cudaMalloc(&din, n * 32 * sizeof(uint32_t)));
    DEVSIM_TRY(cudaMalloc(&dout, n * 16 * sizeof(uint32_t)));
    DEVSIM_TRY(cudaMemcpy(din, in, n * 32 * sizeof(uint32_t), cudaMemcpyHostToDevice));
    DEVSIM_TRY(dispatch(op, 0, din, dout, n, 0, 0, nullptr));
    DEVSIM_TRY(cudaDeviceSynchronize());
    DEVSIM_TRY(cudaMemcpy(out, dout, n * 16 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
done:
    cudaFree(din);
    cudaFree(dout);
    return (int)e;
}

// stats[0] = items where the product form and the portable twin differ, stats[1] = the first such index (~0 if none);
// samples[(n + stride - 1) / stride][16] = the product form's output of items 0, stride, 2 stride, ...
int devsim_bulk(int op, uint64_t seed, uint64_t n, uint64_t stride, uint32_t* samples, unsigned long long* stats) {
    if (op < 0 || op >= OP_COUNT || stride == 0) return (int)cudaErrorInvalidValue;
    const uint64_t ns = (n + stride - 1) / stride;
    uint32_t* dsam = nullptr;
    unsigned long long* dstats = nullptr;
    const unsigned long long init[2] = {0ull, ~0ull};
    cudaError_t e = cudaSuccess;
    DEVSIM_TRY(cudaMalloc(&dsam, (ns ? ns : 1) * 16 * sizeof(uint32_t)));
    DEVSIM_TRY(cudaMalloc(&dstats, sizeof(init)));
    DEVSIM_TRY(cudaMemcpy(dstats, init, sizeof(init), cudaMemcpyHostToDevice));
    DEVSIM_TRY(dispatch(op, 1, nullptr, dsam, n, seed, stride, dstats));
    DEVSIM_TRY(cudaDeviceSynchronize());
    DEVSIM_TRY(cudaMemcpy(samples, dsam, ns * 16 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    DEVSIM_TRY(cudaMemcpy(stats, dstats, sizeof(init), cudaMemcpyDeviceToHost));
done:
    cudaFree(dsam);
    cudaFree(dstats);
    return (int)e;
}

// the OP_* numbering this library was built with, so the tests can refuse a stale build
int devsim_op_count(void) { return OP_COUNT; }

}  // extern "C"
