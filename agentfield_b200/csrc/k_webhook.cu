// Execution webhook deliveries built and signed on the device (afc_webhook_sign_batch, include/afcrypto.h; afc_webhook.cuh).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_wh_sizes / k_wh_emit   determineWebhookEvent + buildPayload + json.Marshal   internal/services/webhook_dispatcher.go:296-299, 394-468
//   k_wh_hmac / k_wh_header  generateWebhookSignature                             internal/services/webhook_dispatcher.go:318-320, 470-474
//
// One delivery per thread.  k_wh_sizes decides each delivery's plan (event, result kind, or WH_HOST), checks and counts its body —
// the result's re-marshalling included — and the existing scan turns the lengths into offsets; k_wh_emit writes the bodies; k_wh_hmac
// computes the HMAC over each body and k_wh_header writes the 71-character header (zeros without a secret or for a WH_HOST delivery).  A batch
// waits for its longest result: one thread walks each.
#include "afc_launch.h"
#include "afc_webhook.cuh"

namespace afc {

static constexpr int WH_THREADS = 128;

__device__ __forceinline__ WhItem wh_item(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* flags,
                                          const uint8_t* results, const uint64_t* result_off, uint32_t i) {
    WhItem it;
    it.cols = cols; it.coff = col_off + (size_t)i * WH_COLUMNS; it.duration = duration[i]; it.flags = flags[i];
    const uint64_t r0 = result_off[i];
    it.result = results + r0; it.result_len = result_off[i + 1] - r0;
    return it;
}
// the delivery's tape: one uint32 entry per two bytes of result text, at its place in the batch's result bytes
__device__ __forceinline__ uint32_t* wh_tape(uint32_t* tape, const uint64_t* result_off, uint32_t i) {
    return tape + (result_off[i] - result_off[0]) / 2;
}

__global__ void __maxnreg__(64)
k_wh_sizes(const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off, const int64_t* __restrict__ duration,
           const uint8_t* __restrict__ flags, const uint8_t* __restrict__ results, const uint64_t* __restrict__ result_off, uint32_t n,
           uint32_t* __restrict__ tape, uint8_t* __restrict__ plan, uint64_t* __restrict__ body_len, uint8_t* __restrict__ status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const WhItem it = wh_item(cols, col_off, duration, flags, results, result_off, i);
    uint32_t p = wh_plan(it);
    ByteCounter c; c.init();
    if (!(p & WH_P_HOST) && !wh_body(c, it, p, wh_tape(tape, result_off, i))) p = WH_P_HOST;
    plan[i] = (uint8_t)p;
    status[i] = (p & WH_P_HOST) ? WH_HOST : WH_BUILT;
    body_len[i] = (p & WH_P_HOST) ? 0 : c.n;
}

__global__ void __maxnreg__(64)
k_wh_emit(const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off, const int64_t* __restrict__ duration,
          const uint8_t* __restrict__ flags, const uint8_t* __restrict__ results, const uint64_t* __restrict__ result_off, uint32_t n,
          uint32_t* __restrict__ tape, const uint8_t* __restrict__ plan, const uint64_t* __restrict__ body_off, uint8_t* __restrict__ bodies) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t p = plan[i];
    if (p & WH_P_HOST) return;
    ByteWriter w; w.init(bodies + body_off[i]);
    wh_body(w, wh_item(cols, col_off, duration, flags, results, result_off, i), p, wh_tape(tape, result_off, i));
    w.finish();
}

// HMAC-SHA256 of each built body under its secret (the digest at mac + 32 i); skips the rest.  Under __launch_bounds__(128) ptxas
// holds hmac_sha256_msg in 80 registers and spills 60 bytes; 92 registers hold it without.
__global__ void __maxnreg__(128)
k_wh_hmac(const uint8_t* __restrict__ secrets, const uint32_t* __restrict__ secret_off, const uint8_t* __restrict__ flags,
          const uint8_t* __restrict__ status, const uint8_t* __restrict__ bodies, const uint64_t* __restrict__ body_off, uint32_t n,
          uint8_t* __restrict__ mac) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || status[i] != WH_BUILT || !(flags[i] & WH_HAS_SECRET)) return;
    const uint32_t k0 = secret_off[i];
    const uint64_t b0 = body_off[i];
    uint32_t st[8];
    hmac_sha256_msg(st, secrets + k0, secret_off[i + 1] - k0, bodies + b0, body_off[i + 1] - b0);
    store_digest256(mac + 32ull * i, st);
}

// the 71 header characters of each delivery: "sha256=" + hex(mac), or zeros
__global__ void __launch_bounds__(WH_THREADS)
k_wh_header(const uint8_t* __restrict__ flags, const uint8_t* __restrict__ status, const uint8_t* __restrict__ mac, uint32_t n,
            uint8_t* __restrict__ headers) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    wh_header_text(headers + (size_t)i * WH_HEADER_CHARS, status[i] == WH_BUILT && (flags[i] & WH_HAS_SECRET) ? mac + 32ull * i : nullptr);
}

namespace launch {

static inline uint32_t wh_blocks(uint64_t n) { return (uint32_t)((n + WH_THREADS - 1) / WH_THREADS); }

cudaError_t wh_sizes(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* flags, const uint8_t* results,
                     const uint64_t* result_off, uint32_t n, uint32_t* tape, uint8_t* plan, uint64_t* body_len, uint8_t* status, cudaStream_t s,
                     LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_wh_sizes", s, k_wh_sizes<<<wh_blocks(n), WH_THREADS, 0, s>>>(cols, col_off, duration, flags, results, result_off, n, tape, plan,
                                                                                  body_len, status));
    return cudaGetLastError();
}
cudaError_t wh_emit(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* flags, const uint8_t* results,
                    const uint64_t* result_off, uint32_t n, uint32_t* tape, const uint8_t* plan, const uint64_t* body_off, uint8_t* bodies,
                    cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_wh_emit", s, k_wh_emit<<<wh_blocks(n), WH_THREADS, 0, s>>>(cols, col_off, duration, flags, results, result_off, n, tape, plan,
                                                                                body_off, bodies));
    return cudaGetLastError();
}
cudaError_t wh_sign(const uint8_t* secrets, const uint32_t* secret_off, const uint8_t* flags, const uint8_t* status, const uint8_t* bodies,
                    const uint64_t* body_off, uint32_t n, uint8_t* mac, uint8_t* headers, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_wh_hmac", s, k_wh_hmac<<<wh_blocks(n), WH_THREADS, 0, s>>>(secrets, secret_off, flags, status, bodies, body_off, n, mac));
    AFC_LAUNCH(lg, "k_wh_header", s, k_wh_header<<<wh_blocks(n), WH_THREADS, 0, s>>>(flags, status, mac, n, headers));
    return cudaGetLastError();
}
uint64_t wh_fixed_bytes() { return afc::wh_fixed_bytes(); }

}  // namespace launch
}  // namespace afc
