/*
 * stream_ceiling.cu -- the streaming ceiling of a 4-read / 1-write fp32 kernel on this GPU (tools/stream_probe.py).
 *
 * No interpreter, no staging: a grid-stride loop that reads four arrays with 128-bit ld.global.nc, adds them and
 * writes one array with 128-bit st.global.cs.  Its time is what HBM allows for C2's traffic (16 B read + 4 B written
 * per element), the figure the fused sweep kernel is compared with.
 */
#include <cuda_runtime.h>
#include <stddef.h>

namespace {

__global__ void stream4to1(const float4 *__restrict__ x0, const float4 *__restrict__ x1, const float4 *__restrict__ x2,
                           const float4 *__restrict__ x3, float4 *__restrict__ out, size_t n4) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t) gridDim.x * blockDim.x) {
        const float4 a = __ldg(x0 + i), b = __ldg(x1 + i), c = __ldg(x2 + i), d = __ldg(x3 + i);
        __stcs(out + i, make_float4((a.x + b.x) + (c.x + d.x), (a.y + b.y) + (c.y + d.y),
                                    (a.z + b.z) + (c.z + d.z), (a.w + b.w) + (c.w + d.w)));
    }
}

} // namespace

/* Times `reps` launches of the ceiling kernel over n fp32 elements (n a multiple of 4) with `block` threads and
   `ctas_per_sm` CTAs per SM, each launch between its own pair of CUDA events, after `warmup` untimed launches.
   Writes the best launch time to *best_ms.  Returns 0 or a cudaError_t. */
extern "C" __attribute__((visibility("default")))
int sc_ceiling(size_t n, int block, int ctas_per_sm, int warmup, int reps, float *best_ms) {
    float *buf[5] = {};
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int dev = 0, sms = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err == cudaSuccess) err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    for (int k = 0; k < 5 && err == cudaSuccess; ++k) {
        err = cudaMalloc(&buf[k], n * sizeof(float));
        if (err == cudaSuccess) err = cudaMemset(buf[k], 0, n * sizeof(float));
    }
    if (err == cudaSuccess) err = cudaEventCreate(&e0);
    if (err == cudaSuccess) err = cudaEventCreate(&e1);
    const size_t n4 = n / 4;
    const unsigned grid = (unsigned) sms * (unsigned) ctas_per_sm;
    float best = 1e30f;
    for (int r = 0; r < warmup + reps && err == cudaSuccess; ++r) {
        cudaEventRecord(e0);
        stream4to1<<<grid, block>>>((const float4 *) buf[0], (const float4 *) buf[1], (const float4 *) buf[2],
                                    (const float4 *) buf[3], (float4 *) buf[4], n4);
        cudaEventRecord(e1);
        err = cudaEventSynchronize(e1);
        if (err == cudaSuccess) err = cudaGetLastError();
        float ms = 0.f;
        if (err == cudaSuccess) err = cudaEventElapsedTime(&ms, e0, e1);
        if (err == cudaSuccess && r >= warmup && ms < best) best = ms;
    }
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    for (float *p : buf) if (p) cudaFree(p);
    *best_ms = best;
    return (int) err;
}
