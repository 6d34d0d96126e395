/*
 * ek_scan.cu -- prefix sum and stream compaction on raw device memory.
 *
 * ABI-compatible with cuda_psum / cuda_compress (src/cuda/horiz.cu:124-200), which the
 * reference implements with cub::DeviceScan::InclusiveSum / DeviceSelect::Flagged.
 * Hand-written three-phase scan: (1) per-tile reduction, (2) single-CTA scan of the
 * tile totals, (3) per-tile scan + carry-in.  Tiles are TILE = 256 threads x 8 items;
 * warp-shuffle scans inside the tile.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <algorithm>
#include <cstdlib>
#include "ek_internal.h"

namespace {

constexpr int THREADS = 256, ITEMS = 8, TILE = THREADS * ITEMS;

template <typename T> __device__ __forceinline__ T warp_incl_scan(T v) {
    unsigned lane = threadIdx.x & 31u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= (unsigned) d) v = v + o;
    }
    return v;
}

/* inclusive scan of one value per thread across the CTA; returns the CTA total in `total` */
template <typename T> __device__ __forceinline__ T block_incl_scan(T v, T &total) {
    __shared__ __align__(16) unsigned char raw[32 * sizeof(T) + sizeof(T)];
    T *warp_tot = reinterpret_cast<T *>(raw);
    unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    T s = warp_incl_scan(v);
    __syncthreads();
    if (lane == 31) warp_tot[w] = s;
    __syncthreads();
    if (w == 0) {
        T t = lane < (blockDim.x >> 5) ? warp_tot[lane] : T(0);
        t = warp_incl_scan(t);
        warp_tot[lane] = t;
    }
    __syncthreads();
    if (w > 0) s = s + warp_tot[w - 1];
    total = warp_tot[(blockDim.x >> 5) - 1];
    return s;
}

template <typename T, typename In, typename F>
__global__ void __launch_bounds__(THREADS) tile_reduce(const In *in, T *tile_sum, size_t n, F conv) {
    size_t base = (size_t) blockIdx.x * TILE;
    T acc = T(0);
    /* blocked order: thread t owns items [t*ITEMS, t*ITEMS+ITEMS) so that phase 3 can scan serially */
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        size_t i = base + (size_t) threadIdx.x * ITEMS + j;
        if (i < n) acc = acc + conv(in[i]);
    }
    T total;
    block_incl_scan(acc, total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

template <typename T> __global__ void __launch_bounds__(THREADS) scan_tile_sums(T *tile_sum, size_t n_tiles) {
    /* single CTA, exclusive scan in place (carry kept in a register across rounds) */
    T carry = T(0);
    for (size_t base = 0; base < n_tiles; base += THREADS) {
        size_t i = base + threadIdx.x;
        T v = i < n_tiles ? tile_sum[i] : T(0);
        T total;
        T s = block_incl_scan(v, total);
        if (i < n_tiles) tile_sum[i] = carry + (s - v);
        carry = carry + total;
        __syncthreads();
    }
}

template <typename T> __global__ void __launch_bounds__(THREADS)
tile_scan_incl(const T *in, T *out, const T *tile_off, size_t n) {
    size_t base = (size_t) blockIdx.x * TILE + (size_t) threadIdx.x * ITEMS;
    T v[ITEMS];
    T acc = T(0);
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) { v[j] = base + j < n ? in[base + j] : T(0); acc = acc + v[j]; v[j] = acc; }
    T total;
    T s = block_incl_scan(acc, total);
    T off = tile_off[blockIdx.x] + (s - acc);
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) if (base + j < n) out[base + j] = off + v[j];
}

template <typename T> __global__ void __launch_bounds__(THREADS)
tile_compact(const T *in, const uint8_t *mask, T *out, const uint32_t *tile_off, size_t n) {
    size_t base = (size_t) blockIdx.x * TILE + (size_t) threadIdx.x * ITEMS;
    uint32_t flag[ITEMS], cnt = 0;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) { flag[j] = (base + j < n && mask[base + j]) ? 1u : 0u; cnt += flag[j]; }
    uint32_t total;
    uint32_t s = block_incl_scan(cnt, total);
    uint32_t pos = tile_off[blockIdx.x] + (s - cnt);
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) if (flag[j]) out[pos++] = in[base + j];
}

struct ConvId { template <typename T> __device__ T operator()(T v) const { return v; } };
struct ConvFlag { __device__ uint32_t operator()(uint8_t v) const { return v ? 1u : 0u; } };

template <typename T> void scan_incl(const T *in, T *out, size_t n) {
    EkContext &ctx = ek_ctx();
    size_t n_tiles = (n + TILE - 1) / TILE;
    T *tile = (T *) ek_malloc(n_tiles * sizeof(T));
    tile_reduce<T, T, ConvId><<<(unsigned) n_tiles, THREADS, 0, ctx.stream>>>(in, tile, n, ConvId());
    scan_tile_sums<T><<<1, THREADS, 0, ctx.stream>>>(tile, n_tiles);
    tile_scan_incl<T><<<(unsigned) n_tiles, THREADS, 0, ctx.stream>>>(in, out, tile, n);
    ek_cuda_check(cudaGetLastError());
    ctx.stats.launches += 3;
    ek_free(tile);
}

template <typename T> void *psum_impl(size_t n, const void *data) {
    T *out = (T *) ek_malloc(n * sizeof(T));
    scan_incl<T>((const T *) data, out, n);
    return out;
}

template <typename T> int compress_impl(size_t n, const void *data, const uint8_t *mask, void **out_data, size_t *out_size) {
    EkContext &ctx = ek_ctx();
    size_t n_tiles = (n + TILE - 1) / TILE;
    uint32_t *tile = (uint32_t *) ek_malloc((n_tiles + 1) * sizeof(uint32_t));
    tile_reduce<uint32_t, uint8_t, ConvFlag><<<(unsigned) n_tiles, THREADS, 0, ctx.stream>>>(mask, tile, n, ConvFlag());
    /* keep the grand total: read the last tile's exclusive offset + its count */
    uint32_t last_count = 0, last_off = 0;
    ek_cuda_check(cudaMemcpyAsync(&last_count, tile + n_tiles - 1, 4, cudaMemcpyDeviceToHost, ctx.stream));
    scan_tile_sums<uint32_t><<<1, THREADS, 0, ctx.stream>>>(tile, n_tiles);
    ek_cuda_check(cudaMemcpyAsync(&last_off, tile + n_tiles - 1, 4, cudaMemcpyDeviceToHost, ctx.stream));
    ek_cuda_check(cudaStreamSynchronize(ctx.stream));          /* blocking like horiz.cu:143 */
    size_t total = (size_t) last_off + last_count;
    T *out = (T *) ek_malloc(std::max<size_t>(total, 1) * sizeof(T));
    tile_compact<T><<<(unsigned) n_tiles, THREADS, 0, ctx.stream>>>((const T *) data, mask, out, tile, n);
    ek_cuda_check(cudaGetLastError());
    ctx.stats.launches += 3;
    ek_free(tile);
    *out_data = out; *out_size = total;
    return 0;
}


} // namespace

void ek_scan_incl_u32(const uint32_t *in, uint32_t *out, size_t n) { scan_incl<uint32_t>(in, out, n); }

extern "C" {

void *ek_psum(ek_type type, size_t n, const void *data) {
    if (n == 0) { ek_set_error("ek_psum(): empty array"); return nullptr; }
    if (ek_init() != 0) return nullptr;
    switch (type) {
        case EK_INT32: case EK_UINT32: return psum_impl<uint32_t>(n, data);
        case EK_INT64: case EK_UINT64: return psum_impl<unsigned long long>(n, data);
        case EK_FLOAT32: return psum_impl<float>(n, data);
        case EK_FLOAT64: return psum_impl<double>(n, data);
        case EK_FLOAT16: ek_set_error("ek_psum(): Float16 is a storage format: convert to Float32 to compute"); return nullptr;
        default: ek_set_error("ek_psum(): unsupported type"); return nullptr;
    }
}

int ek_compress(ek_type type, size_t n, const void *data, const uint8_t *mask, void **out_data, size_t *out_size) {
    if (n == 0) { *out_data = nullptr; *out_size = 0; return 0; }
    if (ek_init() != 0) return -1;
    switch (ek_type_size(type)) {
        case 1: return compress_impl<uint8_t>(n, data, mask, out_data, out_size);
        case 2: return compress_impl<uint16_t>(n, data, mask, out_data, out_size);
        case 4: return compress_impl<uint32_t>(n, data, mask, out_data, out_size);
        case 8: return compress_impl<uint64_t>(n, data, mask, out_data, out_size);
        default: ek_set_error("ek_compress(): unsupported type"); return -1;
    }
}

} /* extern "C" */
