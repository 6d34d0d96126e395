/*
 * ek_partition.cu -- cuda_partition (horiz.cu:35-122): groups the indices 0..n-1 of a pointer array by pointer value
 * for virtual-call dispatch.  Results: the distinct pointers ascending, and per pointer the ascending list of the
 * indices that hold it (what the reference's stable radix sort + run-length encode produce).
 *
 * Device path, up to PART_MAX_GROUPS distinct values:
 *   (1) part_insert: one pass over the keys.  An open-addressed table (linear probing, CAS on an empty marker) gives
 *       every distinct key a slot and a dense id; lanes of a warp holding the same key elect one leader with
 *       __match_any_sync, so a warp probes once per distinct key.  Every element writes its slot (4 B).
 *       part_count: slot -> dense id in place, and the count per id from privatised shared-memory bins.
 *   (2) host: read back K, the K keys and counts (O(K) bytes, the only synchronisation), sort the keys, upload an
 *       id -> rank map and the K output lists, each ek_malloc'd from its count.
 *   (3) LSD radix passes over the rank, 8 bits each (one pass for K <= 256, two above): per-tile digit histogram,
 *       inclusive scan of the digit-major [digit][tile] counts (ek_scan.cu's three-phase scan), stable scatter
 *       (warp ranking with __match_any_sync + __popc, warps combined in order in shared memory).  The last pass writes
 *       each index straight into its group's list.
 * More distinct values than PART_MAX_GROUPS set the overflow flag and the call falls back to a host-side stable sort.
 *
 * Bytes per element moved, against the algorithmic 12 (8 B key read, 4 B index written): insert 8 + 4, count 4 + 4,
 * and per radix pass 256 digit counts per 4096-element tile (written, scanned with two reads and a write, read by the
 * scatter: 1.25 B).  One pass (K <= 256): histogram 4, scatter 4 + 4 -> 33.25 B.  Two passes: histogram 4, scatter
 * 4 + 8 to (rank, index) pairs, histogram 8, scatter 8 + 4 -> 58.5 B.  The id -> rank and group tables are O(K) and
 * stay in L2.
 */
#ifndef EK_HOST_EMU          /* tests/cpu_kernel compiles the kernels of this file as host code (cuda_shim.h) */
#include <cuda_runtime.h>
#include <algorithm>
#include <numeric>
#include <vector>
#include "ek_internal.h"
#endif
#include <stdint.h>

namespace {

constexpr uint32_t PART_THREADS = 256, PART_WARPS = PART_THREADS / 32;
constexpr uint32_t PART_MAX_GROUPS = 1u << 16;      /* distinct values grouped on the device (two 8-bit radix passes) */
constexpr uint32_t PART_SLOTS = 1u << 17;           /* hash table slots: load factor <= 1/2 at PART_MAX_GROUPS */
constexpr uint32_t PART_TOP_SLOT = PART_SLOTS;      /* slot of the key ~0, which is the table's empty marker */
constexpr uint64_t PART_EMPTY = ~0ull;
constexpr uint32_t PART_COUNT_BINS = 1u << 13;      /* shared count bins per CTA (32 KiB); higher ids count in global */
constexpr uint32_t RADIX_BINS = 256, RADIX_ITEMS = 16, RADIX_TILE = PART_THREADS * RADIX_ITEMS;
constexpr uint32_t NO_DIGIT = RADIX_BINS;           /* lanes past the end */
static_assert(RADIX_BINS == PART_THREADS, "one digit per thread in the histogram and the warp combine");

struct PartHeader { uint32_t n_ids, overflow, top_claimed, pad; };

#ifdef EK_HOST_EMU
#define PART_SMEM(name) uint32_t *name = reinterpret_cast<uint32_t *>(emu::smem_)
#else
#define PART_SMEM(name) extern __shared__ uint32_t name[]
#endif

/* pointers are 16-byte aligned and share their high bits: mix every bit into the slot (murmur3 finaliser) */
__device__ __forceinline__ uint32_t part_hash(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (uint32_t) k & (PART_SLOTS - 1u);
}

__device__ __forceinline__ void part_new_id(uint32_t s, uint64_t k, uint32_t *slot_id, uint64_t *id_key, PartHeader *hdr) {
    const uint32_t id = atomicAdd(&hdr->n_ids, 1u);
    if (id < PART_MAX_GROUPS) { slot_id[s] = id; id_key[id] = k; }
    else *(volatile uint32_t *) &hdr->overflow = 1u;
}

/* slot of key k, inserting it if it is new; every probe loop is bounded by the table size */
__device__ uint32_t part_find_or_insert(uint64_t k, uint64_t *table, uint32_t *slot_id, uint64_t *id_key, PartHeader *hdr) {
    if (k == PART_EMPTY) {
        if (atomicCAS(&hdr->top_claimed, 0u, 1u) == 0u) part_new_id(PART_TOP_SLOT, k, slot_id, id_key, hdr);
        return PART_TOP_SLOT;
    }
    uint32_t s = part_hash(k);
    for (uint32_t probe = 0; probe < PART_SLOTS; ++probe, s = (s + 1u) & (PART_SLOTS - 1u)) {
        uint64_t cur = table[s];                /* a stale EMPTY only costs a CAS: occupied slots never change */
        if (cur == PART_EMPTY) {
            cur = atomicCAS((unsigned long long *) &table[s], (unsigned long long) PART_EMPTY, (unsigned long long) k);
            if (cur == PART_EMPTY) { part_new_id(s, k, slot_id, id_key, hdr); return s; }
        }
        if (cur == k) return s;
    }
    *(volatile uint32_t *) &hdr->overflow = 1u;
    return 0;
}

/* (1) slot_of[i] = table slot of keys[i]; the grid strides over warps of 32 consecutive elements */
__global__ void __launch_bounds__(PART_THREADS)
part_insert(const uint64_t *keys, size_t n, uint32_t *slot_of, uint64_t *table, uint32_t *slot_id, uint64_t *id_key,
            PartHeader *hdr) {
    const uint32_t lane = threadIdx.x & 31u;
    const size_t stride = (size_t) gridDim.x * PART_THREADS;
    for (size_t base = (size_t) blockIdx.x * PART_THREADS + (threadIdx.x & ~31u); base < n; base += stride) {
        /* once the table has overflowed the result is discarded: stop probing */
        const uint32_t over = __shfl_sync(~0u, lane == 0 ? *(volatile uint32_t *) &hdr->overflow : 0u, 0);
        if (over) return;
        const size_t i = base + lane;
        const unsigned active = __ballot_sync(~0u, i < n);
        if (i < n) {
            const uint64_t k = keys[i];
            const unsigned peers = __match_any_sync(active, k);
            const uint32_t leader = (uint32_t) __ffs(peers) - 1u;
            uint32_t s = 0;
            if (lane == leader) s = part_find_or_insert(k, table, slot_id, id_key, hdr);
            slot_of[i] = __shfl_sync(active, s, leader);
        }
    }
}

/* (1b) ids[i] = dense id of slot ids[i], counts[id] += 1.  Ids below PART_COUNT_BINS count in shared bins flushed once
   per CTA (the first-seen, typically hottest keys); the rest -- only when K > PART_COUNT_BINS -- with one global atomic
   per distinct id per warp. */
__global__ void __launch_bounds__(PART_THREADS)
part_count(uint32_t *ids, size_t n, const uint32_t *slot_id, const PartHeader *hdr, uint32_t *counts) {
    PART_SMEM(bins);
    if (hdr->overflow) return;
    const uint32_t nb = min(hdr->n_ids, PART_COUNT_BINS);
    for (uint32_t b = threadIdx.x; b < nb; b += PART_THREADS) bins[b] = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u;
    const size_t stride = (size_t) gridDim.x * PART_THREADS;
    for (size_t base = (size_t) blockIdx.x * PART_THREADS + (threadIdx.x & ~31u); base < n; base += stride) {
        const size_t i = base + lane;
        const unsigned active = __ballot_sync(~0u, i < n);
        if (i < n) {
            const uint32_t id = slot_id[ids[i]];
            ids[i] = id;
            const unsigned peers = __match_any_sync(active, id);
            if (lane == (uint32_t) __ffs(peers) - 1u)
                atomicAdd(id < PART_COUNT_BINS ? &bins[id] : &counts[id], (uint32_t) __popc(peers));
        }
    }
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < nb; b += PART_THREADS)
        if (bins[b]) atomicAdd(&counts[b], bins[b]);
}

/* element i of a radix pass: the first pass reads its id (rank through id_rank), later ones the pair the previous pass
   wrote */
template <bool FIRST>
__device__ __forceinline__ void part_load(const uint32_t *ids, const uint64_t *pairs, const uint32_t *id_rank, size_t i,
                                          uint32_t &rank, uint32_t &idx) {
    if (FIRST) { rank = id_rank[ids[i]]; idx = (uint32_t) i; }
    else { const uint64_t p = pairs[i]; rank = (uint32_t) (p >> 32); idx = (uint32_t) p; }
}

/* (3a) hist[d * n_tiles + tile] = number of elements of the tile whose digit is d */
template <bool FIRST>
__global__ void __launch_bounds__(PART_THREADS)
part_hist(const uint32_t *ids, const uint64_t *pairs, const uint32_t *id_rank, size_t n, uint32_t shift,
          uint32_t *hist, uint32_t n_tiles) {
    PART_SMEM(bins);
    bins[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u;
    const size_t base = (size_t) blockIdx.x * RADIX_TILE + (size_t) (threadIdx.x >> 5) * (32u * RADIX_ITEMS) + lane;
    for (uint32_t j = 0; j < RADIX_ITEMS; ++j) {
        const size_t i = base + (size_t) j * 32u;
        uint32_t d = NO_DIGIT;
        if (i < n) { uint32_t r, x; part_load<FIRST>(ids, pairs, id_rank, i, r, x); d = (r >> shift) & 0xffu; }
        const unsigned peers = __match_any_sync(~0u, d);
        if (d != NO_DIGIT && lane == (uint32_t) __ffs(peers) - 1u) atomicAdd(&bins[d], (uint32_t) __popc(peers));
    }
    __syncthreads();
    hist[(size_t) threadIdx.x * n_tiles + blockIdx.x] = bins[threadIdx.x];
}

/* (3c) stable scatter by digit.  Warp w owns the tile's elements [w * 512, (w + 1) * 512) and ranks them round by round
   (32 consecutive elements per round) with a per-warp running count per digit; warps are then combined in warp order,
   tiles in tile order through the scanned histogram.  The last pass writes index idx of rank r to
   lists[r][position - group_start[r]], earlier ones (rank, idx) pairs. */
template <bool FIRST, bool LAST>
__global__ void __launch_bounds__(PART_THREADS)
part_scatter(const uint32_t *ids, const uint64_t *pairs_in, const uint32_t *id_rank, size_t n, uint32_t shift,
             const uint32_t *hist_incl, uint32_t n_tiles, uint64_t *pairs_out, uint32_t *const *lists,
             const uint32_t *group_start) {
    PART_SMEM(smem);
    uint32_t *warp_cnt = smem;                                   /* [warp][digit] */
    uint32_t *tile_off = smem + PART_WARPS * RADIX_BINS;         /* [digit]       */
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    for (uint32_t k = threadIdx.x; k < PART_WARPS * RADIX_BINS; k += PART_THREADS) warp_cnt[k] = 0;
    __syncthreads();
    uint32_t *my_cnt = warp_cnt + w * RADIX_BINS;
    const uint32_t lt = (1u << lane) - 1u;
    const size_t base = (size_t) blockIdx.x * RADIX_TILE + (size_t) w * (32u * RADIX_ITEMS) + lane;
    uint32_t rank[RADIX_ITEMS], idx[RADIX_ITEMS], pos[RADIX_ITEMS];
#pragma unroll
    for (uint32_t j = 0; j < RADIX_ITEMS; ++j) {
        const size_t i = base + (size_t) j * 32u;
        uint32_t d = NO_DIGIT;
        rank[j] = 0; idx[j] = 0;
        if (i < n) { part_load<FIRST>(ids, pairs_in, id_rank, i, rank[j], idx[j]); d = (rank[j] >> shift) & 0xffu; }
        const unsigned peers = __match_any_sync(~0u, d);
        const uint32_t leader = (uint32_t) __ffs(peers) - 1u;
        uint32_t before = 0;
        if (lane == leader && d != NO_DIGIT) { before = my_cnt[d]; my_cnt[d] = before + (uint32_t) __popc(peers); }
        pos[j] = __shfl_sync(~0u, before, leader) + (uint32_t) __popc(peers & lt);
        __syncwarp();
    }
    __syncthreads();
    {   /* thread d: exclusive scan of digit d over the warps; the tile's first position for d */
        const uint32_t d = threadIdx.x;
        uint32_t run = 0;
        for (uint32_t v = 0; v < PART_WARPS; ++v) {
            const uint32_t c = warp_cnt[v * RADIX_BINS + d];
            warp_cnt[v * RADIX_BINS + d] = run;
            run += c;
        }
        tile_off[d] = hist_incl[(size_t) d * n_tiles + blockIdx.x] - run;
    }
    __syncthreads();
#pragma unroll
    for (uint32_t j = 0; j < RADIX_ITEMS; ++j) {
        if (base + (size_t) j * 32u >= n) break;
        const uint32_t d = (rank[j] >> shift) & 0xffu;
        const uint32_t p = tile_off[d] + my_cnt[d] + pos[j];
        if (LAST) lists[rank[j]][p - group_start[rank[j]]] = idx[j];
        else pairs_out[p] = ((uint64_t) rank[j] << 32) | idx[j];
    }
}

} // namespace

#ifndef EK_HOST_EMU
namespace {

int partition_host_sort(EkContext &ctx, size_t n, const uint64_t *keys, std::vector<uint64_t> &uniq,
                        std::vector<uint32_t> &cnts, uint32_t **&perm_h) {
    std::vector<uint64_t> hk(n);
    ek_cuda_check(cudaMemcpyAsync(hk.data(), keys, n * 8, cudaMemcpyDeviceToHost, ctx.stream));
    ek_cuda_check(cudaStreamSynchronize(ctx.stream));
    std::vector<uint32_t> order(n);
    for (size_t i = 0; i < n; ++i) order[i] = (uint32_t) i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return hk[a] < hk[b]; });
    std::vector<size_t> starts;
    for (size_t i = 0; i < n; ++i) if (i == 0 || hk[order[i]] != hk[order[i - 1]]) { starts.push_back(i); uniq.push_back(hk[order[i]]); }
    starts.push_back(n);
    perm_h = (uint32_t **) malloc(sizeof(uint32_t *) * uniq.size());
    for (size_t k = 0; k < uniq.size(); ++k) {
        uint32_t c = (uint32_t) (starts[k + 1] - starts[k]);
        cnts.push_back(c);
        perm_h[k] = (uint32_t *) ek_malloc((size_t) c * 4);
        ek_cuda_check(cudaMemcpyAsync(perm_h[k], order.data() + starts[k], (size_t) c * 4, cudaMemcpyHostToDevice, ctx.stream));
    }
    ek_cuda_check(cudaStreamSynchronize(ctx.stream));
    return 0;
}

/* returns false (and allocates nothing that outlives the call) when there are more than PART_MAX_GROUPS distinct keys */
bool partition_device(EkContext &ctx, size_t n, const uint64_t *keys, std::vector<uint64_t> &uniq,
                      std::vector<uint32_t> &cnts, uint32_t **&perm_h) {
    cudaStream_t st = ctx.stream;
    /* scratch: hash table (keys, slot -> id), header + counts + id -> key, one id per element */
    const size_t table_bytes = (size_t) PART_SLOTS * 8, slot_id_bytes = (size_t) (PART_SLOTS + 1) * 4;
    const size_t counts_off = sizeof(PartHeader), keys_off = counts_off + (size_t) PART_MAX_GROUPS * 4;
    uint8_t *table = (uint8_t *) ek_malloc(table_bytes + slot_id_bytes);
    uint8_t *meta = (uint8_t *) ek_malloc(keys_off + (size_t) PART_MAX_GROUPS * 8);
    uint32_t *ids = (uint32_t *) ek_malloc(n * 4);
    PartHeader *hdr = (PartHeader *) meta;
    uint32_t *counts = (uint32_t *) (meta + counts_off);
    uint64_t *id_key = (uint64_t *) (meta + keys_off);
    uint32_t *slot_id = (uint32_t *) (table + table_bytes);
    ek_cuda_check(cudaMemsetAsync(table, 0xff, table_bytes, st));
    ek_cuda_check(cudaMemsetAsync(meta, 0, keys_off, st));
    const unsigned grid = (unsigned) std::min<size_t>((n + PART_THREADS - 1) / PART_THREADS, (size_t) ctx.num_sms * 8);
    part_insert<<<grid, PART_THREADS, 0, st>>>(keys, n, ids, (uint64_t *) table, slot_id, id_key, hdr);
    part_count<<<grid, PART_THREADS, PART_COUNT_BINS * 4, st>>>(ids, n, slot_id, hdr, counts);
    ek_cuda_check(cudaGetLastError());
    ctx.stats.launches += 2;

    /* (2) read back K, the keys and their counts: the first 256 with the header, the rest only when there are more */
    constexpr uint32_t FIRST_READ = 256;
    PartHeader h;
    std::vector<uint64_t> hkey(FIRST_READ);
    std::vector<uint32_t> hcnt(FIRST_READ);
    ek_cuda_check(cudaMemcpyAsync(&h, hdr, sizeof(h), cudaMemcpyDeviceToHost, st));
    ek_cuda_check(cudaMemcpyAsync(hcnt.data(), counts, FIRST_READ * 4, cudaMemcpyDeviceToHost, st));
    ek_cuda_check(cudaMemcpyAsync(hkey.data(), id_key, FIRST_READ * 8, cudaMemcpyDeviceToHost, st));
    ek_cuda_check(cudaStreamSynchronize(st));
    auto release = [&]() { ek_free(table); ek_free(meta); ek_free(ids); };
    if (h.overflow || h.n_ids > PART_MAX_GROUPS) { release(); return false; }
    const uint32_t K = h.n_ids;
    hkey.resize(K); hcnt.resize(K);
    if (K > FIRST_READ) {
        ek_cuda_check(cudaMemcpyAsync(hcnt.data() + FIRST_READ, counts + FIRST_READ, (K - FIRST_READ) * 4, cudaMemcpyDeviceToHost, st));
        ek_cuda_check(cudaMemcpyAsync(hkey.data() + FIRST_READ, id_key + FIRST_READ, (size_t) (K - FIRST_READ) * 8, cudaMemcpyDeviceToHost, st));
        ek_cuda_check(cudaStreamSynchronize(st));
    }
    std::vector<uint32_t> by_rank(K);                  /* rank -> id */
    std::iota(by_rank.begin(), by_rank.end(), 0u);
    std::sort(by_rank.begin(), by_rank.end(), [&](uint32_t a, uint32_t b) { return hkey[a] < hkey[b]; });
    /* group table uploaded in one copy: [K list pointers][K group starts][K id -> rank] */
    std::vector<uint8_t> gt((size_t) K * 16);
    uint64_t *g_list = (uint64_t *) gt.data();
    uint32_t *g_start = (uint32_t *) (gt.data() + (size_t) K * 8), *g_rank = g_start + K;
    perm_h = (uint32_t **) malloc(sizeof(uint32_t *) * K);
    uint32_t start = 0;
    for (uint32_t r = 0; r < K; ++r) {
        const uint32_t id = by_rank[r], c = hcnt[id];
        uniq.push_back(hkey[id]); cnts.push_back(c);
        perm_h[r] = (uint32_t *) ek_malloc((size_t) c * 4);
        g_list[r] = (uint64_t) (uintptr_t) perm_h[r]; g_start[r] = start; g_rank[id] = r;
        start += c;
    }
    uint8_t *gt_d = (uint8_t *) ek_malloc(gt.size());
    ek_cuda_check(cudaMemcpyAsync(gt_d, gt.data(), gt.size(), cudaMemcpyHostToDevice, st));
    uint32_t *const *lists = (uint32_t *const *) gt_d;
    const uint32_t *group_start = (const uint32_t *) (gt_d + (size_t) K * 8), *id_rank = group_start + K;

    /* (3) radix passes over the rank */
    const uint32_t n_tiles = (uint32_t) ((n + RADIX_TILE - 1) / RADIX_TILE);
    const size_t n_hist = (size_t) RADIX_BINS * n_tiles;
    uint32_t *hist = (uint32_t *) ek_malloc(n_hist * 4 * 2), *hist_incl = hist + n_hist;
    const size_t hist_smem = RADIX_BINS * 4, scatter_smem = (PART_WARPS + 1) * RADIX_BINS * 4;
    if (K <= RADIX_BINS) {
        part_hist<true><<<n_tiles, PART_THREADS, hist_smem, st>>>(ids, nullptr, id_rank, n, 0, hist, n_tiles);
        ek_scan_incl_u32(hist, hist_incl, n_hist);
        part_scatter<true, true><<<n_tiles, PART_THREADS, scatter_smem, st>>>(ids, nullptr, id_rank, n, 0, hist_incl, n_tiles,
                                                                             nullptr, lists, group_start);
        ctx.stats.launches += 2;
    } else {
        uint64_t *pairs = (uint64_t *) ek_malloc(n * 8);
        part_hist<true><<<n_tiles, PART_THREADS, hist_smem, st>>>(ids, nullptr, id_rank, n, 0, hist, n_tiles);
        ek_scan_incl_u32(hist, hist_incl, n_hist);
        part_scatter<true, false><<<n_tiles, PART_THREADS, scatter_smem, st>>>(ids, nullptr, id_rank, n, 0, hist_incl, n_tiles,
                                                                              pairs, nullptr, nullptr);
        part_hist<false><<<n_tiles, PART_THREADS, hist_smem, st>>>(nullptr, pairs, nullptr, n, 8, hist, n_tiles);
        ek_scan_incl_u32(hist, hist_incl, n_hist);
        part_scatter<false, true><<<n_tiles, PART_THREADS, scatter_smem, st>>>(nullptr, pairs, nullptr, n, 8, hist_incl, n_tiles,
                                                                              nullptr, lists, group_start);
        ctx.stats.launches += 4;
        ek_free(pairs);
    }
    ek_cuda_check(cudaGetLastError());
    ek_free(hist); ek_free(gt_d);
    release();
    ctx.stats.partition_device++;
    return true;
}

} // namespace

extern "C" int ek_partition(size_t n, const void **ptrs, void ***unique_out, uint32_t **counts_out, uint32_t ***perm_out) {
    if (ek_init() != 0) return -1;
    EkContext &ctx = ek_ctx();
    if (n == 0 || n > 0xffffffffull) { ek_set_error("ek_partition(): unsupported size"); return -1; }
    const uint64_t *keys = reinterpret_cast<const uint64_t *>(ptrs);
    std::vector<uint64_t> uniq;
    std::vector<uint32_t> cnts;
    uint32_t **perm_h = nullptr;
    if (!partition_device(ctx, n, keys, uniq, cnts, perm_h))
        if (partition_host_sort(ctx, n, keys, uniq, cnts, perm_h) != 0) return -1;
    /* outputs with the reference's ownership: pinned-host unique / counts (counts[0] = number of groups,
       horiz.cu:83-121), malloc'd array of device permutation pointers */
    const size_t K = uniq.size();
    uint32_t *counts_h = (uint32_t *) ek_host_malloc(sizeof(uint32_t) * (K + 1));
    void **unique_h = (void **) ek_host_malloc(sizeof(void *) * std::max<size_t>(K, 1));
    counts_h[0] = (uint32_t) K;
    for (size_t k = 0; k < K; ++k) { counts_h[k + 1] = cnts[k]; unique_h[k] = (void *) (uintptr_t) uniq[k]; }
    *unique_out = unique_h; *counts_out = counts_h; *perm_out = perm_h;
    return 0;
}
#endif
