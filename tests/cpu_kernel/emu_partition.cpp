/*
 * emu_partition.cpp -- runs the kernels of enoki_b200/csrc/ek_partition.cu ON THE CPU (cuda_shim.h): every CUDA thread
 * of a CTA becomes a POSIX thread, CTAs run one after the other.  TEST INFRASTRUCTURE (tests/test_cpu_partition.py,
 * which plays the host side of ek_partition around these launches); races between CTAs are left to the GPU tests.
 *
 * The emulator's runtime (CTA barrier, warp rendezvous, trap) is the one emu_fast.cpp defines: that file is compiled
 * into this library as well rather than copied.  The shim's additions the partition kernels need follow it.
 */
#include "emu_fast.cpp"
#include <functional>

inline uint32_t atomicCAS(uint32_t *p, uint32_t cmp, uint32_t v) {
    __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return cmp;
}
inline unsigned long long atomicCAS(unsigned long long *p, unsigned long long cmp, unsigned long long v) {
    __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return cmp;
}
inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_exchange(mask, 0); emu::warp_release(mask); }

#include "../../enoki_b200/csrc/ek_partition.cu"

namespace {
struct PartThreadArg { const std::function<void()> *body; unsigned tid; };
void *part_thread_main(void *p) {
    const PartThreadArg *a = (const PartThreadArg *) p;
    emu::tid_.x = a->tid;
    (*a->body)();
    return nullptr;
}

int launch(unsigned grid, size_t smem_bytes, const std::function<void()> &body) {
    const unsigned T = PART_THREADS;
    emu::gdim_.x = grid; emu::bdim_.x = T;
    void *raw = nullptr;
    if (posix_memalign(&raw, 1024, smem_bytes + 1024) != 0) return -3;
    emu::smem_ = (uint8_t *) raw;
    pthread_barrier_init(&emu::cta_bar_, nullptr, T);
    std::vector<pthread_t> th(T);
    std::vector<PartThreadArg> ta(T);
    pthread_attr_t attr; pthread_attr_init(&attr); pthread_attr_setstacksize(&attr, 256 * 1024);
    for (unsigned b = 0; b < grid; ++b) {
        emu::bid_.x = b;
        memset(emu::smem_, 0xCD, smem_bytes + 1024);       /* shared memory starts out as garbage on the device, too */
        for (unsigned t = 0; t < T; ++t) { ta[t] = { &body, t }; pthread_create(&th[t], &attr, part_thread_main, &ta[t]); }
        for (unsigned t = 0; t < T; ++t) pthread_join(th[t], nullptr);
    }
    pthread_attr_destroy(&attr);
    pthread_barrier_destroy(&emu::cta_bar_);
    free(raw);
    emu::smem_ = nullptr;
    return 0;
}
} // namespace

extern "C" {

/* constants the host side needs: {threads, max groups, table slots, count bins, radix tile} */
void emu_part_constants(uint32_t *out) {
    out[0] = PART_THREADS; out[1] = PART_MAX_GROUPS; out[2] = PART_SLOTS; out[3] = PART_COUNT_BINS; out[4] = RADIX_TILE;
}

/* hdr = {n_ids, overflow, top_claimed, pad}; table = PART_SLOTS keys (all ~0), slot_id = PART_SLOTS + 1 words */
int emu_part_insert(const uint64_t *keys, uint64_t n, uint32_t grid, uint32_t *ids, uint64_t *table, uint32_t *slot_id,
                    uint64_t *id_key, uint32_t *hdr, uint32_t *counts) {
    PartHeader *h = reinterpret_cast<PartHeader *>(hdr);
    int rc = launch(grid, 0, [&] { part_insert(keys, n, ids, table, slot_id, id_key, h); });
    if (rc == 0) rc = launch(grid, PART_COUNT_BINS * 4, [&] { part_count(ids, n, slot_id, h, counts); });
    return rc;
}

/* one radix pass: histogram into hist, then (after the caller's inclusive scan into hist_incl) the scatter */
int emu_part_hist(int first, const uint32_t *ids, const uint64_t *pairs, const uint32_t *id_rank, uint64_t n,
                  uint32_t shift, uint32_t *hist, uint32_t n_tiles) {
    if (first) return launch(n_tiles, RADIX_BINS * 4, [&] { part_hist<true>(ids, pairs, id_rank, n, shift, hist, n_tiles); });
    return launch(n_tiles, RADIX_BINS * 4, [&] { part_hist<false>(ids, pairs, id_rank, n, shift, hist, n_tiles); });
}

int emu_part_scatter(int first, int last, const uint32_t *ids, const uint64_t *pairs_in, const uint32_t *id_rank, uint64_t n,
                     uint32_t shift, const uint32_t *hist_incl, uint32_t n_tiles, uint64_t *pairs_out,
                     uint32_t *const *lists, const uint32_t *group_start) {
    const size_t smem = (PART_WARPS + 1) * RADIX_BINS * 4;
    if (first && last)
        return launch(n_tiles, smem, [&] { part_scatter<true, true>(ids, pairs_in, id_rank, n, shift, hist_incl, n_tiles, pairs_out, lists, group_start); });
    if (first)
        return launch(n_tiles, smem, [&] { part_scatter<true, false>(ids, pairs_in, id_rank, n, shift, hist_incl, n_tiles, pairs_out, lists, group_start); });
    if (last)
        return launch(n_tiles, smem, [&] { part_scatter<false, true>(ids, pairs_in, id_rank, n, shift, hist_incl, n_tiles, pairs_out, lists, group_start); });
    return -1;
}

} /* extern "C" */
