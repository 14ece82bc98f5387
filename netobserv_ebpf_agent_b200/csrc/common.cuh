// common.cuh — record/table layouts, hash spec and PTX helpers shared by all kernels.
//
// Record ABI: 144-byte flow_record = 9 x 16-byte chunks (reference bpf/types.h:94-126,
// 191-215; SURVEY.md §8a).  Everything on this path is integer / byte work.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#ifndef FA_HD
#define FA_HD __host__ __device__ __forceinline__
#endif

namespace fa {

// ------------------------------------------------------------------ record layout
constexpr int kRecBytes   = 144;
constexpr int kRecChunks  = 9;      // 16-byte chunks per record
constexpr int kKeyBytes   = 40;
constexpr int kDnsRecBytes = 104;   // flow_id + dns_metrics
constexpr int kAddRecBytes = 72;    // flow_id + additional_metrics
constexpr int kDropRecBytes = 72;   // flow_id + pkt_drop_metrics

// byte offsets inside the 144-byte record
constexpr int R_START = 40, R_END = 48, R_BYTES = 56, R_PACKETS = 64, R_ETH = 68, R_FLAGS = 70, R_DESC = 72;

// ------------------------------------------------------------------ table layout
// One slot = one 128-byte "identity line" + one 32-byte "hot line".
//
// identity line (read-mostly; written once when the flow is created):
//   [  0.. 40) key (byte 39 forced to 0)
//   [ 40.. 48) tag   u64: 0 = EMPTY, else (epoch << 24) | (tcp flags already OR-ed into the hot line << 8) | bits
//   [ 48.. 52) start mirror, low 32 bits   } m48 = (0 - start_at_insert) >> 16: an immutable lower bound of
//   [ 52.. 54) eth_protocol                } hot.nstart, so records that cannot lower the start skip that RED
//   [ 54.. 56) start mirror, high 16 bits  }
//   [ 56..128) descriptor = record bytes [72..144) with padding zeroed
// so that line chunk j (16 B) lines up with record chunk {0,1,2,4,5,6,7,8}[j].
//
// hot line (updated with fire-and-forget reductions; all-zero == identity):
//   [ 0.. 8) bytes   (add)
//   [ 8..16) nstart  = 0 - start_mono_time_ts (max)  -> min over non-zero starts, 0 if none
//   [16..24) end     (max)
//   [24..28) packets (add, wraps mod 2^32 like the Go u32)
//   [28..32) flags   (or; low 16 bits)
constexpr int kIdentBytes = 128;
constexpr int kHotBytes   = 32;

constexpr uint64_t TAG_STATE_MASK = 0x3ull;
constexpr uint64_t TAG_CLAIMED    = 0x1ull;
constexpr uint64_t TAG_PUBLISHED  = 0x2ull;
constexpr uint64_t TAG_DIRTY      = 0x4ull;   // order-dependent fields must be re-folded in stream order
constexpr uint64_t TAG_HAS_BASE   = 0x8ull;   // at least one base flow record was folded (vs feature-only entry)
constexpr int      TAG_FLAGS_SHIFT = 8;    // 16 bits: flag bits known to be set in hot.flags already
constexpr int      TAG_EPOCH_SHIFT = 24;   // 40-bit launch counter

struct Table {
    uint4*   ident;      // slots x 8 uint4
    uint4*   hot;        // slots x 2 uint4 (ACCOUNTER mode), or nullptr
    uint8_t* met;        // slots x 128 B flow_metrics lines (KERNEL_MAP mode, kmap_body.cuh), or nullptr
    uint4*   feat_add;  // slots x 5 uint4 (80 B) or nullptr: additional_metrics fold state
    uint4*   feat_dns;   // slots x 8 uint4 (128 B) or nullptr: dns_metrics fold state
    uint4*   feat_drop;  // slots x 6 uint4 (96 B) or nullptr: pkt_drop_metrics fold state
    uint32_t* occ;       // occupancy bitmap, 1 bit per slot: eviction visits live flows only
    uint64_t mask;       // slots - 1 (slots is a power of two)
};

// Device-side counters (one struct per engine, zeroed at create / evict as noted).
struct Counters {
    unsigned long long live;          // live flows in the active table (reset at evict)
    unsigned long long spills;        // records that could not be placed (table physically full)
    unsigned long long dirty;         // flows flagged for ordered re-fold in the current launch (reset per launch)
    unsigned long long fixups_total;  // running total of ordered re-folds
    unsigned long long evict_out;     // output cursor of the evict kernel
    unsigned long long scratch[3];
    unsigned long long launch_n;      // record count of a launch whose size is only known on the device (opt bit 4)
    // ACCOUNTER: the host's ring of live-flow counts (mapped pinned memory, kLiveRing entries; nullptr in KERNEL_MAP
    // mode).  The last CTA of K1 number `live_seq` writes `live` into entry live_seq % kLiveRing, so the host reads
    // each launch's count without a copy after it.
    unsigned long long* live_ring;
    unsigned long long live_seq;      // K1 launches that have written the ring
};
constexpr int kLiveRing = 8;

// ------------------------------------------------------------------ hash spec (DESIGN.md §hash)
FA_HD uint64_t fmix64(uint64_t x) {
    x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
    return x;
}
// 5 little-endian words of the 40-byte key; byte 39 (padding) masked out.
FA_HD uint64_t key_premix(uint64_t w0, uint64_t w1, uint64_t w2, uint64_t w3, uint64_t w4) {
    const uint64_t P1 = 0x9E3779B97F4A7C15ull, P2 = 0xC2B2AE3D27D4EB4Full;
    w4 &= 0x00FFFFFFFFFFFFFFull;
    uint64_t h = 0x243F6A8885A308D3ull;
    h = (h ^ w0) * P1; h ^= h >> 32;
    h = (h ^ w1) * P2; h ^= h >> 29;
    h = (h ^ w2) * P1; h ^= h >> 32;
    h = (h ^ w3) * P2; h ^= h >> 29;
    h = (h ^ w4) * P1; h ^= h >> 32;
    return h;
}
FA_HD uint64_t slot_hash(uint64_t premix)  { return fmix64(premix); }
FA_HD uint64_t owner_hash(uint64_t premix) { return fmix64(premix ^ 0xA0761D6478BD642Full); }
FA_HD uint64_t cms_hash_a(uint64_t premix, uint64_t seed) { return fmix64(premix ^ 0xE7037ED1A0B428DBull ^ seed); }
FA_HD uint64_t cms_hash_b(uint64_t premix, uint64_t seed) { return fmix64(premix ^ 0x8EBC6AF09C88C6E3ull ^ seed) | 1ull; }
FA_HD uint64_t hll_hash(uint64_t premix, uint64_t seed)   { return fmix64(premix ^ 0x589965CC75374CC3ull ^ seed); }
FA_HD uint32_t cms_index(uint64_t a, uint64_t b, uint32_t row, uint32_t log2w) {
    return (uint32_t)(((a + (uint64_t)row * b) * 0x9E3779B97F4A7C15ull) >> (64 - log2w));
}

// ------------------------------------------------------------------ chunk masks
// Which bits of line chunk j (as 4 LE u32 words) take part in the identity compare /
// are stored on insert.  j: 0,1 key | 2 key tail (+tag, excluded) | 3 eth + desc[0..8) |
// 4..7 desc[8..72).  Padding bytes (key byte 39, metrics bytes 66-67 and 100-103) are
// excluded: binary.Read leaves them zero (reference pkg/model/record.go:227-231).
FA_HD uint4 chunk_mask(int j) {
    switch (j) {
        case 2:  return make_uint4(0xFFFFFFFFu, 0x00FFFFFFu, 0u, 0u);
        case 3:  return make_uint4(0u, 0x0000FFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
        case 5:  return make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0x0000FFFFu, 0xFFFFFFFFu);
        case 7:  return make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u);
        default: return make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
    }
}
// record chunk index that line chunk j is compared with
FA_HD int rec_chunk_of_line_chunk(int j) { return j < 3 ? j : j + 1; }

FA_HD uint4 and4(uint4 a, uint4 m) { return make_uint4(a.x & m.x, a.y & m.y, a.z & m.z, a.w & m.w); }
FA_HD bool  eq4_masked(uint4 a, uint4 b, uint4 m) {
    return (((a.x ^ b.x) & m.x) | ((a.y ^ b.y) & m.y) | ((a.z ^ b.z) & m.z) | ((a.w ^ b.w) & m.w)) == 0u;
}

// OR of the masked differences of two chunks: 0 iff equal (for OR-accumulated, branch-free compares)
FA_HD uint32_t diff4_masked(uint4 a, uint4 b, uint4 m) {
    return ((a.x ^ b.x) & m.x) | ((a.y ^ b.y) & m.y) | ((a.z ^ b.z) & m.z) | ((a.w ^ b.w) & m.w);
}

// dynamic shared memory of a kernel; the host emulation of the tests (tests/emul/simt.h) hands out a per-CTA buffer
#ifdef FA_HOST_EMUL
#define FA_DYN_SMEM(name) uint8_t* name = simt::ctx().cta->smem
#define FA_EMUL_COUNT(which, n) simt::count(which, n)      // path counters of the emulation (nothing on the device)
#else
#define FA_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#define FA_EMUL_COUNT(which, n) ((void)0)
#endif

// A kernel launch written once for the device and the host emulation of the tests.  The emulation runs every CUDA
// thread as an OS thread, so it caps the grid at 2 CTAs: only kernels whose loops are grid-stride may be launched this
// way.  Dynamic shared memory is handed out per CTA (FA_DYN_SMEM).
#ifdef FA_HOST_EMUL
#define FA_LAUNCH(kernel, grid, block, smem, st, ...) \
    simt::launch((unsigned)(grid) < 2u ? (unsigned)(grid) : 2u, (block), (smem), [=] { kernel(__VA_ARGS__); })
#else
#define FA_LAUNCH(kernel, grid, block, smem, st, ...) kernel<<<(grid), (block), (smem), (st)>>>(__VA_ARGS__)
#endif

#ifdef __CUDACC__
// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// named barrier over `count` threads of the CTA (SASS: BAR.SYNC id, count)
__device__ __forceinline__ void named_barrier_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Same copy with an L2 evict-first policy: the record stream is read once, the table lines it would push out of L2 are
// read again and again (SASS: UBLKCP with a cache-hint operand).
__device__ __forceinline__ void tma_load_1d_stream(void* smem_dst, const void* gmem_src, uint32_t bytes, unsigned long long* bar) {
    unsigned long long policy;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}

// Ask L2 to fetch a byte range (SASS: UBLKPF); used to run the HBM read of the next tiles ahead of
// the shared-memory staging of the current one.
__device__ __forceinline__ void tma_prefetch_l2(const void* gmem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// L2-coherent 128-bit load (bypasses L1: table lines are written by other SMs in the same launch).
__device__ __forceinline__ uint4 ld_cg_u4(const uint4* p) { return __ldcg(p); }
__device__ __forceinline__ unsigned long long ld_cg_u64(const unsigned long long* p) { return __ldcg(p); }
__device__ __forceinline__ void st_cg_u4(uint4* p, uint4 v) { __stcg(p, v); }
// streaming (evict-first) 128-bit load for the record stream
__device__ __forceinline__ uint4 ld_stream_u4(const uint4* p) { return __ldcs(p); }

// fire-and-forget reductions (SASS: RED.E.*)
__device__ __forceinline__ void red_add_u64(void* p, unsigned long long v) { asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_max_u64(void* p, unsigned long long v) { asm volatile("red.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_min_u64(void* p, unsigned long long v) { asm volatile("red.global.min.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_add_u32(void* p, uint32_t v) { asm volatile("red.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_or_u64(void* p, unsigned long long v) { asm volatile("red.global.or.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void red_or_u32(void* p, uint32_t v) { asm volatile("red.global.or.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_max_u32(void* p, uint32_t v) { asm volatile("red.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_min_u32(void* p, uint32_t v) { asm volatile("red.global.min.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

__device__ __forceinline__ uint64_t u64_of(uint32_t lo, uint32_t hi) { return (uint64_t)lo | ((uint64_t)hi << 32); }

// A kernel launched with programmatic stream serialization may start while the kernel before it on the stream is still
// draining; it calls this before its first access to global memory that kernel may write, and waits there until that
// kernel has completed and its writes are visible.  A no-op for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#else
inline void pdl_wait() {}                     // host emulation of the tests: kernels run one after the other
#endif  // __CUDACC__

// ------------------------------------------------------------------ read-only table probe
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;   // a key without a live flow
#if defined(__CUDACC__) || defined(FA_HOST_EMUL)
// The slot of the key whose first three 16-byte chunks are k0, k1, k2 (slot hash h; the tag half of k2 and key byte 39
// are ignored), or kNoSlot.  Linear probing from the home slot, one round trip per slot for the three line chunks that
// hold the key and the tag (the tag shares a chunk with the key tail).  An EMPTY tag ends the walk (a miss), an equal
// key is a hit; feature-only entries (published without TAG_HAS_BASE) are live flows and are found.  The walk visits
// each slot at most once, so it also ends on a physically full table (FA_F_NO_FULL_CUT).  For a table no launch is
// writing: the "full" cut pre-pass and fa_lookup_flows.
__device__ __forceinline__ uint32_t table_find(const Table& t, uint64_t h, uint4 k0, uint4 k1, uint4 k2) {
    uint64_t slot = h & t.mask;
    for (uint64_t probes = 0; probes <= t.mask; probes++) {
        const uint4* L = &t.ident[slot * 8];
        const uint4 l0 = ld_cg_u4(L), l1 = ld_cg_u4(L + 1), l2 = ld_cg_u4(L + 2);
        if ((l2.z & TAG_STATE_MASK) == 0) break;
        if (eq4_masked(l0, k0, chunk_mask(0)) && eq4_masked(l1, k1, chunk_mask(1)) && eq4_masked(l2, k2, chunk_mask(2)))
            return (uint32_t)slot;
        slot = (slot + 1) & t.mask;
    }
    return kNoSlot;
}
#endif

}  // namespace fa
