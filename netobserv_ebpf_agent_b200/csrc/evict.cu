// evict.cu — K2 flow_evict: lookup-and-delete every live flow of a table.
// Replaces FlowFetcher.LookupAndDeleteMap (reference pkg/tracer/tracer.go:1063-1157: iterate
// keys + one LookupAndDelete syscall per key) and the map hand-over of Accounter.evict
// (pkg/flow/account.go:67-68,86-87,102-124).
//
// An occupancy bitmap finds the live slots; 8 lanes per live flow: one coalesced 128-byte
// identity-line load, the 32-byte hot line by two of the lanes, shuffles to reassemble the
// 144-byte record (9 x 16-byte stores), one output-cursor atomic per 32 slots, and in-place
// clearing so the table comes out empty.
#include "kernels.cuh"
#include "kmap_body.cuh"

namespace fa {

// The 8 lanes of group g (lane j of the group) assemble the 144-byte record of `slot` from its identity line and hot
// line, and store it at O (9 x 16-byte stores) when `store`.  Every lane of the warp calls it (the hot-line words
// travel by shuffle); live = false for a group without a flow.  Shared by K2 and the fa_top_flows gather.
__device__ __forceinline__ void emit_record(const Table& t, uint64_t slot, bool live, bool store, uint4* O, int g, int j) {
    uint4 line = make_uint4(0, 0, 0, 0), hot = make_uint4(0, 0, 0, 0);
    if (live) line = ld_cg_u4(&t.ident[slot * 8 + j]);
    if (live && j < 2) hot = ld_cg_u4(&t.hot[slot * 2 + j]);
    // hot chunk 0 = (bytes, nstart), hot chunk 1 = (end, packets, flags)
    const uint32_t b_lo = __shfl_sync(0xFFFFFFFFu, hot.x, g * 8), b_hi = __shfl_sync(0xFFFFFFFFu, hot.y, g * 8);
    const uint32_t ns_lo = __shfl_sync(0xFFFFFFFFu, hot.z, g * 8), ns_hi = __shfl_sync(0xFFFFFFFFu, hot.w, g * 8);
    const uint32_t e_lo = __shfl_sync(0xFFFFFFFFu, hot.x, g * 8 + 1), e_hi = __shfl_sync(0xFFFFFFFFu, hot.y, g * 8 + 1);
    const uint32_t pk = __shfl_sync(0xFFFFFFFFu, hot.z, g * 8 + 1), fl = __shfl_sync(0xFFFFFFFFu, hot.w, g * 8 + 1);
    if (!store) return;
    const uint64_t start = 0ull - u64_of(ns_lo, ns_hi);       // nstart = -start; 0 stays 0
    if (j < 2) {
        O[j] = line;                                            // key[0..32)
    } else if (j == 2) {
        O[2] = make_uint4(line.x, line.y & 0x00FFFFFFu, (uint32_t)start, (uint32_t)(start >> 32));
    } else if (j == 3) {
        O[3] = make_uint4(e_lo, e_hi, b_lo, b_hi);              // end, bytes
        O[4] = make_uint4(pk, (line.y & 0xFFFFu) | (fl << 16), line.z, line.w);   // packets, eth|flags, desc[0..8)
    } else {
        O[j + 1] = line;                                        // desc[8..72)
    }
}

// kDrain = false: lookup-and-delete (the flow is removed).  kDrain = true: "lookup-and-reset": flows that
// received records since the last drain are emitted and their hot line is zeroed, but they stay in the table
// (identity line, tag, bitmap untouched) so the next batch hits them on the fast path.
template <bool kDrain>
__global__ void __launch_bounds__(256)
evict_kernel(Table t, uint4* __restrict__ out, uint32_t* __restrict__ slot_of_out, unsigned long long cap, Counters* ctr) {
    const int lane = threadIdx.x & 31, g = lane >> 3, j = lane & 7;
    const uint64_t slots = t.mask + 1;
    const uint64_t n_words = slots >> 5;               // slots is a power of two >= 1024
    const uint64_t warp_global = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    // The occupancy bitmap (1 bit per slot, set when a flow is created) lets a warp skip 1024 empty slots with one
    // coalesced load: eviction costs ~ (128 + 32 + 144) bytes per LIVE flow, not per slot.  One output-cursor
    // atomic per warp iteration (1024 slots).
    for (uint64_t w0 = warp_global * 32; w0 < n_words; w0 += n_warps * 32) {
        const uint64_t wi = w0 + lane;                  // lane l owns bitmap word w0 + l
        uint32_t mybits = wi < n_words ? t.occ[wi] : 0u;
        if (!kDrain && mybits) t.occ[wi] = 0u;
        uint32_t nonempty = __ballot_sync(0xFFFFFFFFu, mybits != 0u);
        if (nonempty == 0u) continue;
        if (kDrain) {
            // which of the live flows received records since the last drain?  Every lane walks the set bits of its
            // own bitmap word (32 independent chains of 32-byte hot-line reads in flight per warp).
            uint32_t rest = mybits, myact = 0;
            while (rest) {
                const int b = __ffs(rest) - 1; rest &= rest - 1;
                const uint64_t slot = wi * 32 + b;
                const uint4 h0 = ld_cg_u4(&t.hot[slot * 2]), h1 = ld_cg_u4(&t.hot[slot * 2 + 1]);
                if ((h0.x | h0.y | h0.z | h0.w | h1.x | h1.y | h1.z | h1.w) != 0u) myact |= 1u << b;
            }
            mybits = myact;
            nonempty = __ballot_sync(0xFFFFFFFFu, mybits != 0u);
            if (nonempty == 0u) continue;
        }
        // one reservation for everything this warp iteration emits; exclusive prefix over the lanes' word counts
        const uint32_t mycnt = __popc(mybits);
        uint32_t incl = mycnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += v; }
        const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(&ctr->evict_out, (unsigned long long)total);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        // rounds of 4 flows (one per 8-lane group), taken across all 32 words of the window
        for (uint32_t f0 = 0; f0 < total; f0 += 4) {
            {
                const uint32_t f = f0 + g;                              // this group's flow number in the window
                const bool live = f < total;
                // owner word = first lane whose inclusive prefix exceeds f (f differs per group: four ballots)
                uint32_t src = 0, within = 0;
                {
                    const uint32_t m0 = __ballot_sync(0xFFFFFFFFu, incl > f0), m1 = __ballot_sync(0xFFFFFFFFu, incl > f0 + 1),
                             m2 = __ballot_sync(0xFFFFFFFFu, incl > f0 + 2), m3 = __ballot_sync(0xFFFFFFFFu, incl > f0 + 3);
                    const uint32_t mm = g == 0 ? m0 : g == 1 ? m1 : g == 2 ? m2 : m3;
                    src = mm ? (uint32_t)(__ffs(mm) - 1) : 0u;
                }
                const uint32_t sbits = __shfl_sync(0xFFFFFFFFu, mybits, src);
                const uint32_t sincl = __shfl_sync(0xFFFFFFFFu, incl, src), scnt = __shfl_sync(0xFFFFFFFFu, mycnt, src);
                within = live ? f - (sincl - scnt) : 0u;                // rank of the flow inside its word
                const uint32_t pos = live ? __fns(sbits, 0, within + 1) : 0u;
                const uint64_t slot = (w0 + src) * 32 + pos;
                const unsigned long long idx = base + f;
                const bool store = live && idx < cap;
                emit_record(t, slot, live, store, out + idx * kRecChunks, g, j);
                if (store && slot_of_out && j == 0) slot_of_out[idx] = (uint32_t)slot;   // for the feature pass
                // delete: tag -> EMPTY, hot line -> identity  (drain: hot line only)
                if (!kDrain && live && j == 2) *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(&t.ident[slot * 8 + 2]) + 8) = make_uint2(0u, 0u);
                if (live && j < 2) t.hot[slot * 2 + j] = make_uint4(0, 0, 0, 0);
            }
        }
    }
}

// ---- what the live-table queries share --------------------------------------------------------------------------------
// The row fa_evict_ex would return for `slot` now: its bytes, packets (widened), flags, start and end from the hot line
// (ACCOUNTER) or the KERNEL_MAP metric line.  All five lie in the first 32-byte sector of that line, and the loads are
// plain ones: a caller that uses one word reads one.  patched: start / end patched by the slot's feature lines as the
// eviction patches them (feature_patch, kernels.cuh), before the other words are read.  Besides this reader, only the
// record assembly (emit_record, km_emit_record) and the slot moves of fa_expire_flows (slot_clear, slot_move) know
// these lines.
struct RowVals { uint64_t bytes, packets, start, end; uint32_t flags; };
__device__ __forceinline__ RowVals row_read(const Table& t, uint64_t slot, bool patched) {
    const uint8_t* M = t.met + slot * kMetLineBytes;
    const uint64_t* H = reinterpret_cast<const uint64_t*>(t.hot + slot * 2);   // bytes, nstart, end, packets | flags
    RowVals r;
    if (t.met) { r.start = km_ld64(M + KM_START); r.end = km_ld64(M + KM_END); }
    else { r.start = 0ull - H[1]; r.end = H[2]; }                              // nstart = 0 - start; 0 stays 0
    uint32_t eth = 0;                                                          // not part of RowVals: never read
    if (patched) feature_patch(t, slot, r.start, r.end, eth);
    if (t.met) { r.bytes = km_ld64(M + KM_BYTES); r.packets = km_ld32(M + KM_PACKETS); r.flags = km_ld16(M + KM_FLAGS); }
    else { r.bytes = H[0]; r.packets = (uint32_t)H[3]; r.flags = (uint32_t)(H[3] >> 32) & 0xFFFFu; }
    return r;
}

// Exclusive prefix of cnt over the warp and one cursor atomic for the warp's total: this lane's first index.  Every lane
// of the warp calls it.
__device__ __forceinline__ unsigned long long warp_reserve(uint32_t cnt, unsigned long long* cursor) {
    const int lane = threadIdx.x & 31;
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += v; }
    const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    unsigned long long base = 0;
    if (lane == 0 && total) base = atomicAdd(cursor, (unsigned long long)total);
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    return base + incl - cnt;
}

// Every thread owns one occupancy bitmap word per grid-stride step (a warp: 1024 slots in one coalesced load) and walks
// its set bits.  n_words and the stride are multiples of 32, so the lanes of a warp take the same number of steps.
#define FOR_OCC_WORDS(t, w) \
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < (((t).mask + 1) >> 5); w += (uint64_t)gridDim.x * blockDim.x)

// Blocks of 256 threads for a grid-stride loop over `threads` threads: no more than needed, at most 8 per SM.
static int grid_for(uint64_t threads, int sm_count) {
    const uint64_t blocks = (threads + 255) / 256, cap = (uint64_t)sm_count * 8;
    return (int)(blocks < cap ? blocks : cap);
}

// ---- fa_top_flows: the exact top-k of the live flows, without removing or changing anything ------------------------
// Rank order: metric descending, then slot hash ascending, then key bytes ascending.  A radix select over the 128-bit
// composite (metric, ~slot hash) in 8-bit digits, from the byte that holds the largest metric's top bit, finds the
// bucket of the k-th flow; it stops as soon as every flow above the bucket plus the bucket fit the scratch (or every
// bit is resolved).  Those flows are compacted, sorted by a bitonic network (key compare for equal hashes) and the
// first k gathered.  Passes read the bitmap and the metric word of the live flows; the key, for the hash, only where
// the metric bits are tied with the prefix.

FA_HD uint64_t shr64(uint64_t x, uint32_t s) { return s >= 64 ? 0ull : x >> s; }
FA_HD uint64_t bswap64(uint64_t x) {
    x = ((x & 0x00FF00FF00FF00FFull) << 8) | ((x >> 8) & 0x00FF00FF00FF00FFull);
    x = ((x & 0x0000FFFF0000FFFFull) << 16) | ((x >> 16) & 0x0000FFFF0000FFFFull);
    return (x << 32) | (x >> 32);
}
__device__ __forceinline__ uint64_t top_metric(const Table& t, uint64_t slot, bool by_bytes) {
    if (by_bytes) return row_read(t, slot, false).bytes;   // a branch, not a select: one load per flow
    return row_read(t, slot, false).packets;
}
FA_HD uint64_t top_hash(const Table& t, uint64_t slot) {
    const uint64_t* L = reinterpret_cast<const uint64_t*>(t.ident) + slot * (kIdentBytes / 8);
    return slot_hash(key_premix(L[0], L[1], L[2], L[3], L[4]));
}
// The composite's resolved bits [pos, 128) against the prefix: < 0 below, 0 equal, > 0 above.  ~hash goes to lo when it
// had to be computed (the metric bits are all resolved and equal).
FA_HD int top_cmp(const Table& t, uint64_t slot, uint64_t m, const TopState& S, uint64_t& lo, bool& have_lo) {
    if (S.pos >= 64) {
        const uint64_t a = shr64(m, S.pos - 64), b = shr64(S.pm, S.pos - 64);
        return a < b ? -1 : a > b ? 1 : 0;
    }
    if (m != S.pm) return m < S.pm ? -1 : 1;
    lo = ~top_hash(t, slot);
    have_lo = true;
    const uint64_t a = lo >> S.pos, b = S.plo >> S.pos;
    return a < b ? -1 : a > b ? 1 : 0;
}
// a ranks strictly before b; the padding (kTopNoSlot) after every flow
FA_HD bool top_before(const Table& t, const TopEnt& a, const TopEnt& b) {
    if (a.slot == kTopNoSlot || b.slot == kTopNoSlot) return a.slot != kTopNoSlot && b.slot == kTopNoSlot;
    if (a.m != b.m) return a.m > b.m;
    if (a.h != b.h) return a.h < b.h;
    const uint64_t* A = reinterpret_cast<const uint64_t*>(t.ident) + (uint64_t)a.slot * (kIdentBytes / 8);
    const uint64_t* B = reinterpret_cast<const uint64_t*>(t.ident) + (uint64_t)b.slot * (kIdentBytes / 8);
    for (int w = 0; w < 5; w++) {                          // identical premix: the 40 key bytes in memcmp order
        const uint64_t keep = w == 4 ? 0x00FFFFFFFFFFFFFFull : ~0ull;
        const uint64_t x = bswap64(A[w] & keep), y = bswap64(B[w] & keep);
        if (x != y) return x < y;
    }
    return false;
}

__global__ void __launch_bounds__(256) top_max_kernel(Table t, bool by_bytes, TopState* st) {
    unsigned long long mx = 0;
    FOR_OCC_WORDS(t, w) {
        for (uint32_t r = t.occ[w]; r; r &= r - 1) {
            const uint64_t m = top_metric(t, w * 32 + (__ffs(r) - 1), by_bytes);
            mx = m > mx ? m : mx;
        }
    }
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const unsigned long long o = __shfl_sync(0xFFFFFFFFu, mx, lane ^ d);
        mx = o > mx ? o : mx;
    }
    if (lane == 0 && mx) atomicMax(&st->m_max, mx);
}

// One thread.  hist == nullptr: the start (the digits above the largest metric are zero for every flow).  Otherwise fix
// the digit of the pass: the bucket that holds the k_rem-th candidate, counted from the top.
__global__ void top_resolve_kernel(TopState* st, const unsigned* hist, unsigned long long k, unsigned long long live,
                                   unsigned long long cap) {
    if (threadIdx.x != 0) return;
    TopState S = *st;
    if (!hist) {
        const uint32_t bits = 64u - (uint32_t)__clzll((long long)S.m_max);
        S.pos = 64u + 8u * ((bits + 7u) / 8u);
        S.k_rem = k; S.n_cand = live; S.above = 0;
        S.done = live <= cap ? 1u : 0u;
    } else {
        if (S.done) return;
        const uint32_t p = S.pos - 8u;
        unsigned long long cum = 0;
        uint32_t b = 255;
        for (; b > 0; b--) {
            if (cum + hist[b] >= S.k_rem) break;
            cum += hist[b];
        }
        S.above += cum; S.k_rem -= cum; S.n_cand = hist[b];
        if (p >= 64) S.pm |= (unsigned long long)b << (p - 64); else S.plo |= (unsigned long long)b << p;
        S.pos = p;
        S.passes++;
        if (S.above + S.n_cand <= cap) S.done = 1;
        else if (p == 0) { S.done = 1; S.overflow = 1; }
    }
    *st = S;
}

// Histogram of the next digit over the flows that match the prefix (256 bins in shared memory).
__global__ void __launch_bounds__(256) top_hist_kernel(Table t, bool by_bytes, const TopState* st, unsigned* hist) {
    FA_DYN_SMEM(smem);
    unsigned* H = reinterpret_cast<unsigned*>(smem);
    const TopState S = *st;
    if (S.done) return;
    for (int b = threadIdx.x; b < 256; b += blockDim.x) H[b] = 0u;
    __syncthreads();
    const uint32_t p = S.pos - 8u;
    FOR_OCC_WORDS(t, w) {
        for (uint32_t r = t.occ[w]; r; r &= r - 1) {
            const uint64_t slot = w * 32 + (__ffs(r) - 1);
            const uint64_t m = top_metric(t, slot, by_bytes);
            uint64_t lo = 0;
            bool have_lo = false;
            if (top_cmp(t, slot, m, S, lo, have_lo) != 0) continue;
            uint32_t d;
            if (p >= 64) {
                d = (uint32_t)(m >> (p - 64)) & 255u;
            } else {
                if (!have_lo) lo = ~top_hash(t, slot);
                d = (uint32_t)(lo >> p) & 255u;
            }
            atomicAdd(&H[d], 1u);
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < 256; b += blockDim.x)
        if (H[b]) atomicAdd(&hist[b], H[b]);
}

// Every flow at or above the prefix into ents (one cursor atomic per warp step); their count is above + n_cand.
__global__ void __launch_bounds__(256) top_compact_kernel(Table t, bool by_bytes, TopState* st, TopEnt* ents, unsigned long long cap) {
    const TopState S = *st;
    FOR_OCC_WORDS(t, w) {
        const uint32_t bits = t.occ[w];
        uint32_t take = 0;
        for (uint32_t r = bits; r; r &= r - 1) {
            const int b = __ffs(r) - 1;
            const uint64_t slot = w * 32 + b;
            uint64_t lo = 0;
            bool have_lo = false;
            if (top_cmp(t, slot, top_metric(t, slot, by_bytes), S, lo, have_lo) >= 0) take |= 1u << b;
        }
        unsigned long long at = warp_reserve(__popc(take), &st->count);
        for (uint32_t r = take; r; r &= r - 1, at++) {
            const uint64_t slot = w * 32 + (__ffs(r) - 1);
            if (at < cap) {
                TopEnt E;
                E.m = top_metric(t, slot, by_bytes); E.h = top_hash(t, slot); E.slot = (uint32_t)slot; E.pad = 0u;
                ents[at] = E;
            }
        }
    }
}

// Bitonic network over n (a power of two) entries, ascending in top_before order.  size == 0: sort each tile of
// kTopSortTile entries in shared memory (entries past the compaction count become padding).  Otherwise the strides
// below kTopSortTile of the merge of `size`.  kTopSortTile / 2 threads, one pair each per step.
__global__ void __launch_bounds__(kTopSortTile / 2) top_sort_tile_kernel(Table t, TopEnt* e, const TopState* st, unsigned long long n,
                                                                          unsigned long long size) {
    FA_DYN_SMEM(smem);
    TopEnt* S = reinterpret_cast<TopEnt*>(smem);
    const unsigned long long count = st->count;
    const uint32_t q = threadIdx.x;
    for (unsigned long long base = (unsigned long long)blockIdx.x * kTopSortTile; base < n; base += (unsigned long long)gridDim.x * kTopSortTile) {
        for (uint32_t i = q; i < (uint32_t)kTopSortTile; i += blockDim.x) {
            if (size == 0 && base + i >= count) { TopEnt E; E.m = 0; E.h = 0; E.slot = kTopNoSlot; E.pad = 0; S[i] = E; }
            else S[i] = e[base + i];
        }
        __syncthreads();
        const unsigned long long s_lo = size ? size : 2, s_hi = size ? size : kTopSortTile;
        for (unsigned long long s = s_lo; s <= s_hi; s <<= 1) {
            for (uint32_t j = (uint32_t)(s < (unsigned long long)kTopSortTile ? s : kTopSortTile) / 2; j > 0; j >>= 1) {
                const uint32_t i = 2 * j * (q / j) + (q % j), l = i + j;
                const bool up = ((base + i) & s) == 0;
                const TopEnt a = S[i], b = S[l];
                if (up ? top_before(t, b, a) : top_before(t, a, b)) { S[i] = b; S[l] = a; }
                __syncthreads();
            }
        }
        for (uint32_t i = q; i < (uint32_t)kTopSortTile; i += blockDim.x) e[base + i] = S[i];
        __syncthreads();
    }
}
// one step of the merge of `size` at stride j >= kTopSortTile, in global memory
__global__ void __launch_bounds__(256) top_merge_kernel(Table t, TopEnt* e, unsigned long long n, unsigned long long size,
                                                        unsigned long long j) {
    for (unsigned long long q = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; q < n / 2;
         q += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long i = 2 * j * (q / j) + (q % j), l = i + j;
        const bool up = (i & size) == 0;
        const TopEnt a = e[i], b = e[l];
        if (up ? top_before(t, b, a) : top_before(t, a, b)) { e[i] = b; e[l] = a; }
    }
}

// Row i of `out` from the flow at slots[i * stride]: the sorted fa_top_flows candidates (stride: one TopEnt), the
// fa_lookup_flows probe results or the fa_expire_flows list (stride 1).  kNoSlot: no flow; the row is written all zero when zero_miss (a lookup
// miss), else left unwritten (padding in the first n of top-k: fewer candidates than n, the host reports it).
// slot_of_out (optional, for the feature pass): the row's slot, 0 without a flow (read only by the peek).
// ACCOUNTER layout (emit_record, 4 flows per warp step) ...
__global__ void __launch_bounds__(256) gather_kernel(Table t, const uint32_t* __restrict__ slots, uint32_t stride, unsigned long long n,
                                                     bool zero_miss, uint4* __restrict__ out, uint32_t* __restrict__ slot_of_out) {
    const int lane = threadIdx.x & 31, g = lane >> 3, j = lane & 7;
    const unsigned long long warp_global = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5;
    const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long f0 = warp_global * 4; f0 < n; f0 += n_warps * 4) {
        const unsigned long long i = f0 + g;
        const uint32_t s = i < n ? slots[i * stride] : kNoSlot;
        const bool live = s != kNoSlot;
        const uint64_t slot = live ? s : 0u;
        emit_record(t, slot, live, live || (zero_miss && i < n), out + i * kRecChunks, g, j);   // live = false: zeros
        if (slot_of_out && i < n && j == 0) slot_of_out[i] = (uint32_t)slot;
    }
}
// ... and KERNEL_MAP layout (km_emit_record)
__global__ void __launch_bounds__(256) gather_kmap_kernel(Table t, const uint32_t* __restrict__ slots, uint32_t stride,
                                                          unsigned long long n, bool zero_miss, uint8_t* __restrict__ out,
                                                          uint32_t* __restrict__ slot_of_out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t slot = slots[i * stride];
        if (slot_of_out) slot_of_out[i] = slot == kNoSlot ? 0u : slot;
        if (slot != kNoSlot) {
            km_emit_record(t, t.met, slot, out + i * kRecBytes);
        } else if (zero_miss) {
            uint64_t* O = reinterpret_cast<uint64_t*>(out + i * kRecBytes);
            for (int k = 0; k < kRecBytes / 8; k++) O[k] = 0ull;
        }
    }
}

// One text for the device and the host emulation (FA_LAUNCH): both kernels loop grid-stride.
int launch_gather(const Table& t, bool kmap, const uint32_t* slots, uint32_t stride, uint64_t n, bool zero_miss,
                  uint8_t* out_recs, uint32_t* slot_of_out, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    if (kmap) FA_LAUNCH(gather_kmap_kernel, grid_for(n, sm_count), 256, 0, st, t, slots, stride, n, zero_miss, out_recs, slot_of_out);
    else FA_LAUNCH(gather_kernel, grid_for(n * 8, sm_count), 256, 0, st, t, slots, stride, n, zero_miss,
                   reinterpret_cast<uint4*>(out_recs), slot_of_out);
    return 1;
}

#ifndef FA_HOST_EMUL
int launch_evict(const Table& table, uint4* out_recs, uint32_t* slot_of_out,
                 unsigned long long cap, Counters* ctr, int sm_count, cudaStream_t st, bool drain) {
    if (drain) evict_kernel<true><<<sm_count * 8, 256, 0, st>>>(table, out_recs, slot_of_out, cap, ctr);
    else evict_kernel<false><<<sm_count * 8, 256, 0, st>>>(table, out_recs, slot_of_out, cap, ctr);
    return 1;
}
#endif  // FA_HOST_EMUL

// One text for the device and the host emulation (FA_LAUNCH): every kernel of the sequence loops grid-stride.
int launch_top_flows(const Table& t, bool kmap, bool by_bytes, uint64_t n, uint64_t live, const TopScratch& s,
                     uint8_t* out_recs, uint32_t* slot_of_out, int sm_count, cudaStream_t st) {
    const int grid = sm_count * 8;
    const size_t tile_smem = kTopSortTile * sizeof(TopEnt);
    int launches = 0;
    FA_LAUNCH(top_max_kernel, grid, 256, 0, st, t, by_bytes, s.state);
    FA_LAUNCH(top_resolve_kernel, 1, 32, 0, st, s.state, nullptr, n, live, s.cap);
    for (int p = 0; p < kTopPasses; p++) {                 // fixed sequence: passes after the last needed one exit at once
        FA_LAUNCH(top_hist_kernel, grid, 256, 256 * sizeof(unsigned), st, t, by_bytes, s.state, s.hist + p * 256);
        FA_LAUNCH(top_resolve_kernel, 1, 32, 0, st, s.state, s.hist + p * 256, n, live, s.cap);
    }
    FA_LAUNCH(top_compact_kernel, grid, 256, 0, st, t, by_bytes, s.state, s.ents, s.cap);
    launches += 3 + 2 * kTopPasses;
    const unsigned tiles = (unsigned)(s.cap / kTopSortTile);
    FA_LAUNCH(top_sort_tile_kernel, tiles, kTopSortTile / 2, tile_smem, st, t, s.ents, s.state, s.cap, 0ull);
    launches++;
    for (unsigned long long size = 2 * kTopSortTile; size <= s.cap; size <<= 1) {
        for (unsigned long long j = size / 2; j >= (unsigned long long)kTopSortTile; j >>= 1, launches++)
            FA_LAUNCH(top_merge_kernel, grid, 256, 0, st, t, s.ents, s.cap, size, j);
        FA_LAUNCH(top_sort_tile_kernel, tiles, kTopSortTile / 2, tile_smem, st, t, s.ents, s.state, s.cap, size);
        launches++;
    }
    const uint32_t* ent_slots = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(s.ents) + offsetof(TopEnt, slot));
    const uint32_t ent_stride = sizeof(TopEnt) / sizeof(uint32_t);
    return launches + launch_gather(t, kmap, ent_slots, ent_stride, n, false, out_recs, slot_of_out, sm_count, st);
}

// ---- fa_lookup_flows: exact point lookups of live flows by key, without removing or changing anything -------------
// One thread per key: table_find from the key's home slot, its slot (or kNoSlot) into slots[i] and found[i] (optional),
// one hit-count atomic per warp step.  Keys are 40-byte fa_flow_id rows, read as five 8-byte words.
__global__ void __launch_bounds__(256) lookup_probe_kernel(Table t, const uint64_t* __restrict__ keys, unsigned long long n,
                                                           uint32_t* __restrict__ slots, uint8_t* __restrict__ found,
                                                           unsigned long long* __restrict__ hits) {
    const int lane = threadIdx.x & 31;
    // warp-uniform steps (n is not a multiple of 32): every lane reaches the ballot
    for (unsigned long long i0 = blockIdx.x * (unsigned long long)blockDim.x + (threadIdx.x & ~31u); i0 < n;
         i0 += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long i = i0 + lane;
        uint32_t slot = kNoSlot;
        if (i < n) {
            const uint64_t* K = keys + i * (kKeyBytes / 8);
            const uint64_t w0 = K[0], w1 = K[1], w2 = K[2], w3 = K[3], w4 = K[4];
            const uint4 k0 = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
            const uint4 k1 = make_uint4((uint32_t)w2, (uint32_t)(w2 >> 32), (uint32_t)w3, (uint32_t)(w3 >> 32));
            const uint4 k2 = make_uint4((uint32_t)w4, (uint32_t)(w4 >> 32), 0u, 0u);
            slot = table_find(t, slot_hash(key_premix(w0, w1, w2, w3, w4)), k0, k1, k2);
            slots[i] = slot;
            if (found) found[i] = slot != kNoSlot ? 1 : 0;
        }
        const uint32_t hit = __ballot_sync(0xFFFFFFFFu, slot != kNoSlot);
        if (lane == 0 && hit) atomicAdd(hits, (unsigned long long)__popc(hit));
    }
}

// One text for the device and the host emulation (FA_LAUNCH): the probe, then the gather of the rows (zero for misses).
int launch_lookup_flows(const Table& t, bool kmap, const uint64_t* keys, uint64_t n, uint32_t* slots, uint8_t* found,
                        unsigned long long* hits, uint8_t* out_recs, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    FA_LAUNCH(lookup_probe_kernel, grid_for(n, sm_count), 256, 0, st, t, keys, n, slots, found, hits);
    return 1 + launch_gather(t, kmap, slots, 1u, n, true, out_recs, nullptr, sm_count, st);
}

// ---- fa_expire_flows: remove only the flows past an idle or active timeout, in place -------------------------------
// Mark (bitmap-driven, like top_hist_kernel): each live flow's row start / end, patched by its feature lines as the
// eviction patches them, against the two timeouts -> expire bitmap + slot list.  Emit: launch_gather
// over the list, then the clearing feature pass.  Delete: a cluster is a maximal cyclic run of occupied slots; its
// bounds were EMPTY before the call and stay EMPTY, so clusters are independent and one thread takes each cluster that
// holds an expiring flow: it clears the expiring slots, then vacates each survivor in cluster order and re-inserts it
// by linear probing from its home slot (never past its old position, so the walk never overwrites an entry it has not
// reached).  Every key stays reachable from its home slot without crossing an EMPTY slot: K1, K6, the KERNEL_MAP
// resolve and table_find find it as before.  A table without an EMPTY slot has no cluster bound: one thread runs
// backward-shift deletion over it.

__device__ __forceinline__ bool bit_at(const uint32_t* bm, uint64_t s) { return (bm[s >> 5] >> (s & 31)) & 1u; }
__device__ __forceinline__ bool expire_due(uint64_t now, uint64_t ts, uint64_t timeout) {
    return timeout != 0 && (int64_t)(now - ts) >= (int64_t)timeout;   // signed, as time.Duration: a zero ts is infinitely old
}
__global__ void __launch_bounds__(256) expire_mark_kernel(Table t, uint64_t now, uint64_t idle, uint64_t active, uint32_t* __restrict__ bm,
                                                          uint32_t* __restrict__ list, unsigned long long cap, ExpireCtr* c) {
    FOR_OCC_WORDS(t, w) {
        uint32_t bits = 0;
        for (uint32_t r = t.occ[w]; r; r &= r - 1) {
            const int b = __ffs(r) - 1;
            const RowVals v = row_read(t, w * 32 + b, true);
            if (expire_due(now, v.end, idle) || expire_due(now, v.start, active)) bits |= 1u << b;
        }
        bm[w] = bits;                                              // the thread owns the word: every word is written
        unsigned long long at = warp_reserve(__popc(bits), &c->n);
        for (uint32_t r = bits; r; r &= r - 1, at++)
            if (at < cap) list[at] = (uint32_t)(w * 32 + (__ffs(r) - 1));
    }
}

// The first slot of every cluster that holds an expiring flow (a set occupancy bit whose cyclic predecessor is clear)
// into starts.  Reads only: the delete pass changes the occupancy bits the cluster bounds are found from.
__global__ void __launch_bounds__(256) expire_clusters_kernel(Table t, const uint32_t* __restrict__ bm, uint32_t* __restrict__ starts,
                                                              ExpireCtr* c) {
    const uint64_t n_words = (t.mask + 1) >> 5;
    FOR_OCC_WORDS(t, w) {
        const uint32_t o = t.occ[w], prev = t.occ[(w + n_words - 1) & (n_words - 1)];   // wraps at the last slot
        uint32_t take = 0;
        for (uint32_t r = o & ~((o << 1) | (prev >> 31)); r; r &= r - 1) {
            const int b = __ffs(r) - 1;
            for (uint64_t p = w * 32 + b; bit_at(t.occ, p); p = (p + 1) & t.mask)
                if (bit_at(bm, p)) { take |= 1u << b; break; }
        }
        unsigned long long at = warp_reserve(__popc(take), &c->clusters);
        for (uint32_t r = take; r; r &= r - 1, at++) starts[at] = (uint32_t)(w * 32 + (__ffs(r) - 1));
    }
}

// Everything a slot owns: the identity line (key, tag, start mirror), the hot or metric line, the feature lines, the
// occupancy bit (atomic: neighbouring clusters share bitmap words).  A vacated slot ends all zero, so that a flow created
// there later inherits nothing.
__device__ __forceinline__ uint64_t slot_tag(const Table& t, uint64_t s) { return reinterpret_cast<const uint64_t*>(t.ident + s * 8)[5]; }
__device__ __forceinline__ uint64_t slot_home(const Table& t, uint64_t s) { return top_hash(t, s) & t.mask; }
__device__ __forceinline__ void move_line(uint4* base, int chunks, uint64_t from, uint64_t to) {
    for (int k = 0; k < chunks; k++) { base[to * chunks + k] = base[from * chunks + k]; base[from * chunks + k] = make_uint4(0, 0, 0, 0); }
}
__device__ __forceinline__ void zero_line(uint4* base, int chunks, uint64_t s) {
    for (int k = 0; k < chunks; k++) base[s * chunks + k] = make_uint4(0, 0, 0, 0);
}
__device__ __forceinline__ void slot_clear(const Table& t, uint64_t s) {
    zero_line(t.ident, 8, s);
    if (t.met) zero_line(reinterpret_cast<uint4*>(t.met), kMetLineBytes / 16, s); else zero_line(t.hot, 2, s);
    if (t.feat_add) zero_line(t.feat_add, kAddState, s);
    if (t.feat_dns) zero_line(t.feat_dns, kDnsState, s);
    if (t.feat_drop) zero_line(t.feat_drop, kDropState, s);
    atomicAnd(&t.occ[s >> 5], ~(1u << (s & 31)));
}
__device__ __forceinline__ void slot_move(const Table& t, uint64_t from, uint64_t to) {
    move_line(t.ident, 8, from, to);
    if (t.met) move_line(reinterpret_cast<uint4*>(t.met), kMetLineBytes / 16, from, to); else move_line(t.hot, 2, from, to);
    if (t.feat_add) move_line(t.feat_add, kAddState, from, to);
    if (t.feat_dns) move_line(t.feat_dns, kDnsState, from, to);
    if (t.feat_drop) move_line(t.feat_drop, kDropState, from, to);
    atomicOr(&t.occ[to >> 5], 1u << (to & 31));
    atomicAnd(&t.occ[from >> 5], ~(1u << (from & 31)));
}

// One thread per listed cluster.  The cluster's length is read before anything in it changes; within it only this
// thread writes, and the EMPTY slot after it is never written (a survivor's target lies between its home and itself).
__global__ void __launch_bounds__(256) expire_compact_kernel(Table t, const uint32_t* __restrict__ bm, const uint32_t* __restrict__ starts,
                                                             const ExpireCtr* c) {
    const unsigned long long n = c->clusters;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint64_t s = starts[i];
        uint64_t len = 0;
        while (bit_at(t.occ, (s + len) & t.mask)) len++;
        for (uint64_t k = 0; k < len; k++) {
            const uint64_t p = (s + k) & t.mask;
            if (bit_at(bm, p)) slot_clear(t, p);
        }
        for (uint64_t k = 0; k < len; k++) {                      // survivors in cluster order
            const uint64_t p = (s + k) & t.mask;
            if (bit_at(bm, p)) continue;
            uint64_t q = slot_home(t, p);
            while (q != p && slot_tag(t, q) != 0) q = (q + 1) & t.mask;
            if (q != p) slot_move(t, p, q);
        }
    }
}

// A table without an EMPTY slot (FA_F_NO_FULL_CUT with spills): sequential backward-shift deletion on one thread.  An
// entry at j moves into the hole when its home is not cyclically in (hole, j]; its expire bit moves with it.  Entries
// move only towards the hole, so no expiring entry lands before the slot being scanned.
__global__ void expire_full_kernel(Table t, uint32_t* bm) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const uint64_t n_words = (t.mask + 1) >> 5;
    for (uint64_t w = 0; w < n_words; w++) {
        while (bm[w]) {
            const uint64_t i = w * 32 + (__ffs((int)bm[w]) - 1);
            slot_clear(t, i);
            bm[w] &= ~(1u << (i & 31));
            uint64_t hole = i;
            for (uint64_t j = (i + 1) & t.mask; slot_tag(t, j) != 0; j = (j + 1) & t.mask) {
                if (((j - slot_home(t, j)) & t.mask) < ((j - hole) & t.mask)) continue;
                slot_move(t, j, hole);
                if (bit_at(bm, j)) { bm[j >> 5] &= ~(1u << (j & 31)); bm[hole >> 5] |= 1u << (hole & 31); }
                hole = j;
            }
        }
    }
}

__global__ void expire_live_kernel(Counters* ctr, unsigned long long n) {
    if (blockIdx.x == 0 && threadIdx.x == 0) ctr->live -= n;
}

// One text for the device and the host emulation (FA_LAUNCH): every kernel loops grid-stride or runs one thread.
int launch_expire_mark(const Table& t, uint64_t now, uint64_t idle, uint64_t active, const ExpireScratch& s, int sm_count,
                       cudaStream_t st) {
    FA_LAUNCH(expire_mark_kernel, sm_count * 8, 256, 0, st, t, now, idle, active, s.bm, s.list, s.cap, s.ctr);
    return 1;
}

int launch_expire_delete(const Table& t, const ExpireScratch& s, uint64_t n, bool full, Counters* ctr, int sm_count,
                         cudaStream_t st) {
    if (!n) return 0;
    if (full) {
        FA_LAUNCH(expire_full_kernel, 1, 32, 0, st, t, s.bm);
    } else {
        FA_LAUNCH(expire_clusters_kernel, sm_count * 8, 256, 0, st, t, s.bm, s.list, s.ctr);
        FA_LAUNCH(expire_compact_kernel, sm_count * 8, 256, 0, st, t, s.bm, s.list, s.ctr);
    }
    FA_LAUNCH(expire_live_kernel, 1, 32, 0, st, ctr, (unsigned long long)n);
    return full ? 2 : 3;
}

// ---- fa_group_flows: exact roll-ups of the live flows by a key mask, without removing or changing anything --------
// Scan (bitmap-driven, like expire_mark_kernel): each live flow's masked key and its row values (row_read with the
// eviction's feature patch).  The lanes of a warp take one flow each per round; the lanes with an equal masked
// key (every one of its ten 32-bit words: distinct keys can share a premix) form a peer set, and one leader per set
// folds the set's sum into the group table.  Emit / clear: one thread per listed group writes its row and zeroes its slot.
//
// Group-table slot (12 u64): [0, 5) the group key, [5] state (0 EMPTY, kGroupWriting, kGroupPublished), [6] flows,
// [7] bytes, [8] packets, [9] nstart = 0 - start (max: the smallest non-zero start, 0 if none), [10] end (max),
// [11] flags (or).  Every accumulator is commutative with identity 0, so the result does not depend on the order of
// the updates, and a slot that was never claimed or was emitted is all zero.
constexpr unsigned long long kGroupWriting = 1ull, kGroupPublished = 2ull;

struct GroupVals { uint64_t bytes, packets, nstart, end; uint32_t flags; };

__device__ __forceinline__ void group_add(unsigned long long* G, uint64_t flows, const GroupVals& v) {
    red_add_u64(G + 6, flows);
    if (v.bytes) red_add_u64(G + 7, v.bytes);
    if (v.packets) red_add_u64(G + 8, v.packets);
    if (v.nstart) red_max_u64(G + 9, v.nstart);
    if (v.end) red_max_u64(G + 10, v.end);
    if (v.flags) red_or_u64(G + 11, v.flags);
}

// Fold `flows` flows with the summed values v into the group of key k, creating it the way K1 creates a flow: claim an
// EMPTY slot by CAS on its state, write the key, fence, publish; a walk that meets a slot being written waits for the
// publish.  Linear probing from the key's slot hash, at most every slot once.  false: no slot found (the table always
// has more slots than the live flows, so this does not happen).
__device__ __forceinline__ bool group_fold(const GroupScratch& s, const uint64_t k[5], uint64_t flows, const GroupVals& v) {
    uint64_t slot = slot_hash(key_premix(k[0], k[1], k[2], k[3], k[4])) & s.mask;
    for (uint64_t probes = 0; probes <= s.mask; probes++, slot = (slot + 1) & s.mask) {
        unsigned long long* G = s.tab + slot * kGroupSlotWords;
        unsigned long long state = ld_cg_u64(G + 5);
        if (state == 0ull) {
            state = atomicCAS(G + 5, 0ull, kGroupWriting);
            if (state == 0ull) {
#pragma unroll
                for (int w = 0; w < 5; w++) G[w] = k[w];
                __threadfence();
                atomicCAS(G + 5, kGroupWriting, kGroupPublished);
                s.list[atomicAdd(&s.ctr->n, 1ull)] = (uint32_t)slot;     // one group per slot: the list cannot overflow
                group_add(G, flows, v);
                return true;
            }
        }
        // a volatile load: the compiler may not assume the state stays the same and drop the wait
        while (state == kGroupWriting) state = *reinterpret_cast<volatile unsigned long long*>(G + 5);
        __threadfence();
        unsigned long long diff = 0;
#pragma unroll
        for (int w = 0; w < 5; w++) diff |= ld_cg_u64(G + w) ^ k[w];
        if (diff == 0) {
            group_add(G, flows, v);
            return true;
        }
    }
    return false;
}

// The peer set of this lane's key k: the lanes that have a key (have) and whose key equals it in every one of its ten
// 32-bit words (distinct keys can share a premix).  Returns the set's lane mask (0 without a key); the set's leader (its
// lowest lane) ends with v folded over the set.  Every lane of the warp calls it, converged.
__device__ __forceinline__ uint32_t peer_reduce(const uint64_t k[5], bool have, GroupVals& v) {
    const int lane = threadIdx.x & 31;
    const uint32_t active = __ballot_sync(0xFFFFFFFFu, have);
    uint32_t peers = active;
#pragma unroll
    for (int i = 0; i < 5; i++) {
        peers &= __match_any_sync(0xFFFFFFFFu, (uint32_t)k[i]);
        peers &= __match_any_sync(0xFFFFFFFFu, (uint32_t)(k[i] >> 32));
    }
    if (!have) peers = 0u;
    const int np = __popc(peers);
    if (__any_sync(0xFFFFFFFFu, np > 1)) {
        if (__all_sync(0xFFFFFFFFu, !have || peers == active)) {
            // one peer set holds every key of the round (a coarse mask): a butterfly over the warp
            for (int d = 16; d > 0; d >>= 1) {
                const uint64_t b = __shfl_sync(0xFFFFFFFFu, v.bytes, lane ^ d), p = __shfl_sync(0xFFFFFFFFu, v.packets, lane ^ d);
                const uint64_t ns = __shfl_sync(0xFFFFFFFFu, v.nstart, lane ^ d), e = __shfl_sync(0xFFFFFFFFu, v.end, lane ^ d);
                const uint32_t f = __shfl_sync(0xFFFFFFFFu, v.flags, lane ^ d);
                v.bytes += b; v.packets += p; v.nstart = ns > v.nstart ? ns : v.nstart; v.end = e > v.end ? e : v.end; v.flags |= f;
            }
        } else {
            // several sets: step q, every lane reads the q-th lane of its own set (the leader is lane 0 of it)
            GroupVals a = v;
            const int most = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)np);
            for (int q = 1; q < most; q++) {
                const int src = q < np ? (int)__fns(peers, 0, q + 1) : lane;
                const uint64_t b = __shfl_sync(0xFFFFFFFFu, v.bytes, src), p = __shfl_sync(0xFFFFFFFFu, v.packets, src);
                const uint64_t ns = __shfl_sync(0xFFFFFFFFu, v.nstart, src), e = __shfl_sync(0xFFFFFFFFu, v.end, src);
                const uint32_t f = __shfl_sync(0xFFFFFFFFu, v.flags, src);
                if (q < np) { a.bytes += b; a.packets += p; a.nstart = ns > a.nstart ? ns : a.nstart; a.end = e > a.end ? e : a.end; a.flags |= f; }
            }
            v = a;
        }
    }
    return peers;
}

__global__ void __launch_bounds__(256) group_scan_kernel(Table t, GroupMask m, GroupScratch s) {
    const int lane = threadIdx.x & 31;
    FOR_OCC_WORDS(t, w) {
        uint32_t r = t.occ[w];
        while (__any_sync(0xFFFFFFFFu, r != 0u)) {             // converged rounds: at most one flow per lane
            const bool have = r != 0u;
            uint64_t k[5] = {0, 0, 0, 0, 0};
            GroupVals v = {0, 0, 0, 0, 0u};                       // lanes without a flow hold the identity
            if (have) {
                const uint64_t slot = w * 32 + (__ffs(r) - 1);
                r &= r - 1;
                const uint64_t* L = reinterpret_cast<const uint64_t*>(t.ident) + slot * (kIdentBytes / 8);
#pragma unroll
                for (int i = 0; i < 5; i++) k[i] = L[i] & m.w[i];
                const RowVals r = row_read(t, slot, true);
                v = GroupVals{r.bytes, r.packets, 0ull - r.start, r.end, r.flags};
            }
            const uint32_t peers = peer_reduce(k, have, v);
            const int np = __popc(peers);
            if (have && lane == __ffs(peers) - 1 && !group_fold(s, k, (uint64_t)np, v)) atomicAdd(&s.ctr->lost, 1ull);
        }
    }
}

// Row i from the i-th listed group (out != nullptr), then its slot back to all zero.
__global__ void __launch_bounds__(256) group_emit_kernel(GroupScratch s, unsigned long long n, uint64_t* __restrict__ out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long* G = s.tab + (uint64_t)s.list[i] * kGroupSlotWords;
        if (out) {
            uint64_t* O = out + i * (kGroupRowBytes / 8);
            for (int w = 0; w < 5; w++) O[w] = G[w];
            O[5] = G[6]; O[6] = G[7]; O[7] = G[8];              // flows, bytes, packets
            O[8] = 0ull - G[9]; O[9] = G[10];                   // start (0 stays 0), end
            O[10] = G[11] & 0xFFFFull;                          // flags, pad_ = 0
        }
        for (int w = 0; w < kGroupSlotWords; w++) G[w] = 0ull;
    }
}

// One text for the device and the host emulation (FA_LAUNCH): both kernels loop grid-stride.
int launch_group_scan(const Table& t, const GroupMask& m, const GroupScratch& s, int sm_count, cudaStream_t st) {
    FA_LAUNCH(group_scan_kernel, sm_count * 8, 256, 0, st, t, m, s);
    return 1;
}

int launch_group_emit(const GroupScratch& s, uint64_t n, uint64_t* out, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    FA_LAUNCH(group_emit_kernel, grid_for(n, sm_count), 256, 0, st, s, (unsigned long long)n, out);
    return 1;
}

// ---- fa_histogram_flows: per-group histograms of one per-flow value, without removing or changing anything ----------
// Runs on the group table that launch_group_scan built (groups and flow counts).  Index: row_of[slot of group i] = i.
// Scan (bitmap-driven, like group_scan_kernel): each live flow with the value finds its group by a read-only walk (it
// exists: the group scan created it), picks its bucket and lands in row row_of[group].  The lanes of a warp take one
// flow each per round; the lanes with equal (row, bucket) form a peer set and one leader per set folds the set into the
// row.  Emit: one thread per row copies key and flows from the group slot and turns ~min into min.
//
// Row (u64 words, device `out` or staging, zeroed before the scan): [0, 5) key, [5] flows, [6] count (add), [7] sum (add),
// [8] ~min (max), [9] max (max), [10 + b] bucket b (add).  Every accumulator has identity 0, so the rows do not depend on
// the order of the updates.
constexpr uint64_t kHistNoGroup = ~0ull;

// The value of the row fa_evict_ex would return for `slot` now; false when that row has none (the decoder's presence
// rules: duration needs a start, RTT a non-zero flow_rtt, DNS latency a DNS block with a non-zero id).
__device__ __forceinline__ bool hist_value(const Table& t, uint64_t slot, uint32_t which, uint64_t& v) {
    if (which == kHistBytes || which == kHistPackets) {
        const RowVals r = row_read(t, slot, false);
        v = which == kHistBytes ? r.bytes : r.packets;
        return true;
    }
    if (which == kHistDuration) {
        const RowVals r = row_read(t, slot, true);
        v = r.end >= r.start ? r.end - r.start : 0ull;
        return r.start != 0;
    }
    if (which == kHistRtt) {
        const uint64_t* S = reinterpret_cast<const uint64_t*>(t.feat_add + slot * kAddState);
        v = S[0] ? S[1] : 0ull;                                      // additional.flow_rtt: the max of the samples
        return v != 0;
    }
    const uint64_t* S = reinterpret_cast<const uint64_t*>(t.feat_dns + slot * kDnsState);
    v = S[1];                                                        // dns.latency: the max; dns.id: last non-zero id
    return S[0] != 0 && (S[2] & 0xFFFFull) != 0;
}

// The group-table slot of masked key k: linear probing from its slot hash up to the first EMPTY slot, every slot at
// most once.  Nothing is written.
__device__ __forceinline__ uint64_t hist_group(const GroupScratch& s, const uint64_t k[5]) {
    uint64_t slot = slot_hash(key_premix(k[0], k[1], k[2], k[3], k[4])) & s.mask;
    for (uint64_t probes = 0; probes <= s.mask; probes++, slot = (slot + 1) & s.mask) {
        const unsigned long long* G = s.tab + slot * kGroupSlotWords;
        if (G[5] == 0ull) break;
        unsigned long long diff = 0;
#pragma unroll
        for (int w = 0; w < 5; w++) diff |= G[w] ^ k[w];
        if (diff == 0) return slot;
    }
    return kHistNoGroup;
}

__global__ void __launch_bounds__(256) hist_index_kernel(GroupScratch s, unsigned long long n, uint32_t* __restrict__ row_of) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        row_of[s.list[i]] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) hist_scan_kernel(Table t, GroupMask m, GroupScratch s, const uint32_t* __restrict__ row_of,
                                                        HistParams h, unsigned long long* __restrict__ rows) {
    FA_DYN_SMEM(smem);
    unsigned long long* bounds = reinterpret_cast<unsigned long long*>(smem);       // the search reads shared memory
    for (uint32_t i = threadIdx.x; i < h.n_bounds; i += blockDim.x) bounds[i] = h.bounds[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint64_t row_words = kHistHeadWords + h.n_bounds + 1;
    FOR_OCC_WORDS(t, w) {
        uint32_t r = t.occ[w];
        while (__any_sync(0xFFFFFFFFu, r != 0u)) {             // converged rounds: at most one flow per lane
            bool have = false;
            uint32_t row = 0, b = 0;
            uint64_t v = 0;
            if (r != 0u) {
                const uint64_t slot = w * 32 + (__ffs(r) - 1);
                r &= r - 1;
                if (hist_value(t, slot, h.value, v)) {
                    const uint64_t* L = reinterpret_cast<const uint64_t*>(t.ident) + slot * (kIdentBytes / 8);
                    uint64_t k[5];
#pragma unroll
                    for (int i = 0; i < 5; i++) k[i] = L[i] & m.w[i];
                    const uint64_t g = hist_group(s, k);
                    if (g == kHistNoGroup) {
                        atomicAdd(&s.ctr->lost, 1ull);
                    } else {
                        have = true;
                        row = row_of[g];
                        // the number of bounds below v: bucket b holds bounds[b-1] < v <= bounds[b] (b = n_bounds: +Inf)
#pragma unroll
                        for (uint32_t step = 32; step > 0; step >>= 1)
                            if (b + step <= h.n_bounds && bounds[b + step - 1] < v) b += step;
                    }
                }
            }
            uint32_t peers = __ballot_sync(0xFFFFFFFFu, have) & __match_any_sync(0xFFFFFFFFu, row) & __match_any_sync(0xFFFFFFFFu, b);
            if (!have) peers = 0u;
            const int np = __popc(peers);
            // step q: every lane reads the q-th lane of its own set (the leader is lane 0 of it)
            uint64_t sum = v, mx = v, nmin = ~v;
            const int most = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)np);
            for (int q = 1; q < most; q++) {
                const int src = q < np ? (int)__fns(peers, 0, q + 1) : lane;
                const uint64_t x = __shfl_sync(0xFFFFFFFFu, v, src);
                if (q < np) { sum += x; mx = x > mx ? x : mx; nmin = ~x > nmin ? ~x : nmin; }
            }
            if (have && lane == __ffs(peers) - 1) {
                unsigned long long* R = rows + (uint64_t)row * row_words;
                red_add_u64(R + 6, (unsigned long long)np);
                if (sum) red_add_u64(R + 7, sum);
                if (nmin) red_max_u64(R + 8, nmin);
                if (mx) red_max_u64(R + 9, mx);
                red_add_u64(R + kHistHeadWords + b, (unsigned long long)np);
            }
        }
    }
}

__global__ void __launch_bounds__(256) hist_emit_kernel(GroupScratch s, unsigned long long n, uint32_t n_bounds, unsigned long long* __restrict__ rows) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long* G = s.tab + (uint64_t)s.list[i] * kGroupSlotWords;
        unsigned long long* R = rows + i * (kHistHeadWords + n_bounds + 1);
        for (int w = 0; w < 5; w++) R[w] = G[w];
        R[5] = G[6];                                            // flows
        R[8] = R[6] ? ~R[8] : 0ull;                             // min: 0 when no flow of the group has the value
    }
}

int launch_hist_index(const GroupScratch& s, uint64_t n, uint32_t* row_of, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    FA_LAUNCH(hist_index_kernel, grid_for(n, sm_count), 256, 0, st, s, (unsigned long long)n, row_of);
    return 1;
}

int launch_hist_scan(const Table& t, const GroupMask& m, const GroupScratch& s, const uint32_t* row_of, const HistParams& h,
                     uint64_t* rows, int sm_count, cudaStream_t st) {
    FA_LAUNCH(hist_scan_kernel, sm_count * 8, 256, kHistMaxBounds * 8, st, t, m, s, row_of, h,
              reinterpret_cast<unsigned long long*>(rows));
    return 1;
}

int launch_hist_emit(const GroupScratch& s, uint64_t n, uint32_t n_bounds, uint64_t* rows, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    FA_LAUNCH(hist_emit_kernel, grid_for(n, sm_count), 256, 0, st, s, (unsigned long long)n, n_bounds,
              reinterpret_cast<unsigned long long*>(rows));
    return 1;
}

// ---- fa_distinct_flows: per-group distinct counts of a second key mask, without removing or changing anything --------
// Level 1 is launch_group_scan with U = G | D: its groups are the distinct (key & G, key & D) pairs, since both are
// functions of key & U and key & U is their OR.  Level 2 takes the n1 listed level-1 groups, one per lane per round,
// masks each key with G ((key & U) & G == key & G), forms peer sets as group_scan_kernel does and folds each set into
// the second group table: the summed level-1 flow counts into flows (word 6), the set's size into word 7, which in the
// second table holds the distinct count.  Every accumulator adds, so the result does not depend on the order.
__global__ void __launch_bounds__(256) distinct_fold_kernel(GroupScratch s1, unsigned long long n1, GroupMask m, GroupScratch s2) {
    const int lane = threadIdx.x & 31;
    // warp-uniform steps (n1 is not a multiple of 32): every lane reaches the matches
    for (unsigned long long i0 = blockIdx.x * (unsigned long long)blockDim.x + (threadIdx.x & ~31u); i0 < n1;
         i0 += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long i = i0 + lane;
        const bool have = i < n1;
        uint64_t k[5] = {0, 0, 0, 0, 0};
        GroupVals v = {0, 0, 0, 0, 0u};                           // bytes carries the level-1 flow count
        if (have) {
            const unsigned long long* G = s1.tab + (uint64_t)s1.list[i] * kGroupSlotWords;
#pragma unroll
            for (int w = 0; w < 5; w++) k[w] = G[w] & m.w[w];
            v.bytes = G[6];
        }
        const uint32_t peers = peer_reduce(k, have, v);
        const int np = __popc(peers);
        if (have && lane == __ffs(peers) - 1 && !group_fold(s2, k, v.bytes, GroupVals{(uint64_t)np, 0, 0, 0, 0u}))
            atomicAdd(&s2.ctr->lost, 1ull);
    }
}

// The slots of the level-2 groups with distinct >= min_distinct into sel, counted in *n_sel (zeroed before).  The group
// count is read on the device; bound (>= it) sizes the grid.
__global__ void __launch_bounds__(256) distinct_select_kernel(GroupScratch s2, unsigned long long min_distinct, uint32_t* __restrict__ sel,
                                                              unsigned long long* n_sel) {
    const unsigned long long n = s2.ctr->n;
    const int lane = threadIdx.x & 31;
    for (unsigned long long i0 = blockIdx.x * (unsigned long long)blockDim.x + (threadIdx.x & ~31u); i0 < n;
         i0 += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long i = i0 + lane;
        uint32_t slot = 0;
        bool take = false;
        if (i < n) {
            slot = s2.list[i];
            take = s2.tab[(uint64_t)slot * kGroupSlotWords + 7] >= min_distinct;
        }
        const unsigned long long at = warp_reserve(take ? 1u : 0u, n_sel);
        if (take) sel[at] = slot;
    }
}

// Row i (fa_distinct_group: key, flows, distinct) from the level-2 group at slot sel[i].  The table is left as it is
// (launch_group_emit with out == nullptr clears it).
__global__ void __launch_bounds__(256) distinct_emit_kernel(GroupScratch s2, const uint32_t* __restrict__ sel, unsigned long long n,
                                                            uint64_t* __restrict__ out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long* G = s2.tab + (uint64_t)sel[i] * kGroupSlotWords;
        uint64_t* O = out + i * (kDistinctRowBytes / 8);
        for (int w = 0; w < 5; w++) O[w] = G[w];
        O[5] = G[6]; O[6] = G[7];                               // flows, distinct
    }
}

// One text for the device and the host emulation (FA_LAUNCH): every kernel loops grid-stride.
int launch_distinct_fold(const GroupScratch& s1, uint64_t n1, const GroupMask& m, const GroupScratch& s2, int sm_count, cudaStream_t st) {
    if (!n1) return 0;
    FA_LAUNCH(distinct_fold_kernel, grid_for(n1, sm_count), 256, 0, st, s1, (unsigned long long)n1, m, s2);
    return 1;
}

int launch_distinct_select(const GroupScratch& s2, uint64_t bound, uint64_t min_distinct, uint32_t* sel, unsigned long long* n_sel,
                           int sm_count, cudaStream_t st) {
    if (!bound) return 0;
    FA_LAUNCH(distinct_select_kernel, grid_for(bound, sm_count), 256, 0, st, s2, (unsigned long long)min_distinct, sel, n_sel);
    return 1;
}

int launch_distinct_emit(const GroupScratch& s2, const uint32_t* sel, uint64_t n, uint64_t* out, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    FA_LAUNCH(distinct_emit_kernel, grid_for(n, sm_count), 256, 0, st, s2, sel, (unsigned long long)n, out);
    return 1;
}

}  // namespace fa
