// features.cu — K6: per-flow folds of the feature streams the reference keeps in per-CPU BPF maps.
//
//   additional_metrics (RTT / IPsec): bpf/rtt_tracker.h:12-22,73-91 + AccumulateAdditional
//                                     (pkg/model/flow_content.go:154-177)
//   dns_metrics:                      bpf/flows.c:145-158,291-330 + AccumulateDNS (flow_content.go:76-96)
//   pkt_drop_metrics:                 bpf/pkt_drops.h:10-23,80-98 + AccumulateDrops (flow_content.go:98-117)
//   base effects of both:             buildBaseFromAdditional (flow_content.go:63-74)
//   merged view at eviction:          LookupAndDeleteMap (pkg/tracer/tracer.go:1098-1151,1159-1187)
//
// Contract (SURVEY.md §8 a12'): every sample is folded as if it were one per-CPU slot, in stream
// order.  Order-independent parts use plain atomics (rtt / latency = max, flags = or, start = min
// non-zero, end = max; IPsec: max return code, "encrypted" = or over the samples holding that max).
// Order-dependent parts are made exact with a 64-bit running sample number packed into the atomic:
//   first sample of a flow (its block is adopted whole)   -> max of ~seq, then a second pass copies it
//   dns id = last non-zero, errno = last                   -> max of (seq+1)<<16 | value
//   eth_protocol handed to an empty base = first non-zero  -> max of ~(seq<<16 | eth)
// A flow seen only through a feature stream gets a table entry without TAG_HAS_BASE
// (tracer.go:1179-1182: an all-zero base); K1 adopts the first base record whole when it arrives.
#include "kernels.cuh"

namespace fa {

// ---- per-slot state, all-zero == empty ------------------------------------------------------
// additional: 5 x uint4 (80 B)
//   [ 0] nfirst = max ~seq            [ 8] rtt max
//   [16] ipsec  = max (ret ^ 0x80000000) << 1 | enc          [24] nfs = max(0 - start)   (base effect)
//   [32] fe = max end (base effect)   [40] neth = max ~(seq << 16 | eth)  over eth != 0  (base effect)
//   [48] first.start                  [56] first.end
//   [64] first.eth (u16) ...
// dns: 8 x uint4 (128 B)
//   [ 0] nfirst                       [ 8] latency max
//   [16] id_last  = max (seq+1) << 16 | id   over id != 0     [24] errno_last = max (seq+1) << 16 | errno
//   [32] nfs                          [40] fe
//   [48] neth                         [56] flags (or, u32) | first.eth (u16 @60)
//   [64] first.start                  [72] first.end          [80..112) first.name[32]   [112..128) spare
// packet drops: 6 x uint4 (96 B)
//   [ 0] nfirst                       [ 8] bytes sum (add; saturates to u16 at eviction == addUint16 chained)
//   [16] packets sum                  [24] cause_seq = max (seq+1) over latest_drop_cause != 0 (the second pass stores the cause)
//   [32] state_last = max (seq+1) << 8 | latest_state  over latest_state != 0
//   [40] flags (or, u32) | first.eth (u16 @44)           [48] nfs        [56] fe        [64] neth
//   [72] first.start                  [80] first.end                     [88] latest_drop_cause (u32)
// additional, extension (no reference analogue): [72] nrtt_min = max ~rtt over rtt != 0 -> smallest non-zero RTT
// (kAddState / kDnsState / kDropState, the uint4 per slot, are in kernels.cuh: fa_expire_flows moves these lines)

__device__ __forceinline__ uint64_t ld_u64_unaligned8(const uint8_t* p) { return *reinterpret_cast<const uint64_t*>(p); }

#ifndef FA_K6_MINBLOCKS
#define FA_K6_MINBLOCKS 4   // 64 registers: four CTAs per SM (5 -> 48 registers with spills: -3 %, 6: -10 %)
#endif

// Find the flow's slot, creating a feature-only entry when the key is new.  One thread per representative sample.
// The three key chunks and the tag travel in ONE round trip (the tag shares a 16-byte chunk with the key tail).
// Only a slot published during THIS launch (its tag carries the launch epoch) can have been read before its key was
// visible: then, and only then, fence and read the line again.  Entries of earlier launches are complete.
__device__ uint32_t find_or_create(const Table& t, uint64_t epoch, const uint64_t k[5], unsigned long long* n_created) {
    const uint64_t kk4 = k[4] & 0x00FFFFFFFFFFFFFFull;
    const uint64_t h = slot_hash(key_premix(k[0], k[1], k[2], k[3], k[4]));
    uint64_t slot = h & t.mask;
    bool ordered = false;
    for (uint32_t probes = 0; probes < 65536; ) {
        const uint4* L4 = &t.ident[slot * 8];
        const uint4 c0 = ld_cg_u4(L4), c1 = ld_cg_u4(L4 + 1), c2 = ld_cg_u4(L4 + 2);
        const unsigned long long tag = u64_of(c2.z, c2.w);
        const uint32_t state = (uint32_t)(tag & TAG_STATE_MASK);
        unsigned long long* L = reinterpret_cast<unsigned long long*>(&t.ident[slot * 8]);
        unsigned long long* tagp = L + 5;
        if (state == 0) {
            if (atomicCAS(tagp, 0ull, TAG_CLAIMED) == 0ull) {
                L[0] = k[0]; L[1] = k[1]; L[2] = k[2]; L[3] = k[3]; L[4] = kk4;
#pragma unroll
                for (int c = 6; c < 16; c++) L[c] = 0ull;
                __threadfence();
                *reinterpret_cast<volatile unsigned long long*>(tagp) = (epoch << TAG_EPOCH_SHIFT) | TAG_PUBLISHED;   // no TAG_HAS_BASE
                red_or_u32(&t.occ[slot >> 5], 1u << (slot & 31));
                atomicAdd(n_created, 1ull);
                return (uint32_t)slot;
            }
            continue;                                   // lost the race: look at the slot again
        }
        if (state == (uint32_t)TAG_CLAIMED) continue;   // being published by someone else
        if ((tag >> TAG_EPOCH_SHIFT) == epoch && !ordered) { __threadfence(); ordered = true; continue; }
        const bool same = (u64_of(c0.x, c0.y) == k[0]) & (u64_of(c0.z, c0.w) == k[1]) & (u64_of(c1.x, c1.y) == k[2]) &
                          (u64_of(c1.z, c1.w) == k[3]) & ((u64_of(c2.x, c2.y) & 0x00FFFFFFFFFFFFFFull) == kk4);
        if (same) return (uint32_t)slot;
        slot = (slot + 1) & t.mask;
        probes++;
        ordered = false;
    }
    return 0xFFFFFFFFu;
}

__device__ __forceinline__ void load_key(const uint8_t* rec, uint64_t k[5]) {
#pragma unroll
    for (int i = 0; i < 5; i++) k[i] = ld_u64_unaligned8(rec + 8 * i);    // records are 8-byte aligned (72 / 104 B)
}

// ---- the fold: one CTA per tile of 256 samples ------------------------------------------------------------------
// The tile is staged in shared memory with coalesced 8-byte loads (samples are 72 / 104 bytes: a thread-per-sample
// read would touch 18-26 lines per warp instruction).  Samples of one flow elect a representative inside the tile
// (shared-memory hash set on the slot hash, keys compared in shared memory); the others fold their values into the
// representative's accumulators with shared-memory atomics, so a hot flow costs ONE table probe and ONE set of global
// reductions per tile instead of one per sample (every value below is a max / add / or, and the order-dependent ones
// carry the sample number, so folding early does not change the result).
constexpr int kFeatTile = 256;          // samples per tile == threads per CTA
constexpr int kFeatRep = 512;           // tile-local election set
constexpr uint32_t kFeatNone = 0xFFFFFFFFu;

// 64-bit shared-memory max / or are compare-and-swap loops: look first, most samples of a hot flow cannot change the value
__device__ __forceinline__ void smem_max_u64(uint64_t* p, uint64_t v) { if (v > *reinterpret_cast<volatile uint64_t*>(p)) atomicMax(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v); }
__device__ __forceinline__ void smem_add_u64(uint64_t* p, uint64_t v) { if (v) atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v); }
__device__ __forceinline__ void smem_or_u64(uint64_t* p, uint64_t v) { if (v & ~*reinterpret_cast<volatile uint64_t*>(p)) atomicOr(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v); }
__device__ __forceinline__ void gmax(uint8_t* p, uint64_t v) { if (v) red_max_u64(p, v); }
__device__ __forceinline__ void gadd(uint8_t* p, uint64_t v) { if (v) red_add_u64(p, v); }
__device__ __forceinline__ void gor32(uint8_t* p, uint64_t v) { if (v) red_or_u32(p, (uint32_t)v); }

struct AddFeat {                        // additional_metrics samples, 72 B
    static constexpr int kRec = kAddRecBytes, kAcc = 7, kCand2 = -1;
    static __device__ __forceinline__ uint8_t* state(const Table& t, uint32_t slot) { return reinterpret_cast<uint8_t*>(t.feat_add) + (size_t)slot * (kAddState * 16); }
    static __device__ __forceinline__ void extract(const uint8_t* R, uint64_t seq, uint64_t* v) {
        const uint64_t start = ld_u64_unaligned8(R + 40), end = ld_u64_unaligned8(R + 48), rtt = ld_u64_unaligned8(R + 56);
        const uint32_t ret = *reinterpret_cast<const uint32_t*>(R + 64);
        const uint32_t w = *reinterpret_cast<const uint32_t*>(R + 68);         // eth u16 | enc u8 | pad
        const uint32_t eth = w & 0xFFFFu, enc = ((w >> 16) & 0xFFu) ? 1u : 0u;
        v[0] = ~seq;
        v[1] = rtt;
        v[2] = rtt ? ~rtt : 0ull;
        v[3] = ((uint64_t)(ret ^ 0x80000000u) << 1) | enc | (1ull << 40);       // bit 40: "has a sample"
        v[4] = start ? 0ull - start : 0ull;
        v[5] = end;
        v[6] = eth ? ~((seq << 16) | eth) : 0ull;
    }
    static __device__ __forceinline__ void fold(uint64_t* a, int st, const uint64_t* v) {
#pragma unroll
        for (int k = 0; k < kAcc; k++) smem_max_u64(a + k * st, v[k]);
    }
    static __device__ __forceinline__ void flush(uint8_t* S, const uint64_t* a, int st) {
        gmax(S + 0, a[0 * st]); gmax(S + 8, a[1 * st]); gmax(S + 72, a[2 * st]); gmax(S + 16, a[3 * st]); gmax(S + 24, a[4 * st]); gmax(S + 32, a[5 * st]); gmax(S + 40, a[6 * st]);
    }
};
struct DnsFeat {                        // dns_metrics samples, 104 B
    static constexpr int kRec = kDnsRecBytes, kAcc = 8, kCand2 = -1;
    static __device__ __forceinline__ uint8_t* state(const Table& t, uint32_t slot) { return reinterpret_cast<uint8_t*>(t.feat_dns) + (size_t)slot * (kDnsState * 16); }
    static __device__ __forceinline__ void extract(const uint8_t* R, uint64_t seq, uint64_t* v) {
        const uint64_t start = ld_u64_unaligned8(R + 40), end = ld_u64_unaligned8(R + 48), lat = ld_u64_unaligned8(R + 56);
        const uint32_t w0 = *reinterpret_cast<const uint32_t*>(R + 64);        // id u16 | flags u16
        const uint32_t w1 = *reinterpret_cast<const uint32_t*>(R + 68);        // eth u16 | errno u8 | name[0]
        const uint32_t id = w0 & 0xFFFFu, flags = w0 >> 16, eth = w1 & 0xFFFFu, err = (w1 >> 16) & 0xFFu;
        v[0] = ~seq;
        v[1] = lat;
        v[2] = id ? ((seq + 1) << 16) | id : 0ull;
        v[3] = ((seq + 1) << 16) | err;
        v[4] = start ? 0ull - start : 0ull;
        v[5] = end;
        v[6] = eth ? ~((seq << 16) | eth) : 0ull;
        v[7] = flags;
    }
    static __device__ __forceinline__ void fold(uint64_t* a, int st, const uint64_t* v) {
#pragma unroll
        for (int k = 0; k < 7; k++) smem_max_u64(a + k * st, v[k]);
        smem_or_u64(a + 7 * st, v[7]);
    }
    static __device__ __forceinline__ void flush(uint8_t* S, const uint64_t* a, int st) {
        gmax(S + 0, a[0 * st]); gmax(S + 8, a[1 * st]); gmax(S + 16, a[2 * st]); gmax(S + 24, a[3 * st]); gmax(S + 32, a[4 * st]); gmax(S + 40, a[5 * st]); gmax(S + 48, a[6 * st]);
        gor32(S + 56, a[7 * st]);
    }
};
// pkt_drop_metrics samples (flow_id 40 B + start 8, end 8, bytes u16, packets u16, latest_drop_cause u32, latest_flags u16,
// eth_protocol u16, latest_state u8), 72 B: AccumulateDrops in sample order
struct DropFeat {
    static constexpr int kRec = kDropRecBytes, kAcc = 9, kCand2 = 3;     // accumulator 3 names the last sample with a drop cause
    static __device__ __forceinline__ uint8_t* state(const Table& t, uint32_t slot) { return reinterpret_cast<uint8_t*>(t.feat_drop) + (size_t)slot * (kDropState * 16); }
    static __device__ __forceinline__ void extract(const uint8_t* R, uint64_t seq, uint64_t* v) {
        const uint64_t start = ld_u64_unaligned8(R + 40), end = ld_u64_unaligned8(R + 48);
        const uint32_t w0 = *reinterpret_cast<const uint32_t*>(R + 56);        // bytes u16 | packets u16
        const uint32_t cause = *reinterpret_cast<const uint32_t*>(R + 60);
        const uint32_t w1 = *reinterpret_cast<const uint32_t*>(R + 64);        // latest_flags u16 | eth u16
        const uint32_t state = R[68];
        const uint32_t flags = w1 & 0xFFFFu, eth = w1 >> 16;
        v[0] = ~seq;
        v[1] = w0 & 0xFFFFu;
        v[2] = w0 >> 16;
        v[3] = cause ? seq + 1 : 0ull;
        v[4] = state ? ((seq + 1) << 8) | state : 0ull;
        v[5] = flags;
        v[6] = start ? 0ull - start : 0ull;
        v[7] = end;
        v[8] = eth ? ~((seq << 16) | eth) : 0ull;
    }
    static __device__ __forceinline__ void fold(uint64_t* a, int st, const uint64_t* v) {
        smem_max_u64(a + 0 * st, v[0]); smem_add_u64(a + 1 * st, v[1]); smem_add_u64(a + 2 * st, v[2]); smem_max_u64(a + 3 * st, v[3]);
        smem_max_u64(a + 4 * st, v[4]); smem_or_u64(a + 5 * st, v[5]); smem_max_u64(a + 6 * st, v[6]); smem_max_u64(a + 7 * st, v[7]);
        smem_max_u64(a + 8 * st, v[8]);
    }
    static __device__ __forceinline__ void flush(uint8_t* S, const uint64_t* a, int st) {
        gmax(S + 0, a[0 * st]); gadd(S + 8, a[1 * st]); gadd(S + 16, a[2 * st]); gmax(S + 24, a[3 * st]); gmax(S + 32, a[4 * st]); gor32(S + 40, a[5 * st]);
        gmax(S + 48, a[6 * st]); gmax(S + 56, a[7 * st]); gmax(S + 64, a[8 * st]);
    }
};

// CTA-wide cache of hot flows, alive across the tiles of one launch: a flow with >= 3 samples in one tile is installed
// (key, table slot, zeroed accumulators); later samples of that flow fold into the entry with shared-memory atomics and
// touch neither the election nor the table; the entries are flushed with one set of reductions when the CTA runs out of
// tiles.  Without it every tile sends its own reductions for the hottest flows to the same few L2 addresses.
constexpr int kFeatHot = 32;
constexpr uint32_t kFeatCached = 0xFFFFFFFEu;
template <class F> struct FeatHot {
    uint64_t key[5];
    uint32_t state, slot;                       // state: 0 empty, 1 being filled, 2 live
    uint64_t acc[F::kAcc];
};

template <class F> constexpr size_t feature_fold_smem() {
    // tile (re-used for the representatives' accumulators once the keys are no longer needed) | election set | 1 KB spare |
    // duplicate counts | hot-flow cache
    constexpr size_t tile = (size_t)kFeatTile * (F::kRec > F::kAcc * 8 ? F::kRec : F::kAcc * 8);
    return tile + kFeatRep * 4 + kFeatTile * 4 + kFeatTile * 4 + kFeatHot * sizeof(FeatHot<F>);
}

// kDevN: the sample count is min(*n_dev, max_n), read from device memory (a count another GPU's route stored); the grid
// is sized from max_n and the CTAs past the count only start and stop.  Otherwise n_dev is unused and n = max_n.
template <class F, bool kDevN = false>
__global__ void __launch_bounds__(kFeatTile, FA_K6_MINBLOCKS)
feature_fold_kernel(const uint8_t* __restrict__ recs, uint32_t max_n, Table t, uint64_t epoch, uint64_t seq0,
                    uint32_t* __restrict__ slot_of, Counters* ctr, const unsigned long long* __restrict__ n_dev = nullptr) {
    const uint32_t n = kDevN ? (uint32_t)min((unsigned long long)max_n, *n_dev) : max_n;
    FA_DYN_SMEM(sm);
    constexpr size_t kTileBytes = (size_t)kFeatTile * (F::kRec > F::kAcc * 8 ? F::kRec : F::kAcc * 8);
    uint64_t* tile = reinterpret_cast<uint64_t*>(sm);                         // kFeatTile samples ...
    uint64_t* acc = tile;                                                     // ... then [kAcc][kFeatTile] accumulators
    uint32_t* rep = reinterpret_cast<uint32_t*>(sm + kTileBytes);             // [kFeatRep] election set
    uint32_t* dupc = rep + kFeatRep + kFeatTile;                              // (1 KB kept free after the election set: the measured layout)
                                                                              //                                      // [kFeatTile] duplicates folded into it
    FeatHot<F>* hot = reinterpret_cast<FeatHot<F>*>(dupc + kFeatTile);
    const uint32_t tid = threadIdx.x;
    if (tid < kFeatHot) hot[tid].state = 0u;
    const uint32_t n_tiles = (n + kFeatTile - 1) / kFeatTile;
    for (uint32_t tix = blockIdx.x; tix < n_tiles; tix += gridDim.x) {
        const uint32_t first = tix * kFeatTile, cnt = min((uint32_t)kFeatTile, n - first);
        const uint64_t* G = reinterpret_cast<const uint64_t*>(recs + (size_t)first * F::kRec);
        {   // the CTA's next tile: ask L2 for it now, one 128-byte line per thread
            const uint32_t ntx = tix + gridDim.x;
            if (ntx < n_tiles) {
                const uint8_t* nb = recs + (size_t)ntx * kFeatTile * F::kRec;
                const uint32_t nbytes = min((uint32_t)kFeatTile, n - ntx * kFeatTile) * F::kRec;
                if (tid * 128u < nbytes) prefetch_l2(nb + tid * 128u);
            }
        }
        if (cnt == (uint32_t)kFeatTile) {                                    // all loads in flight before the first store
            uint64_t tmp[F::kRec / 8];
#pragma unroll
            for (int w = 0; w < F::kRec / 8; w++) tmp[w] = G[tid + w * kFeatTile];
#pragma unroll
            for (int w = 0; w < F::kRec / 8; w++) tile[tid + w * kFeatTile] = tmp[w];
        } else {
            for (uint32_t w = tid; w < cnt * (F::kRec / 8); w += kFeatTile) tile[w] = G[w];
        }
        for (uint32_t w = tid; w < kFeatRep; w += kFeatTile) rep[w] = kFeatNone;
        if (tid < cnt) slot_of[first + tid] = kFeatNone;                      // only a flow's candidates for "first" / "last" get a slot below
        __syncthreads();
        const bool valid = tid < cnt;
        const uint8_t* R = reinterpret_cast<const uint8_t*>(tile) + (size_t)tid * F::kRec;
        uint32_t r = tid, hq = 0;                                             // my representative (kFeatCached: a hot-flow cache entry)
        uint64_t k[5] = {0, 0, 0, 0, 0}, v[F::kAcc];
        if (valid) {
            load_key(R, k);
            k[4] &= 0x00FFFFFFFFFFFFFFull;
            const uint64_t h = slot_hash(key_premix(k[0], k[1], k[2], k[3], k[4]));
            F::extract(R, seq0 + first + tid, v);
            hq = (uint32_t)(h >> 52) & (kFeatHot - 1);
            FeatHot<F>& e = hot[hq];
            if (e.state == 2u && e.key[0] == k[0] && e.key[1] == k[1] && e.key[2] == k[2] && e.key[3] == k[3] && e.key[4] == k[4]) {
                r = kFeatCached;                                              // hot flow: no election, no probe, no global reduction
            } else {
                uint32_t q = (uint32_t)(h >> 40) & (kFeatRep - 1);
                for (int step = 0; step < 8; step++) {
                    const uint32_t cur = atomicCAS(&rep[q], kFeatNone, tid);
                    if (cur == kFeatNone) break;                              // nobody holds this key yet: I represent it
                    const uint64_t* K = tile + (size_t)cur * (F::kRec / 8);
                    if (K[0] == k[0] && K[1] == k[1] && K[2] == k[2] && K[3] == k[3] && (K[4] & 0x00FFFFFFFFFFFFFFull) == k[4]) { r = cur; break; }
                    q = (q + 1) & (kFeatRep - 1);                             // after 8 steps: stay my own representative (unmerged, still exact)
                }
            }
        }
        if (valid && r == kFeatCached) F::fold(hot[hq].acc, 1, v);
        __syncthreads();                                                      // the samples are parsed: the tile becomes the accumulators
        if (valid && r == tid) {
#pragma unroll
            for (int a = 0; a < F::kAcc; a++) acc[a * kFeatTile + tid] = v[a];   // field-major: neighbours hit neighbouring banks
            dupc[tid] = 0u;
        }
        __syncthreads();
        if (valid && r < (uint32_t)kFeatTile && r != tid) { F::fold(acc + r, kFeatTile, v); atomicAdd(&dupc[r], 1u); }
        __syncthreads();
        if (valid && r == tid) {
            const uint32_t slot = find_or_create(t, epoch, k, &ctr->live);
            if (slot == kFeatNone) atomicAdd(&ctr->spills, 1ull + dupc[tid]);
            else {
                // the tile's earliest sample of the flow (and, for drops, its last one with a cause) are the only ones the
                // second pass has to look at: acc 0 = max ~seq, acc kCand2 = max (seq + 1)
                slot_of[(uint32_t)(~acc[tid] - seq0)] = slot;
                if (F::kCand2 >= 0) { const uint64_t c2 = acc[(F::kCand2 < 0 ? 0 : F::kCand2) * kFeatTile + tid]; if (c2) slot_of[(uint32_t)(c2 - 1 - seq0)] = slot; }
            }
            if (slot != kFeatNone) {
                F::flush(F::state(t, slot), acc + tid, kFeatTile);
                FeatHot<F>& e = hot[hq];
                if (dupc[tid] >= 2u && atomicCAS(&e.state, 0u, 1u) == 0u) {    // three samples in one tile: worth an entry
#pragma unroll
                    for (int c = 0; c < 5; c++) e.key[c] = k[c];
#pragma unroll
                    for (int a = 0; a < F::kAcc; a++) e.acc[a] = 0ull;
                    e.slot = slot;
                    __threadfence_block();
                    *reinterpret_cast<volatile uint32_t*>(&e.state) = 2u;     // readers look at it after the next barrier
                }
            }
        }
        __syncthreads();                                                      // tile / rep are re-used
    }
    __syncthreads();
    if (tid < kFeatHot && hot[tid].state == 2u) {
        F::flush(F::state(t, hot[tid].slot), hot[tid].acc, 1);
        if (hot[tid].acc[0]) slot_of[(uint32_t)(~hot[tid].acc[0] - seq0)] = hot[tid].slot;
        if (F::kCand2 >= 0) { const uint64_t c2 = hot[tid].acc[F::kCand2 < 0 ? 0 : F::kCand2]; if (c2) slot_of[(uint32_t)(c2 - 1 - seq0)] = hot[tid].slot; }
    }
}

// second pass: the sample that turned out to be the flow's first one writes the adopted block fields
template <bool kDevN = false>
__global__ void additional_first_kernel(const uint8_t* __restrict__ recs, uint32_t max_n, Table t, uint64_t seq0,
                                        const uint32_t* __restrict__ slot_of, const unsigned long long* __restrict__ n_dev = nullptr) {
    const uint32_t n = kDevN ? (uint32_t)min((unsigned long long)max_n, *n_dev) : max_n;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t slot = slot_of[i];
        if (slot == 0xFFFFFFFFu) continue;
        uint8_t* S = reinterpret_cast<uint8_t*>(t.feat_add) + (size_t)slot * (kAddState * 16);
        if (*reinterpret_cast<const uint64_t*>(S) != ~(seq0 + i)) continue;
        const uint8_t* R = recs + (size_t)i * kAddRecBytes;
        *reinterpret_cast<uint64_t*>(S + 48) = ld_u64_unaligned8(R + 40);
        *reinterpret_cast<uint64_t*>(S + 56) = ld_u64_unaligned8(R + 48);
        *reinterpret_cast<uint32_t*>(S + 64) = *reinterpret_cast<const uint32_t*>(R + 68) & 0xFFFFu;
    }
}

template <bool kDevN = false>
__global__ void dns_first_kernel(const uint8_t* __restrict__ recs, uint32_t max_n, Table t, uint64_t seq0,
                                 const uint32_t* __restrict__ slot_of, const unsigned long long* __restrict__ n_dev = nullptr) {
    const uint32_t n = kDevN ? (uint32_t)min((unsigned long long)max_n, *n_dev) : max_n;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t slot = slot_of[i];
        if (slot == 0xFFFFFFFFu) continue;
        uint8_t* S = reinterpret_cast<uint8_t*>(t.feat_dns) + (size_t)slot * (kDnsState * 16);
        if (*reinterpret_cast<const uint64_t*>(S) != ~(seq0 + i)) continue;
        const uint8_t* R = recs + (size_t)i * kDnsRecBytes;
        *reinterpret_cast<uint16_t*>(S + 60) = *reinterpret_cast<const uint16_t*>(R + 68);    // first.eth
        *reinterpret_cast<uint64_t*>(S + 64) = ld_u64_unaligned8(R + 40);
        *reinterpret_cast<uint64_t*>(S + 72) = ld_u64_unaligned8(R + 48);
        for (int b = 0; b < 32; b++) S[80 + b] = R[71 + b];                                    // name[32] at +31 of dns_metrics
    }
}

template <bool kDevN = false>
__global__ void pktdrop_first_kernel(const uint8_t* __restrict__ recs, uint32_t max_n, Table t, uint64_t seq0,
                                     const uint32_t* __restrict__ slot_of, const unsigned long long* __restrict__ n_dev = nullptr) {
    const uint32_t n = kDevN ? (uint32_t)min((unsigned long long)max_n, *n_dev) : max_n;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t slot = slot_of[i];
        if (slot == 0xFFFFFFFFu) continue;
        uint8_t* S = reinterpret_cast<uint8_t*>(t.feat_drop) + (size_t)slot * (kDropState * 16);
        const uint8_t* R = recs + (size_t)i * kDropRecBytes;
        const uint64_t seq = seq0 + i;
        if (*reinterpret_cast<const uint64_t*>(S) == ~seq) {                   // the flow's first sample: its block is adopted
            *reinterpret_cast<uint16_t*>(S + 44) = *reinterpret_cast<const uint16_t*>(R + 66);
            *reinterpret_cast<uint64_t*>(S + 72) = ld_u64_unaligned8(R + 40);
            *reinterpret_cast<uint64_t*>(S + 80) = ld_u64_unaligned8(R + 48);
        }
        if (*reinterpret_cast<const uint64_t*>(S + 24) == seq + 1)             // the last sample with a drop cause
            *reinterpret_cast<uint32_t*>(S + 88) = *reinterpret_cast<const uint32_t*>(R + 60);
    }
}

// persistent over tiles: exactly as many CTAs as are resident at once (a partial second wave would leave SMs idle)
template <class F, bool kDevN>
static uint32_t fold_grid(uint32_t n_tiles, int sm_count) {
#ifndef FA_HOST_EMUL
    static int per_sm = 0;
    if (!per_sm) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, feature_fold_kernel<F, kDevN>, kFeatTile, feature_fold_smem<F>()) != cudaSuccess || per_sm < 1) per_sm = 4;
    }
    return std::min<uint32_t>(n_tiles, (uint32_t)(sm_count * per_sm));
#else
    (void)sm_count;
    return n_tiles;
#endif
}

// The fold and its second pass, for a host count (n = max_n) or a device one (min(*n_dev, max_n)); the same launches
// either way, sized from max_n.
using FirstKernel = void (*)(const uint8_t*, uint32_t, Table, uint64_t, const uint32_t*, const unsigned long long*);
template <class F, bool kDevN>
static int launch_fold(FirstKernel first_kernel, const uint8_t* recs, uint32_t max_n, const unsigned long long* n_dev, const Table& t,
                       uint64_t epoch, uint64_t seq0, uint32_t* slot_of, Counters* ctr, int sm_count, cudaStream_t st) {
    const uint32_t n_tiles = (max_n + kFeatTile - 1) / kFeatTile;
    const auto fold = feature_fold_kernel<F, kDevN>;
    const uint32_t grid = fold_grid<F, kDevN>(n_tiles, sm_count);
    FA_LAUNCH(fold, grid, kFeatTile, feature_fold_smem<F>(), st, recs, max_n, t, epoch, seq0, slot_of, ctr, n_dev);
    FA_LAUNCH(first_kernel, sm_count * 8, 256, 0, st, recs, max_n, t, seq0, slot_of, n_dev);
    return 2;
}

#ifndef FA_HOST_EMUL
int launch_feature_fold(int kind, const uint8_t* recs, uint32_t n, const Table& t, uint64_t epoch, uint64_t seq0,
                        uint32_t* slot_of, Counters* ctr, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    static_assert(feature_fold_smem<DnsFeat>() <= 48 * 1024 && feature_fold_smem<DropFeat>() <= 48 * 1024, "K6 tiles fit the default 48 KB");
    if (kind == 2) return launch_fold<DropFeat, false>(pktdrop_first_kernel<false>, recs, n, nullptr, t, epoch, seq0, slot_of, ctr, sm_count, st);
    if (kind == 0) return launch_fold<AddFeat, false>(additional_first_kernel<false>, recs, n, nullptr, t, epoch, seq0, slot_of, ctr, sm_count, st);
    return launch_fold<DnsFeat, false>(dns_first_kernel<false>, recs, n, nullptr, t, epoch, seq0, slot_of, ctr, sm_count, st);
}
#endif  // FA_HOST_EMUL

// One text for the device and the host emulation (FA_LAUNCH): both kernels loop over tiles / samples grid-stride.
int launch_feature_fold_counted(int kind, const uint8_t* recs, const unsigned long long* n_dev, uint32_t max_n, const Table& t,
                                uint64_t epoch, uint64_t seq0, uint32_t* slot_of, Counters* ctr, int sm_count, cudaStream_t st) {
    if (!max_n) return 0;
    if (kind == 2) return launch_fold<DropFeat, true>(pktdrop_first_kernel<true>, recs, max_n, n_dev, t, epoch, seq0, slot_of, ctr, sm_count, st);
    if (kind == 0) return launch_fold<AddFeat, true>(additional_first_kernel<true>, recs, max_n, n_dev, t, epoch, seq0, slot_of, ctr, sm_count, st);
    return launch_fold<DnsFeat, true>(dns_first_kernel<true>, recs, max_n, n_dev, t, epoch, seq0, slot_of, ctr, sm_count, st);
}

// ---- eviction: patch the base with the feature effects (feature_patch, kernels.cuh), emit and clear the feature blocks
// kClear = false: the fa_top_flows / fa_lookup_flows peek, which emits the same rows and leaves the feature lines as
// they are; a row whose slot is kNoSlot (a lookup miss) gets zero feature rows and present = 0.  Launched as 8 CTAs of
// 256 threads per SM: the bound keeps them all resident (32 registers).
template <bool kClear = true>
__global__ void __launch_bounds__(256, 8) evict_features_kernel(Table t, const uint32_t* __restrict__ slot_of_out, unsigned long long n_out,
                                      uint8_t* __restrict__ out_recs, uint8_t* __restrict__ out_dns,
                                      uint8_t* __restrict__ out_add, uint8_t* __restrict__ out_drop,
                                      unsigned long long* __restrict__ out_rtt_min, uint8_t* __restrict__ out_present) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n_out;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t slot = slot_of_out[i];
        if (!kClear && slot == kNoSlot) {
            if (t.feat_dns && out_dns) for (int c = 0; c < 8; c++) reinterpret_cast<uint64_t*>(out_dns + i * 64)[c] = 0ull;
            if (t.feat_drop && out_drop) for (int c = 0; c < 4; c++) reinterpret_cast<uint64_t*>(out_drop + i * 32)[c] = 0ull;
            if (t.feat_add && out_add) for (int c = 0; c < 4; c++) reinterpret_cast<uint64_t*>(out_add + i * 32)[c] = 0ull;
            if (out_rtt_min) out_rtt_min[i] = 0ull;
            if (out_present) out_present[i] = 0;
            continue;
        }
        uint8_t* O = out_recs + i * kRecBytes;
        uint64_t bs = *reinterpret_cast<uint64_t*>(O + R_START), be = *reinterpret_cast<uint64_t*>(O + R_END);
        uint32_t beth = *reinterpret_cast<uint16_t*>(O + R_ETH);
        const uint32_t present = feature_patch(t, slot, bs, be, beth);
        if (t.feat_dns) {
            uint64_t* S = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(t.feat_dns) + (size_t)slot * (kDnsState * 16));
            if (present & 1) {
                if (out_dns) {
                    uint8_t* D = out_dns + i * 64;
                    const uint8_t* Sb = reinterpret_cast<const uint8_t*>(S);
                    *reinterpret_cast<uint64_t*>(D + 0) = S[8];                              // first.start
                    *reinterpret_cast<uint64_t*>(D + 8) = S[9];                              // first.end
                    *reinterpret_cast<uint64_t*>(D + 16) = S[1];                             // latency max
                    *reinterpret_cast<uint16_t*>(D + 24) = (uint16_t)(S[2] & 0xFFFFu);       // id: last non-zero
                    *reinterpret_cast<uint16_t*>(D + 26) = (uint16_t)(*reinterpret_cast<const uint32_t*>(Sb + 56));  // flags
                    *reinterpret_cast<uint16_t*>(D + 28) = *reinterpret_cast<const uint16_t*>(Sb + 60);              // first.eth
                    D[30] = (uint8_t)(S[3] & 0xFFu);                                         // errno: last
                    for (int b = 0; b < 32; b++) D[31 + b] = Sb[80 + b];
                    D[63] = 0;
                }
                if (kClear) {
#pragma unroll
                    for (int c = 0; c < 16; c++) S[c] = 0ull;
                }
            } else if (out_dns) {
                for (int c = 0; c < 8; c++) reinterpret_cast<uint64_t*>(out_dns + i * 64)[c] = 0ull;
            }
        }
        if (t.feat_drop) {
            uint64_t* S = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(t.feat_drop) + (size_t)slot * (kDropState * 16));
            if (present & 4) {
                if (out_drop) {
                    uint8_t* D = out_drop + i * 32;
                    const uint8_t* Sb = reinterpret_cast<const uint8_t*>(S);
                    *reinterpret_cast<uint64_t*>(D + 0) = S[9];                              // first.start
                    *reinterpret_cast<uint64_t*>(D + 8) = S[10];                             // first.end
                    *reinterpret_cast<uint16_t*>(D + 16) = (uint16_t)(S[1] > 0xFFFFull ? 0xFFFFull : S[1]);   // addUint16 saturates
                    *reinterpret_cast<uint16_t*>(D + 18) = (uint16_t)(S[2] > 0xFFFFull ? 0xFFFFull : S[2]);
                    *reinterpret_cast<uint32_t*>(D + 20) = *reinterpret_cast<const uint32_t*>(Sb + 88);   // latest_drop_cause: last non-zero
                    *reinterpret_cast<uint16_t*>(D + 24) = (uint16_t)(*reinterpret_cast<const uint32_t*>(Sb + 40));  // latest_flags: or
                    *reinterpret_cast<uint16_t*>(D + 26) = *reinterpret_cast<const uint16_t*>(Sb + 44);              // first.eth
                    *reinterpret_cast<uint32_t*>(D + 28) = (uint32_t)(S[4] & 0xFFu);          // latest_state: last non-zero; padding
                }
                if (kClear) {
#pragma unroll
                    for (int c = 0; c < 12; c++) S[c] = 0ull;
                }
            } else if (out_drop) {
                for (int c = 0; c < 4; c++) reinterpret_cast<uint64_t*>(out_drop + i * 32)[c] = 0ull;
            }
        }
        if (out_rtt_min) out_rtt_min[i] = 0ull;
        if (t.feat_add) {
            uint64_t* S = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(t.feat_add) + (size_t)slot * (kAddState * 16));
            if (present & 2) {
                if (out_rtt_min) out_rtt_min[i] = S[9] ? ~S[9] : 0ull;                       // extension: smallest non-zero RTT
                if (out_add) {
                    uint8_t* A = out_add + i * 32;
                    *reinterpret_cast<uint64_t*>(A + 0) = S[6];                              // first.start
                    *reinterpret_cast<uint64_t*>(A + 8) = S[7];                              // first.end
                    *reinterpret_cast<uint64_t*>(A + 16) = S[1];                             // rtt max
                    const uint64_t ip = S[2];
                    *reinterpret_cast<uint32_t*>(A + 24) = (uint32_t)((ip >> 1) & 0xFFFFFFFFu) ^ 0x80000000u;
                    *reinterpret_cast<uint16_t*>(A + 28) = (uint16_t)(S[8] & 0xFFFFu);       // first.eth
                    A[30] = (uint8_t)(ip & 1u);
                    A[31] = 0;
                }
                if (kClear) {
#pragma unroll
                    for (int c = 0; c < 10; c++) S[c] = 0ull;
                }
            } else if (out_add) {
                for (int c = 0; c < 4; c++) reinterpret_cast<uint64_t*>(out_add + i * 32)[c] = 0ull;
            }
        }
        if (present) {
            *reinterpret_cast<uint64_t*>(O + R_START) = bs;
            *reinterpret_cast<uint64_t*>(O + R_END) = be;
            *reinterpret_cast<uint16_t*>(O + R_ETH) = (uint16_t)beth;
        }
        if (out_present) out_present[i] = present;
    }
}

#ifndef FA_HOST_EMUL
int launch_evict_features(const Table& t, const uint32_t* slot_of_out, unsigned long long n_out, uint8_t* out_recs,
                          uint8_t* out_dns, uint8_t* out_add, uint8_t* out_drop, unsigned long long* out_rtt_min,
                          uint8_t* out_present, int sm_count, cudaStream_t st) {
    if (!n_out) return 0;
    evict_features_kernel<true><<<sm_count * 8, 256, 0, st>>>(t, slot_of_out, n_out, out_recs, out_dns, out_add, out_drop, out_rtt_min, out_present);
    return 1;
}
#endif  // FA_HOST_EMUL

int launch_peek_features(const Table& t, const uint32_t* slot_of_out, unsigned long long n_out, uint8_t* out_recs,
                         uint8_t* out_dns, uint8_t* out_add, uint8_t* out_drop, unsigned long long* out_rtt_min,
                         uint8_t* out_present, int sm_count, cudaStream_t st) {
    if (!n_out) return 0;
    FA_LAUNCH(evict_features_kernel<false>, sm_count * 8, 256, 0, st, t, slot_of_out, n_out, out_recs, out_dns, out_add, out_drop,
              out_rtt_min, out_present);
    return 1;
}

}  // namespace fa
