// aggregate.cu — K1 flow_aggregate: fold a batch of 144-byte flow records into the
// open-addressed flow table with the semantics of the reference's userspace Accounter
// (pkg/flow/account.go:82-96 + pkg/model/flow_content.go:28-61).
//
// One persistent CTA per SM, 1024 threads = 4 teams of 256 (FA_K1_TILE).  Each team works through
// 256-record tiles and synchronises with a named barrier; all teams share a small cache of the
// hottest flows.  A team's first tile is blockIdx.x * kTeams + team; it claims every later one from
// a per-launch counter while it works on the current one, so teams that run ahead take the tail of
// the batch instead of waiting on a fixed stride.  The last CTA out resets the counter and writes
// the live-flow count into the host's mapped ring (no copy node between launches).  Per tile:
//   TMA bulk copy (cp.async.bulk + mbarrier) stages 36 KB of records in shared memory
//   -> E: each thread hashes one record; a record of a cached hot flow folds straight into
//      the cache's shared-memory accumulators; every other record writes its own values into
//      its accumulator words and enters the tile's election set (shared-memory CAS table whose
//      slots carry hash bits): the first record of a key becomes its representative, later
//      ones fold into the representative's accumulators with 32-bit shared atomics
//   -> probe: the list of representatives is split evenly over the team's warps; 8 lanes
//      per flow, rounds of 4 flows, four identity lines (128 B each, one coalesced load) in
//      flight per warp at all times (the load of round r + 4 is issued when round r has been
//      compared); a masked 16-byte compare per lane and one ballot decide hit / miss; flows
//      whose home slot holds another flow are collected and probed one slot on in a second,
//      compact pass
//   -> general loop (rare): inserts (CAS-claim, write, fence, publish), collisions, flows
//      being published by another SM
//   -> the last warp out of the probe phase re-arms the tile's TMA for the team's next tile
//   -> one lane per flow, from the accumulators alone: three fire-and-forget reductions on
//      the 32-byte hot line (RED.add bytes, RED.add packets, RED.max end; start / flags only
//      when they can change it).
// The cache is flushed with the same reductions when the CTA runs out of tiles: it lives for one launch.
//
// The cache: 96 entries as 12 sets x 8 ways, the set picked by the upper half of the 32-bit slot hash.  A set's eight
// 16-bit tags (lower hash bits | 1) are one 16-byte word, so a lookup is one shared-memory load and eight compares
// before it touches an entry; only a way whose tag matches is checked by its full hash and then by the 114 bytes.  A
// flow with two records in one tile takes a free way of its set, first come first served, and keeps it for the launch.
//
// Exactness of the order-dependent fields (eth_protocol / dscp / sampling = last non-zero,
// MACs = first non-zero, everything else = first record; flow_content.go:45-59,
// account.go:95): while every record of a flow carries the same 74-byte descriptor the
// merge result does not depend on order, so the fast path only *compares* descriptors
// (exactly, all 74 bytes).  Any mismatch flags the flow TAG_DIRTY and the two re-fold kernels
// below recompute those fields from the batch in stream-index order.
#include "kernels.cuh"

namespace fa {

#ifndef FA_K1_TILE
#define FA_K1_TILE 256   // 4 teams x 256-record tiles; on H100 SXM (400 W) +11.6 % zipf10m, -0.6 % uniform10m over 8 x 128
#endif
constexpr int kTile      = FA_K1_TILE;          // records per tile == threads per team
constexpr int kTeams     = 1024 / kTile;        // teams per CTA (one CTA per SM): independent tile pipelines that fill each other's
                                                // bubbles (tile wait, team barriers); 8 x 128 stays selectable (FA_K1_TILE=128)
constexpr int kCtaThreads = kTile * kTeams;
constexpr int kRepSlots  = 2 * kTile;
constexpr int kHotWays = 8;                     // ways of a cache set: their 16-bit tags are one 16-byte shared-memory load
constexpr int kHotSets = 12;
constexpr int kHotEntries = kHotSets * kHotWays;
typedef uint8_t RepIdx;                         // index of a record inside its tile
static_assert(kTile == 128 || kTile == 256, "election slots and lists keep the tile index in 8 bits; 1024 threads per CTA");
#ifndef FA_K1_STREAM_HINT
#define FA_K1_STREAM_HINT 1   // record stream read with an L2 evict-first policy: it is read once, the table lines stay
#endif
#ifndef FA_K1_MINDUPS
#define FA_K1_MINDUPS 1
#endif
constexpr uint32_t kHotMinDups = FA_K1_MINDUPS; // a flow with >= 2 records in one tile becomes a cache candidate
constexpr uint32_t kRepEmpty = 0xFFFFFFFFu;
constexpr uint32_t kResSpill = 0xFFFFFFFFu;
constexpr uint32_t kProbeLimit = 8192;

struct __align__(128) TeamSmem {                  // 26,496 B per team (128-record tiles)
    uint4    tile[kTile * kRecChunks];            // 18,432 B  one TMA-staged tile of records
    uint32_t acc[kTile][8];                       //  4,096 B  per record: bytes lo / hi | packets | flags + duplicates << 16 (+ kSketch packet carries << 24) | ns lo | end lo | ns hi | end hi
    uint32_t hs[kTile];                           //    512 B  low 32 bits of the slot hash
    uint4    res4[kTile];                         //  2,048 B  per representative: table slot | start mirror lo | eth + mirror hi | flag bits the hot line holds
    uint32_t rep[kRepSlots];                      //  1,024 B  tile-local election set: 23 hash bits << 8 | representative index
    uint8_t  tdirty[kTile];                       //    128 B  set by duplicates whose descriptor differs
    RepIdx   glist[kTile];                        //    128 B  team-wide compacted list of representatives
    RepIdx   slow[kTile / 32][32];                //    128 B  per warp: general-loop flows from the front, second-pass flows from the back
};
struct __align__(16) TeamCtl {                    // kept outside TeamSmem so that the teams + the cache fit in 227 KB
    unsigned long long full_bar;                  // mbarrier of the team's tile
    uint32_t nrep, done;                          // representatives of the tile; warps that are through with its probes
    uint32_t next[2];                             // the team's next tile, claimed during tile `it`, in next[it & 1]
    uint32_t pad[2];
};
struct __align__(16) HotEntry {                   // 208 B: a stride of 52 words keeps 8 entries on distinct banks
    uint4    line[8];                             // copy of the flow's identity line
    uint32_t acc[8];                              // bytes lo/hi, packets, flags, ns lo (max), end lo (max), hits, packet carries (kSketch)
    uint32_t state;                               // 0 empty, 1 being filled, 2 live
    uint32_t hash;                                // low 32 bits of the slot hash
    uint32_t slot;
    uint32_t ns_hi, end_hi;                       // high words the 32-bit max windows are relative to
    uint32_t pad[7];
};
static_assert(sizeof(HotEntry) == 208, "HotEntry stride");
static_assert(kTile != 128 || sizeof(TeamSmem) == 26496, "TeamSmem has no padding to spare");
struct __align__(128) AggSmem {                   // 232,320 B (sizeof) of the 232,448 B (227 KB) an sm_90 CTA may use
    TeamSmem team[kTeams];
    HotEntry hot[kHotEntries];
    alignas(16) uint16_t hot_tag[kHotEntries];    // per entry: low 16 hash bits | 1 of the live entry, 0 = none (written after state = 2)
    TeamCtl  ctl[kTeams];
    uint32_t n_insert, n_spill, any_dirty, pad;
};
static_assert(sizeof(AggSmem) <= 232448, "K1 shared memory exceeds what one sm_90 CTA can opt into");

// Cache set and tag of a flow, from the low 32 bits of its slot hash; the ways of `tags` (8 x 16 bit) that hold `tag`.
__device__ __forceinline__ uint32_t hot_set(uint32_t h) { return ((h >> 16) * (uint32_t)kHotSets) >> 16; }
__device__ __forceinline__ uint32_t hot_tag_of(uint32_t h) { return (h & 0xFFFFu) | 1u; }
__device__ __forceinline__ uint32_t hot_ways_with(uint4 tags, uint32_t tag) {
    const uint32_t w[4] = {tags.x, tags.y, tags.z, tags.w};
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t x = w[i] ^ (tag * 0x10001u);
        m |= ((x & 0xFFFFu) == 0u ? 1u : 0u) << (2 * i) | ((x >> 16) == 0u ? 2u : 0u) << (2 * i);
    }
    return m;
}
static_assert(kHotWays * sizeof(uint16_t) == sizeof(uint4), "a set's tags are read as one uint4");

__device__ __forceinline__ void team_sync(int team) { named_barrier_sync(team + 1, kTile); }

// Per-launch words of K1 in Counters::scratch, zero between launches: [0] counts the tiles claimed after each team's
// first, [2] is the ticket of CTAs that are through, whose last holder zeroes both.  ([1] is fixup_apply's ticket.)
__device__ __forceinline__ unsigned int* k1_tile_claims(Counters* c) { return reinterpret_cast<unsigned int*>(&c->scratch[0]); }
__device__ __forceinline__ unsigned int* k1_exit_ticket(Counters* c) { return reinterpret_cast<unsigned int*>(&c->scratch[2]); }

__device__ __forceinline__ void issue_tile_load(TeamSmem& s, TeamCtl& tc, const uint4* recs, uint32_t n, uint32_t tile_idx) {
    const uint32_t first = tile_idx * kTile;
    const uint32_t cnt = min((uint32_t)kTile, n - first);
    const uint32_t bytes = cnt * kRecBytes;
    mbar_expect_tx(&tc.full_bar, bytes);
#if FA_K1_STREAM_HINT
    tma_load_1d_stream(&s.tile[0], recs + (size_t)first * kRecChunks, bytes, &tc.full_bar);    // L2 evict-first for the record stream
#else
    tma_load_1d(&s.tile[0], recs + (size_t)first * kRecChunks, bytes, &tc.full_bar);
#endif
}

// Reductions of one flow's folded totals onto its hot line.  floor_ns <= hot.nstart always
// (immutable start mirror), `seen` are flag bits the hot line is known to hold already.
__device__ __forceinline__ void reduce_to_hot(const Table& t, uint32_t slot, uint64_t bytes, uint32_t packets,
                                              uint64_t ns, uint64_t end, uint32_t flags, uint64_t floor_ns, uint32_t seen) {
    uint8_t* hot = reinterpret_cast<uint8_t*>(t.hot) + (size_t)slot * kHotBytes;
    red_add_u64(hot, bytes);
    if (ns > floor_ns) red_max_u64(hot + 8, ns);
    if (end) red_max_u64(hot + 16, end);
    red_add_u32(hot + 24, packets);
    flags &= ~seen;
    if (flags) {
        red_or_u32(hot + 28, flags);
        red_or_u64(reinterpret_cast<uint8_t*>(&t.ident[(size_t)slot * 8 + 2]) + 8, (unsigned long long)flags << TAG_FLAGS_SHIFT);
    }
}

// Fused sketches (new capability, no reference): count-min += packets, HyperLogLog register = max(rho).
// The tile and cache accumulators hold a flow's packets in 32 bits, like the flow table, while the count-min counters
// are 64-bit sums of every record's packets: with kSketch a fold whose 32-bit add carries also counts the carry
// (tile: bits 24..31 of acc[3], above the duplicate count; cache: acc[7]), and `packets` here is the 64-bit total.
__device__ __forceinline__ void sketch_update(const SketchParams& sk, uint64_t premix, uint64_t packets) {
    const uint64_t a = cms_hash_a(premix, sk.seed), b = cms_hash_b(premix, sk.seed);
    for (uint32_t d = 0; d < sk.depth; d++)
        red_add_u64(sk.cms + ((size_t)d << sk.log2w) + cms_index(a, b, d, sk.log2w), packets);
    const uint64_t hh = hll_hash(premix, sk.seed);
    const uint32_t idx = (uint32_t)(hh >> (64 - sk.p));
    const uint64_t rest = hh << sk.p;
    const uint32_t rho = rest ? (uint32_t)__clzll((long long)rest) + 1u : (64u - sk.p) + 1u;
    if (__ldcg(&sk.hll[idx]) < rho) red_max_u32(&sk.hll[idx], rho);
}

// General probe of one flow per 8-lane group (4 flows per call): claims empty slots, waits for
// slots being published, walks collisions, marks descriptor mismatches.  Returns the slot
// (kResSpill when the table is physically full) in every lane of the group.
__device__ __forceinline__ uint32_t probe_general(const Table& t, uint64_t epoch, bool active, uint32_t start_slot,
                                                  uint4 rchunk, bool cta_dirty, uint64_t ins_ns, int g, int j, uint4 cmask,
                                                  uint32_t& my_inserts, uint32_t* any_dirty) {
    uint64_t slot = start_slot;
    bool done = !active;
    uint32_t nprobe = 0, result = kResSpill;
    uint64_t reload_slot = ~0ull;
    for (;;) {
        uint4 line = make_uint4(0, 0, 0, 0);
        if (!done) line = ld_cg_u4(&t.ident[slot * 8 + j]);
        const uint32_t tag_lo = __shfl_sync(0xFFFFFFFFu, line.z, g * 8 + 2);
        const uint32_t tag_hi = __shfl_sync(0xFFFFFFFFu, line.w, g * 8 + 2);
        const uint64_t tag = u64_of(tag_lo, tag_hi);
        const uint32_t eqb = (__ballot_sync(0xFFFFFFFFu, eq4_masked(line, rchunk, cmask)) >> (g * 8)) & 0xFFu;
        const uint32_t state = (uint32_t)(tag & TAG_STATE_MASK);
        unsigned long long* tagp = reinterpret_cast<unsigned long long*>(&t.ident[slot * 8 + 2]) + 1;
        // Claim either an empty slot, or the base of a flow that so far exists only through feature
        // samples (no TAG_HAS_BASE: its first base record is adopted whole, pkg/flow/account.go:95).
        const bool base_claim = state == (uint32_t)TAG_PUBLISHED && !(tag & TAG_HAS_BASE) && (eqb & 0x07u) == 0x07u;
        uint32_t won = 0;
        if (!done && (state == 0 || base_claim) && j == 2) {
            const unsigned long long expect = state == 0 ? 0ull : (unsigned long long)tag;
            const unsigned long long want = (epoch << TAG_EPOCH_SHIFT) | TAG_HAS_BASE | TAG_CLAIMED;
            won = atomicCAS(tagp, expect, want) == expect ? (state == 0 ? 1u : 2u) : 0u;
        }
        won = __shfl_sync(0xFFFFFFFFu, won, g * 8 + 2);
        if (won) {
            uint4 v = and4(rchunk, cmask);
            if (j == 3) {                                       // start mirror around eth_protocol
                const uint64_t m48 = ins_ns >> 16;
                v.x = (uint32_t)m48; v.y |= (uint32_t)(m48 >> 32) << 16;
            }
            if (j == 2) *reinterpret_cast<uint2*>(&t.ident[slot * 8 + 2]) = make_uint2(v.x, v.y);   // key tail only
            else st_cg_u4(&t.ident[slot * 8 + j], v);
            __threadfence();
        }
        __syncwarp();
        bool hit = false;
        if (won) {
            if (j == 2) {
                const unsigned long long pub = (epoch << TAG_EPOCH_SHIFT) | TAG_HAS_BASE | TAG_PUBLISHED |
                                               (cta_dirty ? TAG_DIRTY : 0ull);
                *reinterpret_cast<volatile unsigned long long*>(tagp) = pub;
                if (won == 1u) {                               // a base claim does not add a flow
                    my_inserts++;
                    red_or_u32(&t.occ[slot >> 5], 1u << (slot & 31));
                }
                if (cta_dirty) *any_dirty = 1;
            }
            hit = true;
        } else if (!done && state == (uint32_t)TAG_PUBLISHED && !base_claim) {
            const bool born_now = (tag >> TAG_EPOCH_SHIFT) == epoch;
            if (born_now && reload_slot != slot) {
                // published during this launch: the chunks read together with the tag may predate
                // it.  Re-read the line once, ordered after the tag observation.
                reload_slot = slot;
                __threadfence();
            } else if ((eqb & 0x07u) == 0x07u) {
                hit = true;
                const bool desc_eq = (eqb & 0xF8u) == 0xF8u;
                if ((!desc_eq || cta_dirty) && j == 2) {
                    if (!(tag & TAG_DIRTY)) atomicOr(tagp, (unsigned long long)TAG_DIRTY);
                    *any_dirty = 1;
                }
            } else {
                slot = (slot + 1) & t.mask;
                if (++nprobe > kProbeLimit) done = true;         // physically full: result stays kResSpill
            }
        }
        // CLAIMED by someone else, or lost the CAS: retry the same slot next iteration
        if (hit) { result = (uint32_t)slot; done = true; }
        if (__all_sync(0xFFFFFFFFu, done)) break;
    }
    return result;
}

// kProf: per-warp cycle counters per phase (FA_PHASE_PROFILE=1), summed into prof[0..7].
#define FA_PROF_MARK(i) do { if (kProf) { const long long now_ = clock64(); pacc[i] += now_ - pt; pt = now_; } } while (0)

template <bool kSketch, bool kProf, bool kDevN>
__global__ void __launch_bounds__(kCtaThreads, 1)
aggregate_kernel(const uint4* __restrict__ recs, uint32_t n, Table t, uint64_t epoch, Counters* ctr,
                 uint32_t* __restrict__ spill_idx, SketchParams sk, unsigned long long* prof, uint32_t opt) {
    FA_DYN_SMEM(smem_raw);
    AggSmem& cs = *reinterpret_cast<AggSmem*>(smem_raw);
    const int team = threadIdx.x / kTile;
    const int tid = threadIdx.x & (kTile - 1), lane = tid & 31, warp = tid >> 5;     // within the team
    TeamSmem& s = cs.team[team];
    TeamCtl& tc = cs.ctl[team];
    // Tile schedule: every team starts on tile blockIdx.x * kTeams + team; each later tile is claimed from the launch's
    // counter (gridDim.x * kTeams + the count of earlier claims), so a team that finishes early takes the next tile
    // instead of the slowest teams' tails being fixed by a static stride.
    const uint32_t tile0 = blockIdx.x * kTeams + team;
    const uint32_t claim_base = gridDim.x * kTeams;
    unsigned int* const tile_claims = k1_tile_claims(ctr);
    const bool use_cache = (opt & 2u) == 0;

    if (threadIdx.x == 0) { cs.n_insert = 0; cs.n_spill = 0; cs.any_dirty = 0; }
    if (threadIdx.x < kHotEntries) { cs.hot[threadIdx.x].state = 0; cs.hot_tag[threadIdx.x] = 0; }
    if (tid == 0) {
        mbar_init(&tc.full_bar, 1);
        fence_barrier_init();
        tc.nrep = 0; tc.done = 0;
    }
    s.rep[tid] = kRepEmpty; s.rep[tid + kTile] = kRepEmpty;
    *reinterpret_cast<uint4*>(&s.acc[tid][0]) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(&s.acc[tid][4]) = make_uint4(0, 0, 0, 0);
    s.tdirty[tid] = 0;
    pdl_wait();                                                    // the kernels before this launch have completed
    if (kDevN) n = min(n, (uint32_t)ctr->launch_n);            // size known on the device only (multi-GPU receive side)
    const uint32_t n_tiles = (n + kTile - 1) / kTile;
    __syncthreads();
    if (tid == 0 && tile0 < n_tiles) issue_tile_load(s, tc, recs, n, tile0);

    const int g = lane >> 3;                  // flow group inside the warp (4 groups of 8 lanes)
    const int j = lane & 7;                   // 16-byte chunk of the identity line handled by this lane
    const uint4 cmask = chunk_mask(j);
    const int rc = rec_chunk_of_line_chunk(j);
    const uint32_t tmask = (uint32_t)t.mask;
    const uint32_t lt_mask = (1u << lane) - 1u;
    uint32_t my_inserts = 0, my_spills = 0;
    const uint4* T = s.tile;
    long long pacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long pt = kProf ? clock64() : 0;
    uint32_t c_cached = 0, c_reps = 0, c_slow = 0, c_install = 0, c_collide = 0, c_p1fast = 0, c_unsettled = 0;   // kProf only

    uint32_t tile_idx = tile0;
    for (uint32_t it = 0; tile_idx < n_tiles; ++it) {               // `it` counts the team's own tiles: mbarrier parity
        const uint32_t first = tile_idx * kTile;
        const uint32_t cnt = min((uint32_t)kTile, n - first);
        // claim the team's next tile now, so that the atomic's round trip overlaps this tile's E phase; it is published
        // in next[it & 1] before S1 and read by the warp that re-arms the TMA (after S1) and by every thread after S2.
        // The other word of the pair is still being read by threads that have not left the previous iteration.
        uint32_t claimed = 0;
        if (tid == 0) claimed = claim_base + atomicAdd(tile_claims, 1u);
        mbar_wait(&tc.full_bar, it & 1u);
        FA_PROF_MARK(0);                                           // waiting for the tile

        // ------------------------------------------------------ E: hash, cache / elect, fold duplicates
        {
            const bool valid = (uint32_t)tid < cnt;
            bool is_rep = valid;
            if (valid) {
                const uint4* R = T + tid * kRecChunks;
                const uint4 r0 = R[0], r1 = R[1], r2 = R[2];
                const uint64_t h = slot_hash(key_premix(u64_of(r0.x, r0.y), u64_of(r0.z, r0.w), u64_of(r1.x, r1.y),
                                                        u64_of(r1.z, r1.w), u64_of(r2.x, r2.y)));
                s.hs[tid] = (uint32_t)h;
                // ---- hot-flow cache: an exact 114-byte match folds the record on-chip, no table traffic
                const uint32_t cset = hot_set((uint32_t)h);
                uint32_t cidx = kHotEntries;                              // the way of the set that holds this hash, if any
                for (uint32_t m = hot_ways_with(*reinterpret_cast<const uint4*>(&cs.hot_tag[cset * kHotWays]), hot_tag_of((uint32_t)h)); m; m &= m - 1u) {
                    const uint32_t i = cset * kHotWays + (uint32_t)__ffs((int)m) - 1u;
                    if (*reinterpret_cast<volatile uint32_t*>(&cs.hot[i].state) == 2u && cs.hot[i].hash == (uint32_t)h) { cidx = i; break; }
                }
                if (use_cache && cidx < (uint32_t)kHotEntries) {
                    HotEntry& ce = cs.hot[cidx];
                    const uint4 r3 = R[3], r4 = R[4];
                    bool same = eq4_masked(ce.line[0], r0, chunk_mask(0)) && eq4_masked(ce.line[1], r1, chunk_mask(1)) &&
                                eq4_masked(ce.line[2], r2, chunk_mask(2)) && eq4_masked(ce.line[3], r4, chunk_mask(3));
#pragma unroll
                    for (int c = 5; c < 9; c++) same = same && eq4_masked(ce.line[c - 1], R[c], chunk_mask(c - 1));
                    const uint64_t v_start = u64_of(r2.z, r2.w), v_end = u64_of(r3.x, r3.y);
                    const uint64_t v_ns = 0ull - v_start;
                    same = same && (v_start == 0 || (uint32_t)(v_ns >> 32) == ce.ns_hi) &&
                           (v_end == 0 || (uint32_t)(v_end >> 32) == ce.end_hi);
                    if (same) {
                        is_rep = false;
                        FA_EMUL_COUNT(2, 1);
                        if (kProf) c_cached++;
                        uint32_t* A = ce.acc;
                        const uint32_t b_lo = r3.z, b_hi = r3.w;
                        const uint32_t prev = atomicAdd(&A[0], b_lo);
                        const uint32_t hi_add = b_hi + ((prev + b_lo) < prev ? 1u : 0u);
                        if (hi_add) atomicAdd(&A[1], hi_add);
                        const uint32_t p_prev = atomicAdd(&A[2], r4.x);
                        if (kSketch && p_prev + r4.x < p_prev) atomicAdd(&A[7], 1u);          // count-min carry
                        const uint32_t fl = r4.y >> 16;
                        if (fl & ~A[3]) atomicOr(&A[3], fl);
                        if (v_start && (uint32_t)v_ns > A[4]) atomicMax(&A[4], (uint32_t)v_ns);
                        if (v_end && (uint32_t)v_end > A[5]) atomicMax(&A[5], (uint32_t)v_end);
                    }
                }
                if (is_rep) {
                    // election: the slot holds (23 hash bits << 8 | tile index), so a slot taken by another key is
                    // walked past without touching the tile; the fold of a duplicate runs after the loop, once per
                    // warp, instead of inside it at whatever iteration each lane found its representative
                    uint32_t rs = (uint32_t)(h >> 40) & (kRepSlots - 1);
                    const uint32_t mine = (((uint32_t)(h >> 16) & 0x7FFFFFu) << 8) | (uint32_t)tid;
                    uint32_t dup_of = kRepEmpty;
                    {   // own values go into the accumulators BEFORE the record can be elected: whoever finds it in the
                        // election set adds to initialised words, and the reduce step no longer needs the tile
                        const uint4 r3 = R[3], r4 = R[4];
                        const uint64_t v_ns = 0ull - u64_of(r2.z, r2.w);
                        *reinterpret_cast<uint4*>(&s.acc[tid][0]) = make_uint4(r3.z, r3.w, r4.x, r4.y >> 16);   // bytes | packets | flags (dups << 16)
                        *reinterpret_cast<uint4*>(&s.acc[tid][4]) = make_uint4((uint32_t)v_ns, r3.x, (uint32_t)(v_ns >> 32), r3.y);   // ns lo, end lo, ns hi, end hi
                        s.tdirty[tid] = 0;
                        __threadfence_block();
                    }
                    for (;;) {
                        const uint32_t old = atomicCAS(&s.rep[rs], kRepEmpty, mine);
                        if (old == kRepEmpty) break;
                        if (((old ^ mine) >> 8) == 0u) {
                            const uint4* O = T + (old & 0xFFu) * kRecChunks;
                            if (eq4_masked(O[2], r2, chunk_mask(2)) && eq4_masked(O[0], r0, chunk_mask(0)) &&
                                eq4_masked(O[1], r1, chunk_mask(1))) { dup_of = old & 0xFFu; break; }
                        }
                        rs = (rs + 1) & (kRepSlots - 1);
                    }
                    if (dup_of != kRepEmpty) {
                        // Same key.  Fold into that representative with 32-bit shared atomics when the high words of
                        // the timestamps agree (the common case); otherwise go to the table on our own.
                        const uint4* O = T + dup_of * kRecChunks;
                        const uint4 r3 = R[3], r4 = R[4], o2 = O[2], o3 = O[3];
                        const uint64_t v_start = u64_of(r2.z, r2.w), v_end = u64_of(r3.x, r3.y);
                        const uint64_t v_ns = 0ull - v_start;
                        const uint64_t o_ns = 0ull - u64_of(o2.z, o2.w), o_end = u64_of(o3.x, o3.y);
                        const bool ok = (v_start == 0 || (uint32_t)(v_ns >> 32) == (uint32_t)(o_ns >> 32)) &&
                                        (v_end == 0 || (uint32_t)(v_end >> 32) == (uint32_t)(o_end >> 32));
                        if (ok) {
                            is_rep = false;
                            uint32_t* A = s.acc[dup_of];
                            const uint32_t b_lo = r3.z, b_hi = r3.w;
                            const uint32_t prev = atomicAdd(&A[0], b_lo);
                            const uint32_t hi_add = b_hi + ((prev + b_lo) < prev ? 1u : 0u);
                            if (hi_add) atomicAdd(&A[1], hi_add);
                            const uint32_t p_prev = atomicAdd(&A[2], r4.x);
                            if (kSketch && p_prev + r4.x < p_prev) atomicAdd(&A[3], 1u << 24);   // count-min carry
                            const uint32_t fl = r4.y >> 16;
                            if (fl) atomicOr(&A[3], fl);
                            if (v_start) atomicMax(&A[4], (uint32_t)v_ns);
                            if (v_end) atomicMax(&A[5], (uint32_t)v_end);
                            atomicAdd(&A[3], 1u << 16);              // duplicates seen (above the 16 flag bits): cache candidacy
                            uint32_t d = diff4_masked(O[4], r4, chunk_mask(3));      // exact 74-byte descriptor compare
#pragma unroll
                            for (int c = 5; c < 9; c++) d |= diff4_masked(O[c], R[c], chunk_mask(c - 1));
                            if (d) s.tdirty[dup_of] = 1;
                        }
                    }
                }
            }
            // team-wide list of representatives, so that every warp probes an equal share
            const uint32_t pending = __ballot_sync(0xFFFFFFFFu, is_rep);
            uint32_t lbase = 0;
            if (lane == 0 && pending) lbase = atomicAdd(&tc.nrep, (uint32_t)__popc(pending));
            lbase = __shfl_sync(0xFFFFFFFFu, lbase, 0);
            if (is_rep) s.glist[lbase + __popc(pending & lt_mask)] = (RepIdx)tid;
        }
        if (tid == 0) tc.next[it & 1u] = claimed;
        FA_PROF_MARK(1);                                           // E phase
        team_sync(team);                                           // S1: folds, hashes and the list are complete
        FA_PROF_MARK(2);                                           // S1 wait

        const uint32_t nrep_total = tc.nrep;
        s.rep[tid] = kRepEmpty; s.rep[tid + kTile] = kRepEmpty;   // nobody reads the election table after S1

        // ------------------------------------------------------ probe: the list is split evenly over the team's warps;
        // a warp walks its share in rounds of 4 flows (8 lanes per flow) with four identity-line loads in flight at all
        // times: the load of round r + 4 is issued as soon as round r has been compared.  Flows whose home slot holds
        // another settled flow are collected and probed one slot further in a second, compact pass (rounds of 4 again)
        // instead of re-running every round; whatever is left goes to the general loop.
        {
            constexpr uint32_t kWarps = kTile / 32;
            const uint32_t per = ((nrep_total + kWarps - 1) / kWarps + 3u) & ~3u;  // <= 32, whole rounds: same longest warp, fewer half-empty rounds
            const uint32_t w0 = min(nrep_total, (uint32_t)warp * per), w1 = min(nrep_total, w0 + per);
            RepIdx* const wl = s.slow[warp];                                       // general-loop flows from the front, second-pass flows from the back
            uint32_t nslow = 0, ncoll = 0;
#pragma unroll 1
            for (int pass = 0; pass < 2; pass++) {
                __syncwarp();
                const RepIdx* const src = pass == 0 ? &s.glist[w0] : &wl[32u - ncoll];
                const uint32_t cnt = pass == 0 ? w1 - w0 : ncoll;
                const uint32_t nrounds = (cnt + 3u) >> 2;
                uint4 line[4];
                uint32_t ridx[4], slot[4];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    ridx[q] = 0u; slot[q] = 0u;
                    line[q] = make_uint4(0, 0, 0, 0);
                    if ((uint32_t)q < nrounds) {                                   // warp-uniform
                        const uint32_t k = (uint32_t)q * 4u + g;
                        const bool a = k < cnt;
                        if (a) ridx[q] = (uint32_t)src[k];
                        slot[q] = (s.hs[ridx[q]] + (uint32_t)pass) & tmask;
                        if (a) line[q] = ld_cg_u4(&t.ident[(size_t)slot[q] * 8 + j]);
                    }
                }
#pragma unroll 1
                for (uint32_t base = 0; base < nrounds; base += 4) {
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const uint32_t round = base + q;
                        if (round >= nrounds) break;                               // warp-uniform
                        const bool act = round * 4u + g < cnt;
                        const uint4 rchunk = T[ridx[q] * kRecChunks + rc];
                        bool eq = eq4_masked(line[q], rchunk, cmask);
                        const uint64_t tag = u64_of(line[q].z, line[q].w);         // meaningful in lane j == 2 only
                        bool settled = false;
                        if (j == 2) {
                            settled = (tag & (TAG_STATE_MASK | TAG_HAS_BASE)) == (TAG_PUBLISHED | TAG_HAS_BASE) &&
                                      (tag >> TAG_EPOCH_SHIFT) != epoch;
                            eq = eq && settled;
                        }
                        const uint32_t eqb = (__ballot_sync(0xFFFFFFFFu, eq) >> (g * 8)) & 0xFFu;
                        const bool fast = act && (eqb & 0x07u) == 0x07u;           // settled flow, key matches
                        uint32_t* const rw = reinterpret_cast<uint32_t*>(&s.res4[ridx[q]]);
                        if (fast && j == 0) rw[0] = slot[q];
                        if (fast && j == 3) { rw[1] = line[q].x; rw[2] = line[q].y; }           // start mirror (eth_protocol in between); rw + 1 is only 4-byte aligned
                        if (fast && j == 2) {
                            rw[3] = (uint32_t)(tag >> TAG_FLAGS_SHIFT);            // flag bits the hot line already holds (low 16)
                            if ((eqb & 0xF8u) != 0xF8u || s.tdirty[ridx[q]] != 0) {
                                unsigned long long* tagp = reinterpret_cast<unsigned long long*>(&t.ident[(size_t)slot[q] * 8 + 2]) + 1;
                                if (!(tag & TAG_DIRTY)) atomicOr(tagp, (unsigned long long)TAG_DIRTY);
                                cs.any_dirty = 1;
                            }
                        }
                        const uint32_t nfb = __ballot_sync(0xFFFFFFFFu, act && !fast && j == 0);
                        if (nfb) {                                                 // some flow of the round is not settled at this slot (uncommon)
                            const bool gsettled = (__ballot_sync(0xFFFFFFFFu, settled) >> (g * 8 + 2)) & 1u;
                            const bool collide = act && !fast && gsettled && pass == 0;   // other settled flow: look one slot on
                            const bool to_slow = act && !fast && !collide;
                            if (kProf && j == 0) {
                                if (collide) c_collide++;
                                if (act && !fast && !gsettled) c_unsettled++;
                            }
                            const uint32_t collb = __ballot_sync(0xFFFFFFFFu, collide && j == 0);
                            const uint32_t slowb = nfb & ~collb;
                            if (collide && j == 0) wl[31u - (ncoll + __popc(collb & lt_mask))] = (RepIdx)ridx[q];
                            ncoll += __popc(collb);
                            if (to_slow && j == 0) wl[nslow + __popc(slowb & lt_mask)] = (RepIdx)ridx[q];
                            nslow += __popc(slowb);
                        }
                        if (kProf && j == 0 && fast && pass == 1) c_p1fast++;
                        if (round + 4u < nrounds) {                                // this register set's next flow: round + 4
                            const uint32_t k = (round + 4u) * 4u + g;
                            const bool a = k < cnt;
                            ridx[q] = a ? (uint32_t)src[k] : 0u;
                            slot[q] = (s.hs[ridx[q]] + (uint32_t)pass) & tmask;
                            line[q] = make_uint4(0, 0, 0, 0);
                            if (a) line[q] = ld_cg_u4(&t.ident[(size_t)slot[q] * 8 + j]);
                        }
                    }
                }
                if (ncoll == 0u) break;
            }
            __syncwarp();
            if (lane == 0) { FA_EMUL_COUNT(0, w1 - w0); FA_EMUL_COUNT(1, nslow); }
            if (kProf && lane == 0) { c_reps += w1 - w0; c_slow += nslow; }
            FA_PROF_MARK(3);                                       // pipelined probe passes
            for (uint32_t base = 0; base < nslow; base += 4) {     // inserts, long collision chains, in-flight publishes
                const uint32_t k = base + g;
                const bool act = k < nslow;
                const uint32_t ri = act ? wl[k] : 0;
                const uint4 rchunk = T[ri * kRecChunks + rc];
                const uint4 c2 = T[ri * kRecChunks + 2];
                const uint64_t own_ns = 0ull - u64_of(c2.z, c2.w);
                const uint64_t dup_ns = u64_of(s.acc[ri][4], (uint32_t)(own_ns >> 32));
                const uint32_t got = probe_general(t, epoch, act, s.hs[ri] & tmask, rchunk, s.tdirty[ri] != 0,
                                                   dup_ns > own_ns ? dup_ns : own_ns, g, j, cmask, my_inserts, &cs.any_dirty);
                if (act && j == 0) s.res4[ri] = make_uint4(got, 0u, 0u, 0u);   // mirror / seen flags unknown: issue every reduction
            }
            __syncwarp();
            FA_PROF_MARK(4);                                       // general probe loop
            if (lane == 0) {                                       // the warp is done with the tile: the last one out re-arms it
                __threadfence_block();
                if (atomicAdd(&tc.done, 1u) == kWarps - 1u) {
                    tc.done = 0;
                    tc.nrep = 0;                                   // every warp has read the list length; reset it before the
                                                                   // next tile can arrive (its E phase starts right after S2)
                    const uint32_t nt = tc.next[it & 1u];
                    if (!kSketch && nt < n_tiles) { fence_proxy_async(); issue_tile_load(s, tc, recs, n, nt); }
                }
            }

            // -------------------------------------------------- one lane per flow: totals, then the reductions
            if (w0 + lane < w1) {
                const uint32_t my_ridx = s.glist[w0 + lane];
                const uint4 rr = s.res4[my_ridx];
                const uint32_t my_slot = rr.x;
                const uint64_t floor_ns = u64_of(rr.y, rr.z >> 16) << 16;                      // <= hot.nstart, always
                const uint32_t seen = rr.w & 0xFFFFu;
                const uint4* R = T + my_ridx * kRecChunks;          // (kSketch only: the tile stays until S2)
                const uint4 a0 = *reinterpret_cast<const uint4*>(&s.acc[my_ridx][0]);
                const uint4 a1 = *reinterpret_cast<const uint4*>(&s.acc[my_ridx][4]);
                const uint64_t t_bytes = u64_of(a0.x, a0.y);
                const uint32_t t_packets = a0.z;
                const uint32_t t_flags = a0.w & 0xFFFFu, n_dups = kSketch ? (a0.w >> 16) & 0xFFu : a0.w >> 16;
                const uint64_t t_ns = u64_of(a1.x, a1.z), t_end = u64_of(a1.y, a1.w);
                const uint64_t v_ns = t_ns, v_end = t_end;           // the cache entry's windows: high words only
                // a flow that shows up several times in one tile is hot: give it a way of its set if one is free and it
                // has none yet (an entry another team is filling right now is not seen: the flow then holds two ways,
                // which costs a way and nothing else, every live entry is flushed)
                if (use_cache && n_dups >= kHotMinDups && my_slot != kResSpill) {
                    const uint32_t hh = s.hs[my_ridx], iset = hot_set(hh);
                    const uint4 tags = *reinterpret_cast<const uint4*>(&cs.hot_tag[iset * kHotWays]);
                    bool cached = false;
                    for (uint32_t m = hot_ways_with(tags, hot_tag_of(hh)); m; m &= m - 1u)
                        cached = cached || cs.hot[iset * kHotWays + (uint32_t)__ffs((int)m) - 1u].hash == hh;
                    uint32_t iidx = kHotEntries;
                    for (uint32_t m = cached ? 0u : hot_ways_with(tags, 0u); m; m &= m - 1u) {
                        const uint32_t i = iset * kHotWays + (uint32_t)__ffs((int)m) - 1u;
                        if (atomicCAS(&cs.hot[i].state, 0u, 1u) == 0u) { iidx = i; break; }
                    }
                    if (iidx < (uint32_t)kHotEntries) {
                        HotEntry& ce = cs.hot[iidx];
#pragma unroll
                        for (int c = 0; c < 8; c++) ce.line[c] = ld_cg_u4(&t.ident[(size_t)my_slot * 8 + c]);
                        *reinterpret_cast<uint4*>(&ce.acc[0]) = make_uint4(0, 0, 0, 0);
                        *reinterpret_cast<uint4*>(&ce.acc[4]) = make_uint4(0, 0, 0, 0);
                        ce.hash = hh; ce.slot = my_slot;
                        ce.ns_hi = (uint32_t)(v_ns >> 32); ce.end_hi = (uint32_t)(v_end >> 32);
                        __threadfence_block();
                        *reinterpret_cast<volatile uint32_t*>(&ce.state) = 2u;
                        __threadfence_block();
                        *reinterpret_cast<volatile uint16_t*>(&cs.hot_tag[iidx]) = (uint16_t)hot_tag_of(hh);
                        if (kProf) c_install++;
                    }
                }
                if (kSketch) {
                    const uint4 r0 = R[0], r1 = R[1], k2 = R[2];
                    sketch_update(sk, key_premix(u64_of(r0.x, r0.y), u64_of(r0.z, r0.w), u64_of(r1.x, r1.y),
                                                 u64_of(r1.z, r1.w), u64_of(k2.x, k2.y)), u64_of(t_packets, a0.w >> 24));
                }
                if (my_slot != kResSpill) {
                    reduce_to_hot(t, my_slot, t_bytes, t_packets, t_ns, t_end, t_flags, floor_ns, seen);
                } else {                                           // table physically full (FA_F_NO_FULL_CUT mis-sizing): counted
                    my_spills++;                                   // in fa_stats.spills, like HASHMAP_FAIL_CREATE_FLOW (flows.c:285)
                }
            }
            FA_PROF_MARK(5);                                       // totals + reductions
        }
        team_sync(team);                                           // S2: nobody reads the tile buffer any more
        FA_PROF_MARK(6);                                           // S2 wait
        tile_idx = tc.next[it & 1u];
        if (tid == 0) {
            if (kSketch) {                                         // the sketch update reads the keys in the reduce step: re-arm here
                if (tile_idx < n_tiles) { fence_proxy_async(); issue_tile_load(s, tc, recs, n, tile_idx); }
            }
        }
        FA_PROF_MARK(7);                                           // reductions
    }
    if (kProf) {
        c_cached = __reduce_add_sync(0xFFFFFFFFu, c_cached);
        c_install = __reduce_add_sync(0xFFFFFFFFu, c_install);
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < 8; i++) atomicAdd(&prof[i], (unsigned long long)pacc[i]);
            atomicAdd(&prof[8], (unsigned long long)c_cached);
            atomicAdd(&prof[9], (unsigned long long)c_reps);
            atomicAdd(&prof[10], (unsigned long long)c_slow);
            atomicAdd(&prof[11], (unsigned long long)c_install);
        }
        c_collide = __reduce_add_sync(0xFFFFFFFFu, c_collide);
        c_p1fast = __reduce_add_sync(0xFFFFFFFFu, c_p1fast);
        c_unsettled = __reduce_add_sync(0xFFFFFFFFu, c_unsettled);
        if (lane == 0) {
            atomicAdd(&prof[12], (unsigned long long)c_collide);
            atomicAdd(&prof[13], (unsigned long long)c_p1fast);
            atomicAdd(&prof[14], (unsigned long long)c_unsettled);
        }
    }

    // ---------------------------------------------------------- counters + cache flush
    my_inserts = __reduce_add_sync(0xFFFFFFFFu, my_inserts);
    my_spills = __reduce_add_sync(0xFFFFFFFFu, my_spills);
    if (lane == 0) {
        if (my_inserts) atomicAdd(&cs.n_insert, my_inserts);
        if (my_spills) atomicAdd(&cs.n_spill, my_spills);
    }
    __syncthreads();                                               // every team is out of tiles
    if (threadIdx.x < kHotEntries) {
        const HotEntry& ce = cs.hot[threadIdx.x];
        if (ce.state == 2u) {
            const uint32_t* A = ce.acc;
            const uint64_t tag = u64_of(ce.line[2].z, ce.line[2].w);
            const uint64_t floor_ns = u64_of(ce.line[3].x, ce.line[3].y >> 16) << 16;
            // ns / end windows: an untouched window (0) reads as a value no larger than the installing
            // record's own, which the table already holds -> a harmless no-op max.
            reduce_to_hot(t, ce.slot, u64_of(A[0], A[1]), A[2], u64_of(A[4], ce.ns_hi), u64_of(A[5], ce.end_hi), A[3],
                          floor_ns, (uint32_t)(tag >> TAG_FLAGS_SHIFT) & 0xFFFFu);
            if (kSketch) {
                const uint4 k0 = ce.line[0], k1 = ce.line[1], k2 = ce.line[2];
                sketch_update(sk, key_premix(u64_of(k0.x, k0.y), u64_of(k0.z, k0.w), u64_of(k1.x, k1.y),
                                             u64_of(k1.z, k1.w), u64_of(k2.x, k2.y)), u64_of(A[2], A[7]));
            }
        }
    }
    if (threadIdx.x == 0) {
        if (cs.n_insert) atomicAdd(&ctr->live, (unsigned long long)cs.n_insert);
        if (cs.n_spill) atomicAdd(&ctr->spills, (unsigned long long)cs.n_spill);
        if (cs.any_dirty) *reinterpret_cast<volatile unsigned long long*>(&ctr->dirty) = 1ull;
        // every team of this CTA has made its last claim and its inserts are counted: the last CTA out zeroes the
        // claim counter for the next launch and hands the live-flow count to the host
        __threadfence();
        unsigned int* const ticket = k1_exit_ticket(ctr);
        if (atomicAdd(ticket, 1u) == gridDim.x - 1u) {
            __threadfence();
            *tile_claims = 0u;
            *ticket = 0u;
            if (ctr->live_ring) {
                const unsigned long long seq = ctr->live_seq;
                ctr->live_seq = seq + 1ull;
                const unsigned long long live = *reinterpret_cast<volatile unsigned long long*>(&ctr->live);
                *reinterpret_cast<volatile unsigned long long*>(&ctr->live_ring[seq % kLiveRing]) = live;
                __threadfence_system();
            }
        }
    }
}

// ------------------------------------------------------------------------------------
// Ordered re-fold of flows flagged TAG_DIRTY (rare path; both kernels exit at once when
// nothing was flagged).  fixup_scan: one thread per record finds its flow and, if dirty,
// reduces min/max record indices into the flow's scratch entry.  fixup_apply: one thread
// per scratch entry gathers the fields from the records those indices name.
// ------------------------------------------------------------------------------------
__device__ __forceinline__ bool key_equal_line(const uint4* line, uint4 k0, uint4 k1, uint4 k2) {
    uint4 l0 = ld_cg_u4(line), l1 = ld_cg_u4(line + 1), l2 = ld_cg_u4(line + 2);
    return eq4_masked(l0, k0, chunk_mask(0)) && eq4_masked(l1, k1, chunk_mask(1)) && eq4_masked(l2, k2, chunk_mask(2));
}

__device__ __forceinline__ uint32_t scratch_home(uint64_t slot, uint32_t smask) {
    return (uint32_t)((slot * 0x9E3779B97F4A7C15ull) >> 32) & smask;
}

__global__ void fixup_scan_kernel(const uint4* __restrict__ recs, uint32_t n, Table t, Counters* ctr, FixupScratch* scratch,
                                  uint32_t smask, uint32_t opt) {
    pdl_wait();
    if (*reinterpret_cast<volatile unsigned long long*>(&ctr->dirty) == 0ull) return;
    if (opt & 16u) n = min(n, (uint32_t)ctr->launch_n);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4* R = recs + (size_t)i * kRecChunks;
        const uint4 k0 = R[0], k1 = R[1], k2 = R[2];
        const uint64_t h = slot_hash(key_premix(u64_of(k0.x, k0.y), u64_of(k0.z, k0.w), u64_of(k1.x, k1.y),
                                                u64_of(k1.z, k1.w), u64_of(k2.x, k2.y)));
        uint64_t slot = h & t.mask;
        bool found = false;
        unsigned long long tag = 0;
        for (uint32_t p = 0; p <= kProbeLimit; p++) {
            tag = ld_cg_u64(reinterpret_cast<const unsigned long long*>(&t.ident[slot * 8 + 2]) + 1);
            if ((tag & TAG_STATE_MASK) == 0) break;
            if (key_equal_line(&t.ident[slot * 8], k0, k1, k2)) { found = true; break; }
            slot = (slot + 1) & t.mask;
        }
        if (!found || !(tag & TAG_DIRTY)) continue;
        uint32_t si = scratch_home(slot, smask);
        for (;;) {                                                   // find-or-insert the flow's scratch entry
            const unsigned long long k = atomicCAS(&scratch[si].key, 0ull, slot + 1);
            if (k == 0ull || k == slot + 1) break;
            si = (si + 1) & smask;
        }
        FixupScratch* sc = &scratch[si];
        const uint4 r4 = R[4], r5 = R[5], r6 = R[6];
        atomicMax(&sc->nfirst, ~i);
        if (r4.y & 0xFFFFu) atomicMax(&sc->eth, i + 1);
        if ((r6.x >> 16) & 0xFFu) atomicMax(&sc->dscp, i + 1);
        if (r5.w) atomicMax(&sc->samp, i + 1);
        if (r4.z | (r4.w & 0xFFFFu)) atomicMax(&sc->nsmac, ~i);
        if ((r4.w >> 16) | r5.x) atomicMax(&sc->ndmac, ~i);
    }
}

__global__ void fixup_apply_kernel(const uint4* __restrict__ recs, Table t, uint64_t epoch, Counters* ctr,
                                   FixupScratch* scratch, uint32_t scratch_slots, unsigned int* ticket) {
    pdl_wait();
    if (*reinterpret_cast<volatile unsigned long long*>(&ctr->dirty) == 0ull) return;
    uint32_t fixed = 0;
    for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < scratch_slots; a += gridDim.x * blockDim.x) {
        const FixupScratch sc = scratch[a];
        if (sc.key == 0ull) continue;
        scratch[a] = FixupScratch{0ull, 0u, 0u, 0u, 0u, 0u, 0u};
        const uint64_t slot = sc.key - 1;
        uint4* L = &t.ident[slot * 8];
        unsigned long long* tagp = reinterpret_cast<unsigned long long*>(&L[2]) + 1;
        const unsigned long long tag = *tagp;
        const bool is_new = (tag >> TAG_EPOCH_SHIFT) == epoch;
        // current descriptor state: line chunks 3..7 <-> record chunks 4..8
        uint4 d3 = L[3], d4 = L[4], d5 = L[5], d6 = L[6], d7 = L[7];
        const uint32_t mir_lo = d3.x, mir_hi = d3.y & 0xFFFF0000u;    // immutable start mirror stays
        if (is_new) {                                      // state = the flow's first record, whole (account.go:95)
            const uint4* F = recs + (size_t)(~sc.nfirst) * kRecChunks;
            d3 = and4(F[4], chunk_mask(3)); d4 = F[5]; d5 = and4(F[6], chunk_mask(5)); d6 = F[7]; d7 = and4(F[8], chunk_mask(7));
        }
        // eth_protocol / dscp / sampling: last non-zero in stream order (flow_content.go:45-47,54-59)
        if (sc.eth)  { const uint4 x = recs[(size_t)(sc.eth - 1) * kRecChunks + 4]; d3.y = x.y & 0xFFFFu; }
        if (sc.dscp) { const uint4 x = recs[(size_t)(sc.dscp - 1) * kRecChunks + 6]; d5.x = (d5.x & 0xFF00FFFFu) | (x.x & 0x00FF0000u); }
        if (sc.samp) { const uint4 x = recs[(size_t)(sc.samp - 1) * kRecChunks + 5]; d4.w = x.w; }
        // MACs: first non-zero in stream order, only while still all-zero (flow_content.go:48-53)
        if ((d3.z | (d3.w & 0xFFFFu)) == 0u && sc.nsmac != 0u) {
            const uint4 x = recs[(size_t)(~sc.nsmac) * kRecChunks + 4];
            d3.z = x.z; d3.w = (d3.w & 0xFFFF0000u) | (x.w & 0xFFFFu);
        }
        if (((d3.w >> 16) | d4.x) == 0u && sc.ndmac != 0u) {
            const uint4 x4 = recs[(size_t)(~sc.ndmac) * kRecChunks + 4], x5 = recs[(size_t)(~sc.ndmac) * kRecChunks + 5];
            d3.w = (d3.w & 0xFFFFu) | (x4.w & 0xFFFF0000u); d4.x = x5.x;
        }
        d3.x = mir_lo; d3.y = (d3.y & 0xFFFFu) | mir_hi;
        L[3] = d3; L[4] = d4; L[5] = d5; L[6] = d6; L[7] = d7;
        atomicAnd(tagp, ~(unsigned long long)TAG_DIRTY);
        fixed++;
    }
    if (fixed) atomicAdd(&ctr->fixups_total, (unsigned long long)fixed);
    // last CTA out resets the per-launch state
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
            *ticket = 0u;
            ctr->dirty = 0ull;
            __threadfence();
        }
    }
}

#ifndef FA_HOST_EMUL
int launch_aggregate(const AggLaunch& a, cudaStream_t st) {
    if (a.n == 0) return 0;
    static bool attr_done_dev[64] = {};                // function attributes are per device
    int dev = 0;
    cudaGetDevice(&dev);
    bool& attr_done = attr_done_dev[dev & 63];
    const int smem = (int)sizeof(AggSmem);
    if (!attr_done) {
        cudaFuncSetAttribute(aggregate_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(aggregate_kernel<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(aggregate_kernel<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(aggregate_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(aggregate_kernel<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        attr_done = true;
    }
    const uint32_t n_tiles = (a.n + kTile - 1) / kTile;
    const int grid = (int)min((uint32_t)a.sm_count, (n_tiles + kTeams - 1) / kTeams);
    const bool dev_n = (a.opt & 16u) != 0;                 // a.n is an upper bound, the count is in ctr->launch_n
    // The three kernels are launched with programmatic stream serialization: each may be scheduled while the kernel
    // before it drains, and waits (pdl_wait) before it reads anything that kernel writes.
    cudaLaunchAttribute pdl[1];
    pdl[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    pdl[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(kCtaThreads); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st;
    cfg.attrs = pdl; cfg.numAttrs = 1;
    auto k1 = aggregate_kernel<false, false, false>;
    if (a.prof) k1 = aggregate_kernel<false, true, false>;
    else if (a.sk.cms && dev_n) k1 = aggregate_kernel<true, false, true>;
    else if (a.sk.cms) k1 = aggregate_kernel<true, false, false>;
    else if (dev_n) k1 = aggregate_kernel<false, false, true>;
    cudaLaunchKernelEx(&cfg, k1, a.recs, a.n, a.table, a.epoch, a.ctr, a.spill_idx, a.sk, a.prof, a.opt);
    cfg.gridDim = dim3((unsigned)(a.sm_count * 2)); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = 0;
    cudaLaunchKernelEx(&cfg, fixup_scan_kernel, a.recs, a.n, a.table, a.ctr, a.scratch, a.scratch_slots - 1, a.opt);
    cudaLaunchKernelEx(&cfg, fixup_apply_kernel, a.recs, a.table, a.epoch, a.ctr, a.scratch, a.scratch_slots,
                       reinterpret_cast<unsigned int*>(&a.ctr->scratch[1]));
    return 3;
}
#endif  // FA_HOST_EMUL

}  // namespace fa
