// misc_kernels.cu — generator, ACCOUNTER "full" cut pre-pass, sketch queries, shard routing (K3).
#include "flowgen.h"
#include "kernels.cuh"

namespace fa {

// ------------------------------------------------------------------ synthetic stream
__global__ void generate_kernel(GenDeviceParams p, uint64_t first_index, uint32_t n, uint4* __restrict__ dst) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint32_t w[36];
        gen_record_words(p, first_index + i, w);
        uint4* o = dst + (size_t)i * kRecChunks;
#pragma unroll
        for (int c = 0; c < kRecChunks; c++) o[c] = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
    }
}
#ifndef FA_HOST_EMUL
int launch_generate(const GenDeviceParams& g, uint64_t first_index, uint32_t n, uint4* dst, cudaStream_t st) {
    if (!n) return 0;
    generate_kernel<<<(n + 255) / 256, 256, 0, st>>>(g, first_index, n, dst);
    return 1;
}
#endif  // FA_HOST_EMUL

// ------------------------------------------------------------------ packet events -> records
// One 64-byte fa_packet_event (4 chunks) becomes the 144-byte record new_flow of bpf/flows.c:228-245 (9 chunks).
// 4 lanes load an event coalesced; every lane of the warp then writes 16-byte chunks of the 8 records of its warp
// round, so loads and stores are both full 128-bit, contiguous per record.
__global__ void expand_events_kernel(const uint4* __restrict__ ev, uint32_t n, uint4* __restrict__ out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4* E = ev + (size_t)i * 4;
        const uint4 e0 = ld_stream_u4(E), e1 = ld_stream_u4(E + 1), e2 = ld_stream_u4(E + 2), e3 = ld_stream_u4(E + 3);
        // e2 = key[32..40) | ts ; e3 = len | flags, dscp, dir | if_index | sampling
        const bool v4 = e0.x == 0u && e0.y == 0u && e0.z == 0xFFFF0000u;       // ::ffff:a.b.c.d
        const uint32_t eth = v4 ? 0x0800u : 0x86DDu;
        const uint32_t flags = e3.y & 0xFFFFu, dscp = (e3.y >> 16) & 0xFFu, dir = e3.y >> 24;
        uint4* O = out + (size_t)i * kRecChunks;
        O[0] = e0; O[1] = e1;
        O[2] = make_uint4(e2.x, e2.y & 0x00FFFFFFu, e2.z, e2.w);               // key tail | start = ts
        O[3] = make_uint4(e2.z, e2.w, e3.x, 0u);                               // end = ts | bytes = len
        O[4] = make_uint4(1u, eth | (flags << 16), 0u, 0u);                    // packets = 1 | eth, flags | MACs = 0
        O[5] = make_uint4(0u, e3.z, 0u, e3.w);                                 // dst_mac tail | if_index | lock | sampling
        O[6] = make_uint4(dir | (dscp << 16), 0u, 0u, 0u);                     // direction, errno, dscp, nb_observed_intf | ...
        O[7] = make_uint4(0u, 0u, 0u, 0u);
        O[8] = make_uint4(0u, 0u, 0u, 0u);
    }
}
#ifndef FA_HOST_EMUL
int launch_expand_events(const uint4* events, uint32_t n, uint4* recs_out, cudaStream_t st) {
    if (!n) return 0;
    expand_events_kernel<<<(n + 255) / 256, 256, 0, st>>>(events, n, recs_out);
    return 1;
}
#endif  // FA_HOST_EMUL

// ------------------------------------------------------------------ "full" cut pre-pass
// Reference pkg/flow/account.go:85-94: the first record whose key is new while the cache
// already holds max_entries flows evicts everything.  Run only when a batch could overflow.
constexpr uint32_t kSetEmpty = 0xFFFFFFFFu;

__device__ __forceinline__ bool rec_key_equal(const uint4* a, const uint4* b) {
    return eq4_masked(a[0], b[0], chunk_mask(0)) && eq4_masked(a[1], b[1], chunk_mask(1)) &&
           eq4_masked(a[2], b[2], chunk_mask(2));
}

__global__ void cut_scan_kernel(const uint4* __restrict__ recs, uint32_t n, Table t, uint32_t* idx_set, uint32_t set_mask) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4* R = recs + (size_t)i * kRecChunks;
        const uint4 k0 = R[0], k1 = R[1], k2 = R[2];
        const uint64_t h = slot_hash(key_premix(u64_of(k0.x, k0.y), u64_of(k0.z, k0.w), u64_of(k1.x, k1.y),
                                                u64_of(k1.z, k1.w), u64_of(k2.x, k2.y)));
        if (table_find(t, h, k0, k1, k2) != kNoSlot) continue;     // the flow exists
        uint32_t s = (uint32_t)(h >> 24) & set_mask;
        for (;;) {
            uint32_t cur = atomicCAS(&idx_set[s], kSetEmpty, i);
            if (cur == kSetEmpty) break;
            if (rec_key_equal(recs + (size_t)cur * kRecChunks, R)) { atomicMin(&idx_set[s], i); break; }
            s = (s + 1) & set_mask;
        }
    }
}
__global__ void cut_mark_kernel(const uint32_t* __restrict__ idx_set, uint32_t set_slots, uint32_t* bitmap) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < set_slots; s += gridDim.x * blockDim.x) {
        const uint32_t i = idx_set[s];
        if (i != kSetEmpty) atomicOr(&bitmap[i >> 5], 1u << (i & 31));
    }
}
// single CTA: cut = index of the (room+1)-th set bit, or n when at most `room` bits are set
__global__ void cut_select_kernel(const uint32_t* __restrict__ bitmap, uint32_t n, unsigned long long room, uint32_t* cut_out) {
    __shared__ unsigned long long partial[1024];
    const uint32_t words = (n + 31) / 32;
    const uint32_t per = (words + blockDim.x - 1) / blockDim.x;
    const uint32_t w0 = threadIdx.x * per, w1 = min(words, w0 + per);
    unsigned long long c = 0;
    for (uint32_t w = w0; w < w1; w++) c += __popc(bitmap[w]);
    partial[threadIdx.x] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long run = 0;
        uint32_t cut = n;
        for (uint32_t tt = 0; tt < blockDim.x && cut == n; tt++) {
            if (run + partial[tt] > room) {
                unsigned long long need = room - run;          // skip `need` bits inside this range
                const uint32_t a = tt * per, b = min(words, a + per);
                for (uint32_t w = a; w < b && cut == n; w++) {
                    uint32_t bits = bitmap[w];
                    const uint32_t pc = __popc(bits);
                    if (need >= pc) { need -= pc; continue; }
                    for (uint32_t k = 0; k < need; k++) bits &= bits - 1;
                    cut = w * 32 + (__ffs(bits) - 1);
                }
            }
            run += partial[tt];
        }
        *cut_out = cut;
    }
}
#ifndef FA_HOST_EMUL
int launch_full_cut(const uint4* recs, uint32_t n, const Table& table, unsigned long long live,
                    unsigned long long max_entries, uint32_t* idx_set, uint32_t set_slots, uint32_t* bitmap,
                    uint32_t* cut_out, int sm_count, cudaStream_t st) {
    // the index set is sized (and cleared) by the window, not by max_batch: a small cache cuts every few thousand records
    uint32_t use = 1024;
    while (use < set_slots && (uint64_t)use < 2ull * n) use <<= 1;
    cudaMemsetAsync(idx_set, 0xFF, (size_t)use * 4, st);
    cudaMemsetAsync(bitmap, 0, ((size_t)n + 31) / 32 * 4, st);
    const int g_scan = (int)min((uint32_t)(sm_count * 8), (n + 255u) / 256u), g_mark = (int)min((uint32_t)(sm_count * 8), (use + 255u) / 256u);
    cut_scan_kernel<<<g_scan, 256, 0, st>>>(recs, n, table, idx_set, use - 1);
    cut_mark_kernel<<<g_mark, 256, 0, st>>>(idx_set, use, bitmap);
    const unsigned long long room = max_entries > live ? max_entries - live : 0ull;
    cut_select_kernel<<<1, 1024, 0, st>>>(bitmap, n, room, cut_out);
    return 3;
}
#endif  // FA_HOST_EMUL

// ------------------------------------------------------------------ sketches
__global__ void cms_query_kernel(SketchParams sk, const uint4* __restrict__ keys, uint32_t n, unsigned long long* est) {
    // keys: n x 40 bytes (not 16-byte aligned per key) -> read as u32 words
    const uint32_t* kw = reinterpret_cast<const uint32_t*>(keys);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t* k = kw + (size_t)i * 10;
        const uint64_t pm = key_premix(u64_of(k[0], k[1]), u64_of(k[2], k[3]), u64_of(k[4], k[5]), u64_of(k[6], k[7]), u64_of(k[8], k[9]));
        const uint64_t a = cms_hash_a(pm, sk.seed), b = cms_hash_b(pm, sk.seed);
        unsigned long long m = ~0ull;
        for (uint32_t d = 0; d < sk.depth; d++) {
            const unsigned long long v = sk.cms[((size_t)d << sk.log2w) + cms_index(a, b, d, sk.log2w)];
            m = v < m ? v : m;
        }
        est[i] = m;
    }
}
#ifndef FA_HOST_EMUL
int launch_cms_query(const SketchParams& sk, const uint4* keys, uint32_t n, unsigned long long* est, cudaStream_t st) {
    if (!n) return 0;
    cms_query_kernel<<<(n + 255) / 256, 256, 0, st>>>(sk, keys, n, est);
    return 1;
}
#endif  // FA_HOST_EMUL
__global__ void hll_pack_kernel(SketchParams sk, uint8_t* out) {
    const uint32_t m = 1u << sk.p;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) out[i] = (uint8_t)sk.hll[i];
}
#ifndef FA_HOST_EMUL
int launch_hll_pack(const SketchParams& sk, uint8_t* out_regs, cudaStream_t st) {
    hll_pack_kernel<<<64, 256, 0, st>>>(sk, out_regs);
    return 1;
}
#endif  // FA_HOST_EMUL

// ------------------------------------------------------------------ K3 route_by_hash
// owner = owner_hash(key) % n_shards.  Stable counting sort: per-CTA histogram -> exclusive
// scan over (shard, cta) -> scatter preserving source order inside a shard.
constexpr int kRouteThreads = 256;
constexpr int kRoutePerCta  = 2048;     // records per CTA
constexpr int kMaxShards    = 16;

__global__ void route_count_kernel(const uint4* __restrict__ recs, uint32_t n, uint32_t n_shards,
                                   uint32_t* __restrict__ owner, uint32_t* __restrict__ cta_hist) {
    __shared__ uint32_t hist[kMaxShards];
    if (threadIdx.x < kMaxShards) hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t base = blockIdx.x * kRoutePerCta;
    for (uint32_t k = threadIdx.x; k < kRoutePerCta; k += kRouteThreads) {
        const uint32_t i = base + k;
        if (i >= n) break;
        const uint4* R = recs + (size_t)i * kRecChunks;
        const uint4 k0 = R[0], k1 = R[1], k2 = R[2];
        const uint64_t pm = key_premix(u64_of(k0.x, k0.y), u64_of(k0.z, k0.w), u64_of(k1.x, k1.y), u64_of(k1.z, k1.w), u64_of(k2.x, k2.y));
        const uint32_t o = (uint32_t)(owner_hash(pm) % n_shards);
        owner[i] = o;
        atomicAdd(&hist[o], 1u);
    }
    __syncthreads();
    if (threadIdx.x < n_shards) cta_hist[threadIdx.x * gridDim.x + blockIdx.x] = hist[threadIdx.x];
}
// single CTA exclusive scan over n_shards * n_ctas counters (shard-major) + per-shard totals
__global__ void route_scan_kernel(uint32_t* cta_hist, uint32_t n_ctas, uint32_t n_shards, unsigned long long* counts) {
    __shared__ uint32_t carry;
    __shared__ uint32_t buf[1024];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const uint32_t total = n_ctas * n_shards;
    for (uint32_t base = 0; base < total; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < total ? cta_hist[i] : 0u;
        buf[threadIdx.x] = v;
        __syncthreads();
        for (uint32_t off = 1; off < 1024; off <<= 1) {           // Hillis-Steele inclusive scan
            uint32_t x = threadIdx.x >= off ? buf[threadIdx.x - off] : 0u;
            __syncthreads();
            buf[threadIdx.x] += x;
            __syncthreads();
        }
        const uint32_t incl = buf[threadIdx.x] + carry;
        if (i < total) cta_hist[i] = incl - v;                      // exclusive
        __syncthreads();
        if (threadIdx.x == 1023) carry = incl;
        __syncthreads();
    }
    // per-shard totals = offset of next shard's first CTA - offset of this shard's first CTA
    if (threadIdx.x < n_shards) {
        const uint32_t s = threadIdx.x;
        const uint32_t begin = cta_hist[s * n_ctas];
        const uint32_t end = (s + 1 < n_shards) ? cta_hist[(s + 1) * n_ctas] : carry;
        counts[s] = (unsigned long long)(end - begin);
    }
}
__global__ void route_scatter_kernel(const uint4* __restrict__ recs, uint32_t n, uint32_t n_shards,
                                     const uint32_t* __restrict__ owner, const uint32_t* __restrict__ cta_off,
                                     uint4* __restrict__ out) {
    // Stable in-CTA partition: per round of 256 records every warp counts its records per shard with
    // ballots, a tiny shared-memory prefix over the 8 warps gives each record its position.
    __shared__ uint32_t wcount[kRouteThreads / 32][kMaxShards];
    __shared__ uint32_t cursor[kMaxShards];
    if (threadIdx.x < n_shards) cursor[threadIdx.x] = cta_off[threadIdx.x * gridDim.x + blockIdx.x];
    const uint32_t base = blockIdx.x * kRoutePerCta;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t round = 0; round < kRoutePerCta / kRouteThreads; round++) {
        const uint32_t i = base + round * kRouteThreads + threadIdx.x;
        const bool valid = i < n;
        const uint32_t o = valid ? owner[i] : 0xFFFFFFFFu;
        uint32_t rank = 0;
        for (uint32_t s = 0; s < n_shards; s++) {
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, o == s);
            if (o == s) rank = __popc(m & ((1u << lane) - 1u));
            if (lane == 0) wcount[warp][s] = __popc(m);
        }
        __syncthreads();
        uint32_t dst = 0;
        if (valid) {
            dst = cursor[o] + rank;
            for (int w = 0; w < warp; w++) dst += wcount[w][o];
        }
        __syncthreads();
        if (threadIdx.x < n_shards) {
            uint32_t t = 0;
            for (int w = 0; w < kRouteThreads / 32; w++) t += wcount[w][threadIdx.x];
            cursor[threadIdx.x] += t;
        }
        __syncthreads();                                  // wcount / cursor are re-used by the next round
        if (valid) {
            const uint4* R = recs + (size_t)i * kRecChunks;
            uint4* O = out + (size_t)dst * kRecChunks;
            uint4 v[kRecChunks];
#pragma unroll
            for (int c = 0; c < kRecChunks; c++) v[c] = ld_stream_u4(R + c);
#pragma unroll
            for (int c = 0; c < kRecChunks; c++) O[c] = v[c];
        }
    }
}

// K3 fused with the exchange: partition the partials of one round by owner and store them straight into the owners'
// receive buffers (peer memory over NVLink, or this GPU's own buffer).  Tiles of 256 records are staged in shared
// memory and sorted by owner there, so that every destination gets ONE contiguous run per tile, written by consecutive
// threads in consecutive 16-byte chunks: peer stores arrive as full 128-byte lines instead of 16-byte fragments (the
// first version stored record by record from one thread each: uncoalesced peer stores).
// One remote atomicAdd per tile and owner reserves the run.  Order inside a destination: tile order is whatever the
// reservations give, records of one tile keep their order.
constexpr int kRouteTile = 256;         // records per tile == threads per CTA

// The in-tile partition by owner shared by the routes over peer memory (route_peer_kernel, sample_place_kernel).
// `o` is the calling thread's owner (0xFF: no record).  Afterwards start[sh] is where owner sh's run begins in the sorted
// tile (start[n_shards] = the tile's records) and wcount[w][sh] where warp w's records of owner sh begin inside it; the
// return value is the thread's rank among its warp's records of the same owner.  Stable: runs are owner-major, records
// keep their tile order inside a run.
__device__ __forceinline__ uint32_t tile_owner_runs(uint32_t o, uint32_t n_shards, uint32_t (*wcount)[kMaxShards], uint32_t* start) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t same = __match_any_sync(0xFFFFFFFFu, o);                 // lanes of this warp bound for the same owner
    const uint32_t rank = __popc(same & ((1u << lane) - 1u));
    if (o != 0xFFu && rank == 0) wcount[warp][o] = __popc(same);
    __syncthreads();
    if (tid == 0) {                                                          // runs: owner-major, warps in order inside a run
        uint32_t acc = 0;
        for (uint32_t sh = 0; sh < n_shards; sh++) {
            start[sh] = acc;
            for (int w = 0; w < kRouteTile / 32; w++) { const uint32_t c = wcount[w][sh]; wcount[w][sh] = acc; acc += c; }
        }
        start[n_shards] = acc;
    }
    __syncthreads();
    return rank;
}
// ... the sorted position of the calling thread's record
__device__ __forceinline__ void tile_owner_perm(uint32_t o, uint32_t rank, uint32_t (*wcount)[kMaxShards], uint8_t* perm, uint8_t* owner_of_pos) {
    if (o != 0xFFu) {
        const uint32_t pos = wcount[threadIdx.x >> 5][o] + rank;
        perm[pos] = (uint8_t)threadIdx.x;
        owner_of_pos[pos] = (uint8_t)o;
    }
}
// ... and the store of the runs: owner sh's run goes to buf[sh] from record cursor[sh] on, W words of T per record, written
// by consecutive threads in consecutive words (full lines over NVLink).  A record at or past `cap` is not stored: counted.
template <class T, int W>
__device__ __forceinline__ void tile_store_runs(uint32_t cnt, const T* tile, const uint8_t* perm, const uint8_t* owner_of_pos,
                                                const uint32_t* start, const unsigned long long* cursor, const PeerTargets& pt,
                                                unsigned long long cap, unsigned long long* overflow) {
    for (uint32_t q = threadIdx.x; q < cnt * W; q += kRouteTile) {
        const uint32_t pos = q / W, c = q - pos * W;
        const uint32_t sh = owner_of_pos[pos];
        const unsigned long long dst = cursor[sh] + (pos - start[sh]);
        if (dst < cap) reinterpret_cast<T*>(pt.buf[sh])[dst * W + c] = tile[(uint32_t)perm[pos] * W + c];   // peer (or local) memory
        else if (c == 0) atomicAdd(overflow, 1ull);                          // receive buffer too small: counted, reported at flush
    }
}

__global__ void __launch_bounds__(kRouteTile)
route_peer_kernel(const uint4* __restrict__ recs, const unsigned long long* __restrict__ n_dev, uint32_t max_n,
                  uint32_t n_shards, uint32_t self_shard, PeerTargets pt, unsigned long long cap,
                  unsigned long long* overflow) {
    __shared__ uint4 tile[kRouteTile * kRecChunks];                 // 36,864 B
    __shared__ uint32_t wcount[kRouteTile / 32][kMaxShards];        // records per warp and owner
    __shared__ uint32_t start[kMaxShards + 1];                      // first position of every owner's run inside the sorted tile
    __shared__ unsigned long long cursor[kMaxShards];               // where the run goes in the owner's receive buffer
    __shared__ uint8_t perm[kRouteTile];                            // sorted position -> record of the tile
    __shared__ uint8_t owner_of_pos[kRouteTile];
    const uint32_t n = n_dev ? (uint32_t)min((unsigned long long)max_n, *n_dev) : max_n;
    const uint32_t tid = threadIdx.x;
    // a preceding drain that produced more than its buffer holds has lost records: count them like a receive overflow
    if (n_dev && blockIdx.x == 0 && tid == 0 && *n_dev > (unsigned long long)max_n) atomicAdd(overflow, *n_dev - max_n);
    const uint32_t n_tiles = (n + kRouteTile - 1) / kRouteTile;
    for (uint32_t tix = blockIdx.x; tix < n_tiles; tix += gridDim.x) {
        const uint32_t first = tix * kRouteTile, cnt = min((uint32_t)kRouteTile, n - first);
        const uint4* G = recs + (size_t)first * kRecChunks;
        if (cnt == (uint32_t)kRouteTile) {                                   // all nine loads in flight before the first store
            uint4 tmp[kRecChunks];
#pragma unroll
            for (int c = 0; c < kRecChunks; c++) tmp[c] = ld_stream_u4(G + tid + c * kRouteTile);
#pragma unroll
            for (int c = 0; c < kRecChunks; c++) tile[tid + c * kRouteTile] = tmp[c];
        } else {
            for (uint32_t q = tid; q < cnt * kRecChunks; q += kRouteTile) tile[q] = ld_stream_u4(G + q);
        }
        if (tid < (kRouteTile / 32) * kMaxShards) (&wcount[0][0])[tid] = 0u;
        __syncthreads();
        uint32_t o = 0xFFu;
        if (tid < cnt) {
            const uint4 k0 = tile[tid * kRecChunks], k1 = tile[tid * kRecChunks + 1], k2 = tile[tid * kRecChunks + 2];
            o = (uint32_t)(owner_hash(key_premix(u64_of(k0.x, k0.y), u64_of(k0.z, k0.w), u64_of(k1.x, k1.y), u64_of(k1.z, k1.w),
                                                 u64_of(k2.x, k2.y))) % n_shards);
        }
        const uint32_t rank = tile_owner_runs(o, n_shards, wcount, start);
        if (tid < n_shards) {                                                // reserve the run in the owner's receive buffer
            const uint32_t c = start[tid + 1] - start[tid];
            cursor[tid] = c ? atomicAdd_system(pt.count[tid], (unsigned long long)c) : 0ull;
            // overflow[1]: records that leave this GPU (x 144 B = the NVLink payload of the exchange)
            if (tid != self_shard && c) atomicAdd(overflow + 1, (unsigned long long)c);
        }
        tile_owner_perm(o, rank, wcount, perm, owner_of_pos);
        __syncthreads();
        tile_store_runs<uint4, kRecChunks>(cnt, tile, perm, owner_of_pos, start, cursor, pt, cap, overflow);
        __syncthreads();                                                      // the tile and its tables are re-used
    }
    __threadfence_system();                                                   // peer stores visible before the kernel retires
}

#ifndef FA_HOST_EMUL
int launch_route_peer(const uint4* recs, const unsigned long long* n_dev, uint32_t max_n, uint32_t n_shards, uint32_t self_shard,
                      const PeerTargets& pt, unsigned long long cap, unsigned long long* overflow, int sm_count, cudaStream_t st) {
    if (!max_n) return 0;
    const uint32_t n_tiles = (max_n + kRouteTile - 1) / kRouteTile;          // the count lives on the device: persistent CTAs over tiles
    const uint32_t grid = std::min<uint32_t>(n_tiles, (uint32_t)sm_count * 5u);
    route_peer_kernel<<<grid, kRouteTile, 0, st>>>(recs, n_dev, max_n, n_shards, self_shard, pt, cap, overflow);
    return 1;
}
#endif  // FA_HOST_EMUL

// K3 for feature samples (72-byte additional / packet-drop, 104-byte DNS), STABLE: the K6 folds of the owners depend on
// the order of a flow's samples (first sample adopted whole, last non-zero DNS id / drop cause ...), so a source's samples
// must reach every owner in the order of the source's slice, not in the order the tiles happen to reserve their runs.
// Source `self` owns segment `self` of every owner's receive buffer (pt.buf[o] points at it, pt.count[o] at its count
// word).  Three passes over tiles of 256 samples: count (keys only) -> exclusive scan over (owner, tile) -> place.
// The place pass sorts each tile by owner in shared memory exactly as route_peer_kernel does, so every owner gets one
// contiguous run per tile, stored as full lines by consecutive threads, at the offset the scan gave that tile.
__device__ __forceinline__ uint32_t sample_owner(const uint64_t* k, uint32_t n_shards) {
    return (uint32_t)(owner_hash(key_premix(k[0], k[1], k[2], k[3], k[4])) % n_shards);
}
__device__ __forceinline__ uint32_t sample_count_of(const unsigned long long* n_dev, uint32_t max_n) {
    return n_dev ? (uint32_t)min((unsigned long long)max_n, *n_dev) : max_n;
}

// hist[o * n_tiles + tile] = samples of the tile bound for owner o; every tile of the max_n bound gets its row (zeros past
// the device count), so that the scan needs no count
template <int kRec>
__global__ void __launch_bounds__(kRouteTile)
sample_count_kernel(const uint8_t* __restrict__ samples, const unsigned long long* __restrict__ n_dev, uint32_t max_n,
                    uint32_t n_shards, uint32_t* __restrict__ hist) {
    FA_DYN_SMEM(sm);
    uint32_t* h = reinterpret_cast<uint32_t*>(sm);                  // [kMaxShards]
    const uint32_t n = sample_count_of(n_dev, max_n), n_tiles = (max_n + kRouteTile - 1) / kRouteTile;
    const uint32_t tid = threadIdx.x;
    for (uint32_t tix = blockIdx.x; tix < n_tiles; tix += gridDim.x) {
        if (tid < kMaxShards) h[tid] = 0u;
        __syncthreads();
        const uint32_t i = tix * kRouteTile + tid;
        uint32_t o = 0xFFu;
        if (i < n) {
            const uint64_t* K = reinterpret_cast<const uint64_t*>(samples + (size_t)i * kRec);
            const uint64_t k[5] = {K[0], K[1], K[2], K[3], K[4]};
            o = sample_owner(k, n_shards);
        }
        const uint32_t same = __match_any_sync(0xFFFFFFFFu, o);
        if (o != 0xFFu && (same & ((1u << (tid & 31u)) - 1u)) == 0u) atomicAdd(&h[o], (uint32_t)__popc(same));
        __syncthreads();
        if (tid < n_shards) hist[tid * n_tiles + tix] = h[tid];
        __syncthreads();
    }
}

// off = route_scan_kernel's exclusive scan of hist (owner-major), tot[o] = owner o's samples.  CTA 0 publishes the
// segment counts (peer stores); the runs go to pt.buf[o] from (off[o][tile] - off[o][0]) on.
template <int kRec>
__global__ void __launch_bounds__(kRouteTile)
sample_place_kernel(const uint8_t* __restrict__ samples, const unsigned long long* __restrict__ n_dev, uint32_t max_n,
                    uint32_t n_shards, PeerTargets pt, unsigned long long cap, const uint32_t* __restrict__ off,
                    const unsigned long long* __restrict__ tot, unsigned long long* overflow) {
    constexpr int W = kRec / 8;                                      // 8-byte words per sample
    FA_DYN_SMEM(sm);
    uint64_t* tile = reinterpret_cast<uint64_t*>(sm);                                            // [kRouteTile * W]
    unsigned long long* cursor = reinterpret_cast<unsigned long long*>(tile + kRouteTile * W);   // [kMaxShards]
    uint32_t (*wcount)[kMaxShards] = reinterpret_cast<uint32_t (*)[kMaxShards]>(cursor + kMaxShards);   // [kRouteTile / 32][kMaxShards]
    uint32_t* start = reinterpret_cast<uint32_t*>(wcount + kRouteTile / 32);                     // [kMaxShards + 1]
    uint8_t* perm = reinterpret_cast<uint8_t*>(start + kMaxShards + 4);                          // [kRouteTile]
    uint8_t* owner_of_pos = perm + kRouteTile;                                                   // [kRouteTile]
    const uint32_t n = sample_count_of(n_dev, max_n), n_tiles = (n + kRouteTile - 1) / kRouteTile, tiles_max = (max_n + kRouteTile - 1) / kRouteTile;
    const uint32_t tid = threadIdx.x;
    if (blockIdx.x == 0 && tid < n_shards) *pt.count[tid] = tot[tid];                           // the owner's count word of this segment
    if (blockIdx.x == 0 && tid == 0 && n_dev && *n_dev > (unsigned long long)max_n) atomicAdd(overflow, *n_dev - max_n);
    for (uint32_t tix = blockIdx.x; tix < n_tiles; tix += gridDim.x) {
        const uint32_t first = tix * kRouteTile, cnt = min((uint32_t)kRouteTile, n - first);
        const uint64_t* G = reinterpret_cast<const uint64_t*>(samples + (size_t)first * kRec);
        if (cnt == (uint32_t)kRouteTile) {                                   // all loads in flight before the first store
            uint64_t tmp[W];
#pragma unroll
            for (int w = 0; w < W; w++) tmp[w] = G[tid + w * kRouteTile];
#pragma unroll
            for (int w = 0; w < W; w++) tile[tid + w * kRouteTile] = tmp[w];
        } else {
            for (uint32_t q = tid; q < cnt * W; q += kRouteTile) tile[q] = G[q];
        }
        if (tid < (kRouteTile / 32) * kMaxShards) (&wcount[0][0])[tid] = 0u;
        if (tid < n_shards) cursor[tid] = off[tid * tiles_max + tix] - off[tid * tiles_max];
        __syncthreads();
        uint32_t o = 0xFFu;
        if (tid < cnt) o = sample_owner(tile + tid * W, n_shards);
        const uint32_t rank = tile_owner_runs(o, n_shards, wcount, start);
        tile_owner_perm(o, rank, wcount, perm, owner_of_pos);
        __syncthreads();
        tile_store_runs<uint64_t, W>(cnt, tile, perm, owner_of_pos, start, cursor, pt, cap, overflow);
        __syncthreads();                                                      // the tile and its tables are re-used
    }
    __threadfence_system();                                                   // peer stores visible before the kernel retires
}

template <int kRec>
constexpr size_t sample_place_smem() { return (size_t)kRouteTile * kRec + kMaxShards * 8 + (kRouteTile / 32 + 1) * kMaxShards * 4 + 16 + 2 * kRouteTile; }

// One text for the device and the host emulation (FA_LAUNCH): every kernel loops over tiles grid-stride or runs one CTA.
// hist: kMaxShards x ceil(max_n / 256) u32, tot: kMaxShards u64 (scratch of the calling engine).
int launch_route_samples(int kind, const uint8_t* samples, const unsigned long long* n_dev, uint32_t max_n, uint32_t n_shards,
                         const PeerTargets& pt, unsigned long long cap, uint32_t* hist, unsigned long long* tot,
                         unsigned long long* overflow, int sm_count, cudaStream_t st) {
    if (!max_n) return 0;
    const uint32_t n_tiles = (max_n + kRouteTile - 1) / kRouteTile;
    const uint32_t grid = std::min<uint32_t>(n_tiles, (uint32_t)sm_count * 5u);
    if (kind == 1) {
        FA_LAUNCH(sample_count_kernel<kDnsRecBytes>, grid, kRouteTile, kMaxShards * 4, st, samples, n_dev, max_n, n_shards, hist);
        FA_LAUNCH(route_scan_kernel, 1, 1024, 0, st, hist, n_tiles, n_shards, tot);
        FA_LAUNCH(sample_place_kernel<kDnsRecBytes>, grid, kRouteTile, sample_place_smem<kDnsRecBytes>(), st, samples, n_dev, max_n,
                  n_shards, pt, cap, hist, tot, overflow);
    } else {                                                          // additional and packet-drop samples: 72 B
        FA_LAUNCH(sample_count_kernel<kAddRecBytes>, grid, kRouteTile, kMaxShards * 4, st, samples, n_dev, max_n, n_shards, hist);
        FA_LAUNCH(route_scan_kernel, 1, 1024, 0, st, hist, n_tiles, n_shards, tot);
        FA_LAUNCH(sample_place_kernel<kAddRecBytes>, grid, kRouteTile, sample_place_smem<kAddRecBytes>(), st, samples, n_dev, max_n,
                  n_shards, pt, cap, hist, tot, overflow);
    }
    return 3;
}

#ifndef FA_HOST_EMUL
int launch_route(const uint4* recs, uint32_t n, uint32_t n_shards, uint4* out, unsigned long long* counts_dev,
                 uint32_t* tmp, int sm_count, cudaStream_t st) {
    if (!n) { cudaMemsetAsync(counts_dev, 0, n_shards * sizeof(unsigned long long), st); return 0; }
    const uint32_t n_ctas = (n + kRoutePerCta - 1) / kRoutePerCta;
    uint32_t* owner = tmp;                    // n
    uint32_t* hist = tmp + n;                 // n_shards * n_ctas
    route_count_kernel<<<n_ctas, kRouteThreads, 0, st>>>(recs, n, n_shards, owner, hist);
    route_scan_kernel<<<1, 1024, 0, st>>>(hist, n_ctas, n_shards, counts_dev);
    route_scatter_kernel<<<n_ctas, kRouteThreads, 0, st>>>(recs, n, n_shards, owner, hist, out);
    return 3;
}
#endif  // FA_HOST_EMUL

}  // namespace fa
