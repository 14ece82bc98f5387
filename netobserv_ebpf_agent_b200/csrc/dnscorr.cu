// dnscorr.cu — K7: DNS query -> response correlation on the device.
//
//   dns_flows map + track_dns_packet:   bpf/dns_tracker.h:23-37 (fill_dns_id), :68-127
//   what flow_monitor does with it:     bpf/flows.c:210-213 (dns_errno = track_dns_packet), :291-330 (one dns_metrics
//                                       sample for the packet's flow when pkt.dns_id != 0 || dns_errno != 0)
//   purge of queries without response:  FlowFetcher.lookupAndDeleteDNSMap, pkg/tracer/tracer.go:1235-1257
//
// The reference runs one sequential program per packet: a query does bpf_map_update_elem(dns_flows, key, ts, NOEXIST),
// a response looks the REVERSED tuple up, turns the stored timestamp into a latency and deletes the entry.  The result
// for one key depends on the order of its packets only, so the batch is processed as
//   resolve   every packet finds or creates its key's entry in the device table and registers its index as a candidate
//             for "smallest unprocessed index of this key" (atomicMin)
//   rounds    a packet whose index IS that minimum applies the reference's step to the entry (plain loads / stores: it is
//             alone on the entry) and retires; the others re-register for the next round in the entry's second index
//             word (the two words alternate by round parity, so one kernel per round is enough).  A key with k packets
//             in the batch needs k rounds: two (query + response) is the normal case; the kernels of later rounds exit
//             at once when nothing is left, and a single-thread tail finishes pathological batches in index order
//   compact   the samples the reference would have produced are packed in stream order (warp ballots + a scan of the
//             per-warp counts) and handed to the K6 DNS fold.
// Entries of answered queries stay in the table as absent keys (open addressing); the engine rebuilds the table from
// its present entries when half of it has been used.
#include "kernels.cuh"

namespace fa {

constexpr uint32_t kDnsNone = 0xFFFFFFFFu;      // no entry (every slot holds another key) / "no index"
constexpr uint32_t kDnsEmit = 0xFFFFFFFEu;      // retired, produced a sample
constexpr uint32_t kDnsSkip = 0xFFFFFFFDu;      // retired, no sample
constexpr uint32_t kDnsQR = 0x8000u;            // DNS_QR_FLAG (dns_tracker.h:10)

struct DnsPkt {                                 // one parsed 104-byte DNS packet record
    uint64_t key[5];                            // dns_flow_id as 5 words: src_ip | dst_ip | src_port, dst_port << 16, id << 32, protocol << 48
    uint64_t ts;
    uint32_t id, flags;
    bool     resp;
};

__device__ __forceinline__ DnsPkt dns_parse(const uint8_t* P) {
    const uint64_t* W = reinterpret_cast<const uint64_t*>(P);
    DnsPkt p;
    const uint64_t w4 = W[4], w8 = W[8];
    p.ts = W[6];                                                    // end_mono_time_ts = pkt.current_ts
    p.id = (uint32_t)(w8 & 0xFFFFu); p.flags = (uint32_t)((w8 >> 16) & 0xFFFFu);
    p.resp = (p.flags & kDnsQR) != 0;
    uint64_t sp = w4 & 0xFFFFu, dp = (w4 >> 16) & 0xFFFFu;
    const uint64_t proto = (w4 >> 32) & 0xFFu;
    if (p.resp) {                                                   // fill_dns_id(..., reverse = true)
        p.key[0] = W[2]; p.key[1] = W[3]; p.key[2] = W[0]; p.key[3] = W[1];
        const uint64_t t = sp; sp = dp; dp = t;
    } else {
        p.key[0] = W[0]; p.key[1] = W[1]; p.key[2] = W[2]; p.key[3] = W[3];
    }
    p.key[4] = sp | (dp << 16) | ((uint64_t)p.id << 32) | (proto << 48);
    return p;
}

// find the key's entry, creating an absent one when the key is new.  The walk may pass every slot of the table: a run
// of occupied slots is not bounded by the pending queries (every packet's key takes an entry until the next rebuild, and
// keys can be chosen to share a home slot), only by the table's fill, which fa_ingest_dns_packets keeps at one half.
// So the walk ends at the key or at an empty slot; kDnsNone (every slot holds another key) cannot happen in such a table.
__device__ uint32_t dns_find_or_create(const DnsCorr& d, const uint64_t k[5]) {
    uint64_t slot = slot_hash(key_premix(k[0], k[1], k[2], k[3], k[4])) & d.mask;
    for (uint64_t probes = 0; probes <= d.mask; ) {
        DnsEntry* E = &d.tab[slot];
        const uint32_t tag = *reinterpret_cast<volatile uint32_t*>(&E->tag);
        if (tag == 0u) {
            if (atomicCAS(&E->tag, 0u, 1u) == 0u) {
#pragma unroll
                for (int c = 0; c < 5; c++) E->key[c] = k[c];
                E->ts = 0ull; E->present = 0u; E->next[0] = kDnsNone; E->next[1] = kDnsNone;
                __threadfence();
                *reinterpret_cast<volatile uint32_t*>(&E->tag) = 2u;
                atomicAdd(&d.ctr[DNSC_CREATED], 1ull);
                return (uint32_t)slot;
            }
            continue;                                               // lost the race: look at the slot again
        }
        if (tag == 1u) continue;                                    // being published
        __threadfence();                                            // the key was written before the tag
        bool same = true;
#pragma unroll
        for (int c = 0; c < 5; c++) same = same && (*reinterpret_cast<volatile unsigned long long*>(&E->key[c]) == k[c]);
        if (same) return (uint32_t)slot;
        slot = (slot + 1) & d.mask;
        probes++;
    }
    return kDnsNone;
}

// The reference's step for one packet whose turn it is (dns_tracker.h:92-110) + the sample of flows.c:291-330.
// `E` may be null: the key has no entry and none could be made (a table with no empty slot, which the engine's fill rule
// rules out; the query is then reported as -E2BIG).  Returns true when a sample was written.
__device__ bool dns_step(const DnsCorr& d, DnsEntry* E, const DnsPkt& p, const uint8_t* P, uint8_t* S) {
    int dns_errno = 0;
    uint64_t latency = 0;
    uint32_t pkt_id = 0, pkt_flags = 0;
    if (!p.resp) {                                                  // query: insert if absent
        if (E && E->present) dns_errno = -17;                       // -EEXIST
        else if (!E || atomicAdd(&d.ctr[DNSC_PRESENT], 1ull) >= d.max_entries) {
            if (E) atomicAdd(&d.ctr[DNSC_PRESENT], ~0ull);          // undo: the map is full
            dns_errno = -7;                                         // -E2BIG
            atomicAdd(&d.ctr[DNSC_FULL], 1ull);
        } else { E->ts = p.ts; E->present = 1u; }
    } else {                                                        // response: lookup + delete
        if (E && E->present) { latency = p.ts - E->ts; E->present = 0u; atomicAdd(&d.ctr[DNSC_PRESENT], ~0ull); }
        else dns_errno = 2;                                         // ENOENT
        pkt_id = p.id; pkt_flags = p.flags;
    }
    if (pkt_id == 0u && dns_errno == 0) return false;
    const uint64_t* W = reinterpret_cast<const uint64_t*>(P);
    uint64_t* O = reinterpret_cast<uint64_t*>(S);
#pragma unroll
    for (int c = 0; c < 5; c++) O[c] = W[c];                        // the packet's flow id
    O[5] = p.ts; O[6] = p.ts; O[7] = latency;                       // start = end = pkt.current_ts
    const uint64_t eth = (W[8] >> 32) & 0xFFFFull;
    const uint64_t err = (uint64_t)(uint8_t)dns_errno;              // u8 field: -17 -> 239, -7 -> 249
    if (p.resp) {
        O[8] = (uint64_t)pkt_id | ((uint64_t)pkt_flags << 16) | (eth << 32) | (err << 48) | (W[8] & 0xFF00000000000000ull);
        O[9] = W[9]; O[10] = W[10]; O[11] = W[11];
        O[12] = W[12] & 0x00FFFFFFFFFFFFFFull;                      // name[25..31], padding byte zero
    } else {                                                        // a query's error sample carries no id / flags / name
        O[8] = (eth << 32) | (err << 48);
        O[9] = 0; O[10] = 0; O[11] = 0; O[12] = 0;
    }
    return true;
}

__global__ void dns_resolve_kernel(const uint8_t* __restrict__ pkts, uint32_t n, DnsCorr d, uint32_t* __restrict__ state,
                                   uint8_t* __restrict__ samples) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint8_t* P = pkts + (size_t)i * kDnsRecBytes;
        const DnsPkt p = dns_parse(P);
        const uint32_t slot = dns_find_or_create(d, p.key);
        if (slot == kDnsNone) {                                     // no entry to order this key by: settled here
            state[i] = dns_step(d, nullptr, p, P, samples + (size_t)i * kDnsRecBytes) ? kDnsEmit : kDnsSkip;
        } else {
            state[i] = slot;
            atomicMin(&d.tab[slot].next[0], i);
            atomicAdd(&d.ctr[DNSC_REMAINING], 1ull);
        }
    }
}

__global__ void dns_round_kernel(const uint8_t* __restrict__ pkts, uint32_t n, DnsCorr d, uint32_t* __restrict__ state,
                                 uint8_t* __restrict__ samples, uint32_t parity) {
    if (*reinterpret_cast<volatile unsigned long long*>(&d.ctr[DNSC_REMAINING]) == 0ull) return;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t s = state[i];
        if (s >= kDnsSkip) continue;                                // retired
        DnsEntry* E = &d.tab[s];
        if (*reinterpret_cast<volatile uint32_t*>(&E->next[parity]) == i) {
            const uint8_t* P = pkts + (size_t)i * kDnsRecBytes;
            const DnsPkt p = dns_parse(P);
            state[i] = dns_step(d, E, p, P, samples + (size_t)i * kDnsRecBytes) ? kDnsEmit : kDnsSkip;
            __threadfence();                                        // the entry's new state before the next round's winner
            *reinterpret_cast<volatile uint32_t*>(&E->next[parity]) = kDnsNone;
            atomicAdd(&d.ctr[DNSC_REMAINING], ~0ull);
        } else {
            atomicMin(&E->next[parity ^ 1u], i);                    // candidate for the next round
        }
    }
}

// whatever the rounds left (a key with more packets in the batch than rounds were launched): one thread, index order
__global__ void dns_tail_kernel(const uint8_t* __restrict__ pkts, uint32_t n, DnsCorr d, uint32_t* __restrict__ state,
                                uint8_t* __restrict__ samples) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    if (*reinterpret_cast<volatile unsigned long long*>(&d.ctr[DNSC_REMAINING]) == 0ull) return;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t s = state[i];
        if (s >= kDnsSkip) continue;
        DnsEntry* E = &d.tab[s];
        const uint8_t* P = pkts + (size_t)i * kDnsRecBytes;
        const DnsPkt p = dns_parse(P);
        state[i] = dns_step(d, E, p, P, samples + (size_t)i * kDnsRecBytes) ? kDnsEmit : kDnsSkip;
        E->next[0] = kDnsNone; E->next[1] = kDnsNone;
    }
    d.ctr[DNSC_REMAINING] = 0ull;
}

// ---- stable compaction of the samples: per-warp counts -> exclusive scan (one warp) -> scatter
__global__ void dns_count_kernel(const uint32_t* __restrict__ state, uint32_t n, uint32_t* __restrict__ warp_count) {
    const uint32_t n_warps = (n + 31) / 32;
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n_warps; w += gridDim.x * blockDim.x / 32) {
        const uint32_t i = w * 32 + lane;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, i < n && state[i] == kDnsEmit);
        if (lane == 0) warp_count[w] = __popc(b);
    }
}

__global__ void dns_scan_kernel(uint32_t* __restrict__ warp_count, uint32_t n_warps, unsigned long long* __restrict__ ctr) {
    if (blockIdx.x != 0 || threadIdx.x >= 32) return;
    const uint32_t lane = threadIdx.x;
    uint32_t run = 0;
    for (uint32_t base = 0; base < n_warps; base += 32) {
        const uint32_t v = base + lane < n_warps ? warp_count[base + lane] : 0u;
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= (uint32_t)o) x += y; }
        if (base + lane < n_warps) warp_count[base + lane] = run + x - v;       // exclusive
        run += __shfl_sync(0xFFFFFFFFu, x, 31);
    }
    if (lane == 0) ctr[DNSC_EMITTED] = run;
}

__global__ void dns_scatter_kernel(const uint32_t* __restrict__ state, uint32_t n, const uint32_t* __restrict__ warp_offset,
                                   const uint8_t* __restrict__ samples, uint8_t* __restrict__ out) {
    const uint32_t n_warps = (n + 31) / 32;
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n_warps; w += gridDim.x * blockDim.x / 32) {
        const uint32_t i = w * 32 + lane;
        const bool emit = i < n && state[i] == kDnsEmit;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, emit);
        if (emit) {
            const uint32_t pos = warp_offset[w] + __popc(b & ((1u << lane) - 1u));
            const uint64_t* S = reinterpret_cast<const uint64_t*>(samples + (size_t)i * kDnsRecBytes);
            uint64_t* O = reinterpret_cast<uint64_t*>(out + (size_t)pos * kDnsRecBytes);
#pragma unroll
            for (int c = 0; c < kDnsRecBytes / 8; c++) O[c] = S[c];
        }
    }
}

// ---- lookupAndDeleteDNSMap (tracer.go:1235-1257): time.Duration(now - ts) >= timeout, a signed 64-bit compare
__global__ void dns_purge_kernel(DnsCorr d, uint64_t now, uint64_t timeout) {
    unsigned long long gone = 0;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= d.mask; s += (uint64_t)gridDim.x * blockDim.x) {
        DnsEntry* E = &d.tab[s];
        if (E->tag == 2u && E->present && (long long)(now - E->ts) >= (long long)timeout) { E->present = 0u; gone++; }
    }
    if (gone) { atomicAdd(&d.ctr[DNSC_PRESENT], 0ull - gone); atomicAdd(&d.ctr[DNSC_PURGED], gone); }
}

// ---- rebuild: the present entries of `from` move into the (zeroed) table `to`; absent keys are dropped
__global__ void dns_rebuild_kernel(DnsCorr from, DnsCorr to) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s <= from.mask; s += (uint64_t)gridDim.x * blockDim.x) {
        const DnsEntry* E = &from.tab[s];
        if (E->tag != 2u || !E->present) continue;
        uint64_t k[5];
#pragma unroll
        for (int c = 0; c < 5; c++) k[c] = E->key[c];
        const uint32_t slot = dns_find_or_create(to, k);            // counts into to.ctr[DNSC_CREATED] (the same counters)
        if (slot != kDnsNone) { to.tab[slot].ts = E->ts; to.tab[slot].present = 1u; }
        else atomicAdd(&to.ctr[DNSC_PRESENT], ~0ull);               // not re-placed (cannot happen at half fill): the query is gone
    }
}

#ifndef FA_HOST_EMUL
int launch_dns_correlate(const uint8_t* pkts, uint32_t n, const DnsCorr& d, uint32_t* state, uint8_t* samples, uint32_t* warp_count,
                         uint8_t* out, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    const int grid = sm_count * 8;
    dns_resolve_kernel<<<grid, 256, 0, st>>>(pkts, n, d, state, samples);
    for (uint32_t r = 0; r < (uint32_t)kDnsRounds; r++) dns_round_kernel<<<grid, 256, 0, st>>>(pkts, n, d, state, samples, r & 1u);
    dns_tail_kernel<<<1, 32, 0, st>>>(pkts, n, d, state, samples);
    dns_count_kernel<<<grid, 256, 0, st>>>(state, n, warp_count);
    dns_scan_kernel<<<1, 32, 0, st>>>(warp_count, (n + 31) / 32, d.ctr);
    dns_scatter_kernel<<<grid, 256, 0, st>>>(state, n, warp_count, samples, out);
    return 5 + kDnsRounds;
}

int launch_dns_purge(const DnsCorr& d, uint64_t now, uint64_t timeout, int sm_count, cudaStream_t st) {
    dns_purge_kernel<<<sm_count * 8, 256, 0, st>>>(d, now, timeout);
    return 1;
}

int launch_dns_rebuild(const DnsCorr& from, const DnsCorr& to, int sm_count, cudaStream_t st) {
    dns_rebuild_kernel<<<sm_count * 8, 256, 0, st>>>(from, to);
    return 1;
}
#endif  // FA_HOST_EMUL

}  // namespace fa
