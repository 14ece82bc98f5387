// kernels.cuh — launch wrappers implemented in the .cu files (internal to libflowagg.so).
#pragma once
#include "common.cuh"

namespace fa {

struct SketchParams {
    unsigned long long* cms;   // depth x 2^log2w u64, or nullptr
    uint32_t*           hll;   // 2^p u32 registers (value = rho), or nullptr
    uint32_t log2w, depth, p;
    uint64_t seed;
};

// scratch entry of the ordered re-fold (one per flow flagged TAG_DIRTY in a launch)
// (an open-addressed set keyed by table slot; capacity = power of two >= 2 x max_batch)
struct FixupScratch {
    unsigned long long key;  // table slot + 1, 0 = empty
    uint32_t nfirst;  // ~(min record index of the flow in this launch)       all-zero == initial state
    uint32_t eth;     // 1 + max index with eth_protocol != 0
    uint32_t dscp;    // 1 + max index with dscp != 0
    uint32_t samp;    // 1 + max index with sampling != 0
    uint32_t nsmac;   // ~(min index with src_mac != 0), 0 = none
    uint32_t ndmac;   // ~(min index with dst_mac != 0), 0 = none
};

struct AggLaunch {
    const uint4* recs;       // n x 144 B, 16-byte aligned, device memory
    uint32_t     n;
    Table        table;
    uint64_t     epoch;
    Counters*    ctr;
    uint32_t*    spill_idx;  // indices of records that found the table physically full
    SketchParams sk;
    FixupScratch* scratch;   // scratch_slots entries, all-zero between launches
    uint32_t     scratch_slots;
    int          sm_count;
    unsigned long long* prof; // 8 phase cycle counters (FA_PHASE_PROFILE=1) or nullptr
    uint32_t     opt;        // switches: 2 = no hot-flow cache (diagnostics), 16 = the record count is on the device (ctr->launch_n)
};

// K1: fold a batch of flow records into the table (ACCOUNTER semantics) and, when any
// flow saw records with differing order-dependent fields, re-fold those flows in stream order.
// Returns the number of kernels launched.
int launch_aggregate(const AggLaunch& a, cudaStream_t st);

// K2: lookup-and-delete every live flow of `table` into out_recs (device pointer, cap records).
// The number found is left in ctr->evict_out (can exceed cap; only cap are written).
// slot_of_out (optional): receives the table slot of every emitted flow, for the feature pass.
// drain: emit + reset only the flows that received records since the last drain; nothing is removed.
int launch_evict(const Table& table, uint4* out_recs, uint32_t* slot_of_out,
                 unsigned long long cap, Counters* ctr, int sm_count, cudaStream_t st, bool drain = false);

// Overflow pre-pass (ACCOUNTER "full" cut, reference pkg/flow/account.go:85-94): finds the index of the
// first record whose key is new when the cache already holds max_entries flows. Result in *cut_out
// (device; == n when the whole batch fits).  idx_set: scratch of set_slots u32 (power of two >= 2n),
// bitmap: scratch of (n+31)/32 u32.
int launch_full_cut(const uint4* recs, uint32_t n, const Table& table, unsigned long long live,
                    unsigned long long max_entries, uint32_t* idx_set, uint32_t set_slots, uint32_t* bitmap,
                    uint32_t* cut_out, int sm_count, cudaStream_t st);

// K6 feature folds (kind 0 = additional_metrics 72-B records, 1 = dns_metrics 104-B records, 2 = pkt_drop_metrics 72-B
// records); slot_of: n u32 scratch
int launch_feature_fold(int kind, const uint8_t* recs, uint32_t n, const Table& t, uint64_t epoch, uint64_t seq0,
                        uint32_t* slot_of, Counters* ctr, int sm_count, cudaStream_t st);
// ... of min(*n_dev, max_n) samples, a count that lives in device memory (grids sized from max_n); slot_of: max_n u32
int launch_feature_fold_counted(int kind, const uint8_t* recs, const unsigned long long* n_dev, uint32_t max_n, const Table& t,
                                uint64_t epoch, uint64_t seq0, uint32_t* slot_of, Counters* ctr, int sm_count, cudaStream_t st);
// feature lines per slot, in uint4 (layouts in features.cu): additional_metrics, dns_metrics, pkt_drop_metrics
constexpr int kAddState = 5;
constexpr int kDnsState = 8;
constexpr int kDropState = 6;
#if defined(__CUDACC__) || defined(FA_HOST_EMUL)
// buildBaseFromAdditional (flow_content.go:63-74) with the fold of all samples of one feature
__device__ __forceinline__ void build_base(uint64_t& bs, uint64_t& be, uint32_t& beth, uint64_t nfs, uint64_t fe, uint64_t neth) {
    const uint64_t s = 0ull - nfs;                       // min non-zero start of the samples, 0 if none
    if (bs == 0 || (bs > s && s != 0)) bs = s;
    if (be == 0 || be < fe) be = fe;
    if (beth == 0 && neth != 0) beth = (uint32_t)(~neth) & 0xFFFFu;
}
// The eviction's patch of a row's start / end / eth_protocol by the non-empty feature lines of `slot`, in its order: DNS,
// then packet drops, then additional (tracer.go:1098-1115,1143-1151).  Returns the present bits: 1 DNS, 2 additional,
// 4 drops.  The eviction's feature pass (evict_features_kernel) and the live-table queries' row reader (evict.cu).
__device__ __forceinline__ uint32_t feature_patch(const Table& t, uint64_t slot, uint64_t& bs, uint64_t& be, uint32_t& beth) {
    uint32_t present = 0;
    if (t.feat_dns) {                                    // nfs, fe, neth: words 4, 5, 6
        const uint64_t* S = reinterpret_cast<const uint64_t*>(t.feat_dns + slot * kDnsState);
        if (S[0]) { present |= 1; build_base(bs, be, beth, S[4], S[5], S[6]); }
    }
    if (t.feat_drop) {                                   // words 6, 7, 8
        const uint64_t* S = reinterpret_cast<const uint64_t*>(t.feat_drop + slot * kDropState);
        if (S[0]) { present |= 4; build_base(bs, be, beth, S[6], S[7], S[8]); }
    }
    if (t.feat_add) {                                    // words 3, 4, 5
        const uint64_t* S = reinterpret_cast<const uint64_t*>(t.feat_add + slot * kAddState);
        if (S[0]) { present |= 2; build_base(bs, be, beth, S[3], S[4], S[5]); }
    }
    return present;
}
#endif
int launch_evict_features(const Table& t, const uint32_t* slot_of_out, unsigned long long n_out, uint8_t* out_recs,
                          uint8_t* out_dns, uint8_t* out_add, uint8_t* out_drop, unsigned long long* out_rtt_min,
                          uint8_t* out_present, int sm_count, cudaStream_t st);
// the same rows for fa_top_flows / fa_lookup_flows, leaving the feature lines as they are (slot kNoSlot: zero rows)
int launch_peek_features(const Table& t, const uint32_t* slot_of_out, unsigned long long n_out, uint8_t* out_recs,
                         uint8_t* out_dns, uint8_t* out_add, uint8_t* out_drop, unsigned long long* out_rtt_min,
                         uint8_t* out_present, int sm_count, cudaStream_t st);

// Rows of the n flows at slots[i * stride] into out_recs (device, n x 144 B), their slots into slot_of_out (optional, for
// the feature pass; 0 without a flow).  A slot kNoSlot is no flow: its row is written all zero when zero_miss, else left
// as it is.  kmap: KERNEL_MAP record layout.
int launch_gather(const Table& t, bool kmap, const uint32_t* slots, uint32_t stride, uint64_t n, bool zero_miss,
                  uint8_t* out_recs, uint32_t* slot_of_out, int sm_count, cudaStream_t st);

// fa_top_flows (evict.cu): radix select over the composite (metric, ~slot hash), compaction, sort, gather.
// one compacted candidate; slot == kTopNoSlot marks the padding that sorts last
struct TopEnt { unsigned long long m, h; uint32_t slot, pad; };
constexpr uint32_t kTopNoSlot = kNoSlot;
constexpr int kTopPasses = 16;                     // 8-bit digits of the 128-bit composite; later passes exit at once
constexpr int kTopSortTile = 1024;                 // entries sorted in shared memory by one CTA
constexpr uint64_t kTopSlack = 4096;               // compaction room beyond k: the select stops once the candidates fit
// select state, on the device: the composite's bits [pos, 128) are resolved to (pm, plo)
struct TopState {
    unsigned long long m_max;                      // largest metric (first kernel)
    unsigned long long pm, plo;                    // resolved prefix: metric bits, ~hash bits
    unsigned long long above;                      // flows strictly above the prefix (all of them are in the result)
    unsigned long long k_rem;                      // result rows still to come from the flows that match the prefix
    unsigned long long n_cand;                     // flows that match the prefix
    unsigned long long count;                      // compaction cursor
    uint32_t pos;                                  // lowest resolved bit
    uint32_t done;                                 // 1: above + n_cand fit the scratch, or every bit is resolved
    uint32_t overflow;                             // every bit resolved and still more candidates than scratch
    uint32_t passes;                               // digit passes taken
};
struct TopScratch {
    TopState* state;                               // zeroed before the launch (with hist)
    unsigned* hist;                                // kTopPasses x 256
    TopEnt* ents;                                  // cap entries (cap: power of two >= k + kTopSlack)
    uint64_t cap;
};
// The n (<= live) highest-ranked live flows of `t` into out_recs (device, n x 144 B) in rank order, and their slots into
// slot_of_out (optional, for the feature pass).  by_bytes: rank by bytes, else by packets.  kmap: KERNEL_MAP record
// layout.  Nothing in `t` changes.
int launch_top_flows(const Table& t, bool kmap, bool by_bytes, uint64_t n, uint64_t live, const TopScratch& s,
                     uint8_t* out_recs, uint32_t* slot_of_out, int sm_count, cudaStream_t st);

// fa_lookup_flows (evict.cu): for each of the n 40-byte keys (device, 8-byte aligned) its slot in `t` or kNoSlot into
// slots (the feature pass reads them), 1 / 0 into found (optional), the number of hits added to *hits, and its row into
// out_recs (device, n x 144 B; all zero without a flow).  kmap: KERNEL_MAP record layout.  Nothing in `t` changes.
int launch_lookup_flows(const Table& t, bool kmap, const uint64_t* keys, uint64_t n, uint32_t* slots, uint8_t* found,
                        unsigned long long* hits, uint8_t* out_recs, int sm_count, cudaStream_t st);

// fa_expire_flows (evict.cu): remove the flows past an idle or active timeout and compact their probe chains in place.
struct ExpireCtr {
    unsigned long long n;                          // expiring flows (mark)
    unsigned long long clusters;                   // clusters that hold one of them (the cluster pass)
};
struct ExpireScratch {
    uint32_t* bm;                                  // expire bitmap, 1 bit per slot (every word written by the mark)
    uint32_t* list;                                // cap entries: the expiring slots; after the gather, the cluster starts
    uint64_t cap;
    ExpireCtr* ctr;                                // zeroed before the mark
};
// Mark: the expire bitmap, the expiring slots (the first cap of them) and their count in s.ctr->n.  Reads only.  Their
// rows: launch_gather over s.list.
int launch_expire_mark(const Table& t, uint64_t now, uint64_t idle, uint64_t active, const ExpireScratch& s, int sm_count,
                       cudaStream_t st);
// Delete the n marked flows with every line they own, move the survivors of their clusters back towards their home slots,
// and take n off ctr->live.  full: the table has no EMPTY slot (one thread, backward-shift deletion).
int launch_expire_delete(const Table& t, const ExpireScratch& s, uint64_t n, bool full, Counters* ctr, int sm_count,
                         cudaStream_t st);

// fa_group_flows (evict.cu): roll the live flows up by a key mask in an open-addressed group table (slot layout in
// evict.cu), list the groups, then emit or clear them.
constexpr int kGroupSlotWords = 12;                // one group-table slot: 12 u64 = 96 B
constexpr int kGroupRowBytes = 88;                 // one fa_flow_group row
struct GroupCtr {
    unsigned long long n;                          // groups created: the list cursor
    unsigned long long lost;                       // folds whose walk met neither their group nor an EMPTY slot (never)
};
struct GroupScratch {
    unsigned long long* tab;                       // (mask + 1) slots, all zero between calls
    uint32_t* list;                                // mask + 1 entries: the slot of every group, in creation order
    uint64_t mask;                                 // slots - 1 (slots: a power of two > 4/3 x the live flows)
    GroupCtr* ctr;                                 // zeroed before the scan
};
struct GroupMask { uint64_t w[5]; };               // the 40-byte key mask as five little-endian words, byte 39 clear
// Scan: fold every live flow of `t` into the group of its masked key (created when absent).  Reads `t` only.
int launch_group_scan(const Table& t, const GroupMask& m, const GroupScratch& s, int sm_count, cudaStream_t st);
// Emit the n listed groups as fa_flow_group rows into out (device, 8-byte aligned; nullptr: write nothing) and zero
// their slots, so that the table is all zero again.
int launch_group_emit(const GroupScratch& s, uint64_t n, uint64_t* out, int sm_count, cudaStream_t st);

// fa_histogram_flows (evict.cu): on the group table of launch_group_scan, a per-group histogram of one per-flow value.
// Row (fa_hist_row): kHistHeadWords u64 of header, then n_bounds + 1 u64 bucket counts.
enum : uint32_t { kHistBytes = 0, kHistPackets = 1, kHistDuration = 2, kHistRtt = 3, kHistDnsLatency = 4 };   // FA_HIST_*
constexpr int kHistMaxBounds = 63;
constexpr int kHistHeadWords = 10;                 // key (5), flows, count, sum, min, max
// Kernel argument (512 B of parameter space): the value and the Prometheus `le` bounds, strictly increasing.
struct HistParams { unsigned long long bounds[kHistMaxBounds]; uint32_t n_bounds, value; };
// row_of[list[i]] = i for the n listed groups (row_of: one u32 per group-table slot).
int launch_hist_index(const GroupScratch& s, uint64_t n, uint32_t* row_of, int sm_count, cudaStream_t st);
// Bin every live flow of `t` that has the value into row row_of[its group] of `rows` (device, all zero before; n rows
// of kHistHeadWords + n_bounds + 1 u64).  Reads `t` and the group table only.
int launch_hist_scan(const Table& t, const GroupMask& m, const GroupScratch& s, const uint32_t* row_of, const HistParams& h,
                     uint64_t* rows, int sm_count, cudaStream_t st);
// Fill row i's key and flows from the i-th listed group and turn its ~min into min.  The group table is left as it is
// (launch_group_emit with out == nullptr clears it).
int launch_hist_emit(const GroupScratch& s, uint64_t n, uint32_t n_bounds, uint64_t* rows, int sm_count, cudaStream_t st);

// fa_distinct_flows (evict.cu): a second level over the groups that launch_group_scan built with G | D (key & (G | D) is
// one (key & G, key & D) pair), folded by key & G into a second group table whose word 7 holds the distinct count.
constexpr int kDistinctRowBytes = 56;              // one fa_distinct_group row
// Fold the n1 listed groups of s1 into s2 (all zero before, its counters zeroed) by their key AND m.  Reads s1 only.
int launch_distinct_fold(const GroupScratch& s1, uint64_t n1, const GroupMask& m, const GroupScratch& s2, int sm_count, cudaStream_t st);
// The slots of s2's groups with distinct >= min_distinct into sel, their number into *n_sel (zeroed before).  bound: at
// least s2's group count (the grid).  Reads s2 only.
int launch_distinct_select(const GroupScratch& s2, uint64_t bound, uint64_t min_distinct, uint32_t* sel, unsigned long long* n_sel,
                           int sm_count, cudaStream_t st);
// Rows of the n groups at slots sel[i] of s2 as fa_distinct_group into out (device, 8-byte aligned).  s2 is left as it is.
int launch_distinct_emit(const GroupScratch& s2, const uint32_t* sel, uint64_t n, uint64_t* out, int sm_count, cudaStream_t st);

// sketches
int launch_cms_query(const SketchParams& sk, const uint4* keys, uint32_t n, unsigned long long* est, cudaStream_t st);
int launch_hll_pack(const SketchParams& sk, uint8_t* out_regs, cudaStream_t st);

// K8: evicted flows -> pbflow.Record wire bytes (pbflow.cu)
struct PbIface { uint32_t if_index; uint8_t mac[6]; uint8_t name_len, udn_len; char name[16]; char udn[64]; };   // == fa_iface_name
struct PbParams {
    uint64_t now_unix_ns, mono_now_ns;
    uint8_t  agent_ip[16];
    uint32_t agent_is_v4;             // 1: agent_ip[12..16) is an IPv4 address
    uint32_t wrap;                    // 1: every record is prefixed with the Records.entries tag + length
    const PbIface* ifaces; uint32_t n_ifaces;
};
struct PbInputs { const uint8_t* recs; const uint8_t* dns; const uint8_t* add; const uint8_t* drop; const uint8_t* present; };
// sizes: n u32 (message bodies), offsets: n + 1 u64, block_sums: ceil(n / 1024) u64 — device scratch
int launch_pb_sizes(const PbInputs& in, uint32_t n, const PbParams& P, uint32_t* sizes, unsigned long long* offsets,
                    unsigned long long* block_sums, int sm_count, cudaStream_t st);
int launch_pb_write(const PbInputs& in, uint32_t n, const PbParams& P, const unsigned long long* offsets, const uint32_t* sizes,
                    uint8_t* out, uint8_t* keys_out, cudaStream_t st);

// 64-byte packet events -> single-packet 144-byte records (misc_kernels.cu)
int launch_expand_events(const uint4* events, uint32_t n, uint4* recs_out, cudaStream_t st);
// (f4) packet snapshots -> records of the packets flow_monitor would submit (and, with a filter, keep), stable order;
// *n_out (device) = how many; filter_ctr[3] (device) += accept / reject / no-match
constexpr int kSnapMaxCtas = 1024;                 // cta_count has this many entries
constexpr int kMaxFilterEntries = 16;              // MAX_FILTER_ENTRIES (bpf/types.h:66)
struct FilterRuleDev {                             // fa_filter_rule with the address as big-endian words
    uint32_t ipw[4]; uint32_t prefix, sample;
    uint16_t dps, dpe, dp1, dp2, sps, spe, sp1, sp2, ps, pe, p1, p2, tcp_flags;
    uint8_t proto, icmp_type, icmp_code, direction, action, filter_drops, peer;
};
struct FilterCidrDev { uint32_t ipw[4]; uint32_t prefix; };
struct FilterSet { uint32_t n_rules, n_peers; FilterRuleDev rules[kMaxFilterEntries]; FilterCidrDev peers[kMaxFilterEntries]; };
int launch_parse_snaps(const uint8_t* snaps, uint32_t n, uint32_t stride, const FilterSet* filter, uint32_t* cta_count, uint8_t* verdict,
                       uint4* out_recs, uint32_t* src_of, unsigned long long* n_out, unsigned long long* filter_ctr, int sm_count,
                       cudaStream_t st);

// K7 DNS query -> response correlation (dnscorr.cu): the dns_flows map of bpf/maps_definition.h:81-89 on the device
struct __align__(64) DnsEntry {                    // one key of dns_flows, 64 B
    unsigned long long key[5];                     // dns_flow_id: src_ip | dst_ip | src_port, dst_port << 16, id << 32, protocol << 48
    unsigned long long ts;                         // the map's value while `present`
    uint32_t tag;                                  // 0 empty, 1 being written, 2 published
    uint32_t present;                              // the map holds the key (a deleted key keeps its entry until the next rebuild)
    uint32_t next[2];                              // per batch: smallest unprocessed packet index of the key, by round parity
};
enum { DNSC_REMAINING = 0, DNSC_CREATED, DNSC_EMITTED, DNSC_PRESENT, DNSC_FULL, DNSC_PURGED, DNSC_N = 8 };
struct DnsCorr { DnsEntry* tab; uint64_t mask; unsigned long long* ctr; unsigned long long max_entries; };
constexpr int kDnsRounds = 6;                      // round kernels per batch (later ones exit at once); the tail takes the rest
// pkts: n x 104 B in stream order; state: n u32; samples: n x 104 B scratch; warp_count: ceil(n / 32) u32; out: n x 104 B,
// receives ctr[DNSC_EMITTED] samples in stream order
int launch_dns_correlate(const uint8_t* pkts, uint32_t n, const DnsCorr& d, uint32_t* state, uint8_t* samples, uint32_t* warp_count,
                         uint8_t* out, int sm_count, cudaStream_t st);
int launch_dns_purge(const DnsCorr& d, uint64_t now, uint64_t timeout, int sm_count, cudaStream_t st);
int launch_dns_rebuild(const DnsCorr& from, const DnsCorr& to, int sm_count, cudaStream_t st);

// generator
struct GenDeviceParams;
int launch_generate(const GenDeviceParams& g, uint64_t first_index, uint32_t n, uint4* dst, cudaStream_t st);

// routing fused with the exchange: destinations are peer-mapped receive buffers + their record counters
struct PeerTargets { uint4* buf[16]; unsigned long long* count[16]; };
int launch_route_peer(const uint4* recs, const unsigned long long* n_dev, uint32_t max_n, uint32_t n_shards, uint32_t self_shard,
                      const PeerTargets& pt, unsigned long long cap, unsigned long long* overflow, int sm_count, cudaStream_t st);
// ... the stable variant for K6 samples (kind as launch_feature_fold): pt.buf[o] / pt.count[o] are the caller's segment of
// owner o's receive buffer (cap samples) and its count word; hist: kMaxShards x ceil(max_n / 256) u32, tot: 16 u64 scratch
int launch_route_samples(int kind, const uint8_t* samples, const unsigned long long* n_dev, uint32_t max_n, uint32_t n_shards,
                         const PeerTargets& pt, unsigned long long cap, uint32_t* hist, unsigned long long* tot,
                         unsigned long long* overflow, int sm_count, cudaStream_t st);

// routing (K3)
int launch_route(const uint4* recs, uint32_t n, uint32_t n_shards, uint4* out, unsigned long long* counts_dev,
                 uint32_t* tmp_owner, int sm_count, cudaStream_t st);

}  // namespace fa
