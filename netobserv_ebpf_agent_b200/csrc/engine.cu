// engine.cu — the C ABI of libflowagg.so (include/flowagg.h) and the host-side engine:
// device memory, streams, staging of host batches, the ACCOUNTER "full" logic, stats.
// There is NO CPU fallback: without a CUDA device fa_create fails with FA_E_NODEV.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "../../include/flowagg.h"
#include "flowgen.h"
#include "kernels.cuh"
#include "kmap_body.cuh"

static_assert(sizeof(fa_flow_id) == 40, "flow_id ABI");
static_assert(sizeof(fa_flow_metrics) == 104, "flow_metrics ABI");
static_assert(sizeof(fa_flow_record) == 144, "flow_record ABI");
static_assert(sizeof(fa_dns_metrics) == 64, "dns_metrics ABI");
static_assert(sizeof(fa_additional_metrics) == 32, "additional_metrics ABI");
static_assert(sizeof(fa_dns_record) == 104 && sizeof(fa_additional_record) == 72, "feature record ABI");
static_assert(offsetof(fa_flow_metrics, if_index_first_seen) == 44 && offsetof(fa_flow_metrics, observed_intf) == 68 &&
              offsetof(fa_flow_metrics, ssl_version) == 92 && offsetof(fa_flow_metrics, misc_flags) == 99, "flow_metrics offsets");
static_assert(offsetof(fa_dns_metrics, name) == 31 && offsetof(fa_additional_metrics, ipsec_encrypted) == 30, "feature offsets");

namespace {

thread_local std::string g_err;
int fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_err = buf;
    return code;
}
#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(FA_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

enum PtrKind { PTR_PAGEABLE, PTR_PINNED, PTR_DEVICE };
PtrKind classify(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return PTR_PAGEABLE; }
    if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) return PTR_DEVICE;
    if (a.type == cudaMemoryTypeHost) return PTR_PINNED;
    return PTR_PAGEABLE;
}

// ---------------------------------------------------------------- Zipf threshold tables
struct ZipfTable {
    std::vector<uint64_t> thresholds;
    std::vector<uint32_t> first, size;
    uint64_t* d_thresholds = nullptr; uint32_t* d_first = nullptr; uint32_t* d_size = nullptr;   // per device, lazily
    int device = -1;
};
std::mutex g_zipf_mu;
std::map<std::pair<uint64_t, uint32_t>, ZipfTable*> g_zipf;

// Ranks 1..N split into octaves [2^o, 2^(o+1)), each octave into <= 256 equal sub-ranges.
ZipfTable* zipf_table(uint64_t n_keys, uint32_t s_milli) {
    std::lock_guard<std::mutex> lk(g_zipf_mu);
    auto key = std::make_pair(n_keys, s_milli);
    auto it = g_zipf.find(key);
    if (it != g_zipf.end()) return it->second;
    ZipfTable* z = new ZipfTable();
    const double s = s_milli / 1000.0;
    std::vector<long double> mass;
    for (uint64_t lo = 1; lo <= n_keys; lo <<= 1) {
        const uint64_t hi = std::min<uint64_t>(n_keys + 1, lo << 1);      // ranks [lo, hi)
        const uint64_t span = hi - lo;
        const uint64_t parts = std::min<uint64_t>(span, 256);
        for (uint64_t pi = 0; pi < parts; pi++) {
            const uint64_t a = lo + span * pi / parts, b = lo + span * (pi + 1) / parts;
            long double m = 0;
            for (uint64_t k = a; k < b; k++) m += std::pow((double)k, -s);
            z->first.push_back((uint32_t)(a - 1));
            z->size.push_back((uint32_t)(b - a));
            mass.push_back(m);
        }
    }
    long double total = 0; for (auto m : mass) total += m;
    long double run = 0;
    z->thresholds.resize(mass.size());
    for (size_t i = 0; i < mass.size(); i++) {
        run += mass[i];
        long double f = run / total * 18446744073709551616.0L;
        z->thresholds[i] = f >= 18446744073709551615.0L ? ~0ull : (uint64_t)f;
    }
    z->thresholds.back() = ~0ull;
    g_zipf[key] = z;
    return z;
}

}  // namespace

// ------------------------------------------------------------------------ engine
struct fa_engine {
    fa_config cfg{};
    int device = 0, sm_count = 132;
    cudaStream_t stream = nullptr; bool own_stream = false;
    cudaStream_t copy_stream = nullptr;
    std::mutex mu;

    fa::Table table{};
    uint64_t slots = 0, epoch = 0;
    // FA_F_NONBLOCKING_EVICT: a second, empty table.  fa_evict swaps the two under `mu` (the Accounter hands its map
    // over and goes on with a fresh one, pkg/flow/account.go:67-68,86-87; in KERNEL_MAP mode a packet racing
    // LookupAndDeleteMap lands in a fresh entry) and scans the retired one on its own stream.
    fa::Table table_spare{};
    bool double_buffered = false;
    std::mutex evict_mu;                      // one eviction at a time (the reference's evictor is single-flight)
    cudaStream_t evict_stream = nullptr;
    cudaEvent_t ev_swap = nullptr;
    fa::Counters* d_ctr_ev = nullptr;         // evict_out cursor of the scan of the retired table
    unsigned long long* h_ev_out = nullptr;   // pinned
    fa::Counters* d_ctr = nullptr;
    fa::Counters* h_ctr = nullptr;            // pinned mirror
    uint64_t max_batch = 0;

    // staging for host input (double buffered)
    uint8_t* d_stage[2] = {nullptr, nullptr};
    uint8_t* h_stage[2] = {nullptr, nullptr};
    cudaEvent_t ev_stage_free[2] = {nullptr, nullptr};   // kernel that consumed the stage finished
    cudaEvent_t ev_copied[2] = {nullptr, nullptr};       // H2D copy into the stage finished
    int stage_cur = 0;

    fa::FixupScratch* d_scratch = nullptr; uint32_t scratch_slots = 0;
    uint32_t* d_spill_idx = nullptr;
    uint32_t* d_cut_set = nullptr; uint32_t cut_set_slots = 0;
    uint32_t* d_cut_bitmap = nullptr; uint32_t* d_cut_out = nullptr; uint32_t* h_cut_out = nullptr;

    uint8_t* d_expanded = nullptr;            // ... and their 144-byte expansion (events handed in as device memory)
    uint32_t* d_snap_src = nullptr;           // fa_ingest_snaps: snapshot index of every record parsed out of a chunk
    uint32_t* d_snap_cnt = nullptr;           // ... records per CTA of the parse kernels, then the total + 3 filter counters (u64)
    uint8_t* d_snap_verdict = nullptr;        // ... with a flow filter: keep / skip per snapshot of the chunk
    fa::FilterSet filter{};                   // fa_set_flow_filter (n_rules == 0: no filter)
    // device staging of the host-bound fa_evict_ex blocks and the feature pass's slot list, grown on demand
    struct Staging {
        uint8_t* rec = nullptr; uint64_t cap = 0;
        uint8_t *dns = nullptr, *add = nullptr, *drop = nullptr, *present = nullptr;
        unsigned long long* rttmin = nullptr; uint32_t* slot_of = nullptr; uint64_t feat_cap = 0;
    };
    Staging evict_stage;                      // eviction: under `mu` (blocking) or `evict_mu` alone (non-blocking)
    Staging top_stage;                        // fa_top_flows: under `mu`
    fa::TopScratch top{};                     // fa_top_flows select state, histograms and candidates (cap entries)
    fa::TopState* h_top_state = nullptr;      // pinned
    Staging lookup_stage;                     // fa_lookup_flows: under `mu`
    uint32_t* d_lookup_slot = nullptr;        // fa_lookup_flows scratch of one chunk: each key's slot (or kNoSlot) ...
    uint8_t* d_lookup_found = nullptr;        // ... and found flag (for a host `found`); lookup_cap keys
    uint64_t lookup_cap = 0;
    unsigned long long* d_lookup_hits = nullptr; unsigned long long* h_lookup_hits = nullptr;   // hit count; pinned mirror
    Staging expire_stage;                     // fa_expire_flows: under `mu`
    fa::ExpireScratch expire{};               // fa_expire_flows: expire bitmap, slot list (cap entries), counters
    fa::ExpireCtr* h_expire_ctr = nullptr;    // pinned
    fa::GroupScratch group{};                 // fa_group_flows, under `mu`: group table (all zero between calls), list, counters
    fa::GroupCtr* h_group_ctr = nullptr;      // pinned
    uint8_t* d_group_out = nullptr;           // ... and its staging of host-bound rows, group_out_bytes
    uint64_t group_out_bytes = 0;
    uint32_t* d_hist_row_of = nullptr;        // fa_histogram_flows, under `mu`: row of each group, one u32 per group-table slot
    uint8_t* d_hist_out = nullptr;            // ... and its staging of host-bound rows, hist_out_bytes
    uint64_t hist_out_bytes = 0;
    fa::GroupScratch distinct{};              // fa_distinct_flows, under `mu`: the second group table (all zero between calls)
    fa::GroupCtr* h_distinct_ctr = nullptr;   // pinned
    uint8_t* d_distinct_out = nullptr;        // ... and its staging of host-bound rows, distinct_out_bytes
    uint64_t distinct_out_bytes = 0;
    uint32_t* d_slot_of = nullptr;            // per-sample slot scratch of the feature folds
    uint64_t feat_seq[3] = {0, 0, 0};         // running sample numbers (additional, dns, packet drops)
    uint32_t* d_route_tmp = nullptr; unsigned long long* d_route_counts = nullptr;
    uint32_t* d_sroute_hist = nullptr; uint64_t sroute_tiles = 0;   // fa_route_peer_samples: per-(owner, tile) counts ...
    unsigned long long* d_sroute_tot = nullptr;                    // ... and per-owner totals

    fa::SketchParams sk{};
    unsigned long long* d_prof = nullptr;     // FA_PHASE_PROFILE=1: per-phase warp-cycle counters of K1
#ifndef FA_K1_DEFAULT_OPT
#define FA_K1_DEFAULT_OPT 0u                  // K1 switches an engine starts with (kernels.cuh, AggLaunch::opt); FA_K1_OPT overrides (diagnostics)
#endif
    uint32_t k1_opt = FA_K1_DEFAULT_OPT;

    // live-flow bookkeeping for the "full" rule: live_known is exact as of the last retired
    // launch; unsynced_records bounds the flows that launches still in flight can add.
    uint64_t live_known = 0;
    uint64_t unsynced_records = 0;
    static constexpr int kLiveRing = fa::kLiveRing;
    unsigned long long* h_live_ring = nullptr;   // mapped pinned, kLiveRing entries (ACCOUNTER: written by K1, Counters::live_ring)
    cudaEvent_t ev_live[kLiveRing] = {};
    uint32_t ring_n[kLiveRing] = {};
    uint32_t ring_head = 0, ring_tail = 0;       // monotonically increasing; slot = idx % kLiveRing

    // KERNEL_MAP mode (kmap.cu): per-batch scratch, fallback ring (the metric lines are table.met)
    uint32_t* km_slot_of = nullptr;
    fa::KmBEntry* km_bset = nullptr; uint32_t km_bset_slots = 0;
    uint32_t* km_blist = nullptr;
    uint32_t *km_touched = nullptr, *km_deferred = nullptr, *km_brec = nullptr;   // v2 work lists
    int km_impl = 2;                          // FA_KMAP_IMPL: 1 = seven per-record passes, 2 = per-flow finalisation
    uint8_t* km_spill = nullptr; uint64_t km_spill_cap = 0;
    fa::KmCounters* d_km_ctr = nullptr;
    fa::KmCounters* h_km_ctr = nullptr;       // pinned mirror
    uint64_t km_spilled_total = 0;            // records read back by fa_read_spilled so far

    // K8 scratch (fa_pb_encode), grown on demand
    uint32_t* d_pb_sizes = nullptr; unsigned long long* d_pb_offsets = nullptr; unsigned long long* d_pb_sums = nullptr;
    uint64_t pb_cap = 0;
    fa::PbIface* d_pb_ifaces = nullptr; uint32_t pb_ifaces_cap = 0;

    // K7 (dnscorr.cu): the dns_flows map + per-chunk scratch, allocated by the first fa_ingest_dns_packets
    fa::DnsCorr dnsc{};                       // tab == nullptr until then
    fa::DnsEntry* dnsc_spare = nullptr;       // the other table of a rebuild
    unsigned long long* h_dnsc_ctr = nullptr; // pinned mirror of dnsc.ctr
    uint32_t* d_dnsc_state = nullptr; uint8_t* d_dnsc_samples = nullptr; uint8_t* d_dnsc_out = nullptr; uint32_t* d_dnsc_warps = nullptr;
    uint64_t dnsc_chunk = 0;                  // packets per launch_dns_correlate
    uint64_t dnsc_used = 0;                   // upper bound of the table entries in use (present + answered keys)
    uint64_t dnsc_slots = 0;                  // 4 x max_entries: answered keys keep their entry until the next rebuild

    fa_stats st{};
};

namespace fa {
int launch_kmap_batch(KmParams P, uint32_t cut, int sm_count, cudaStream_t st);
int launch_kmap_batch_v2(KmParams P, uint32_t cut, int sm_count, cudaStream_t st);
int launch_kmap_evict(const Table& t, uint8_t* met, uint8_t* out, unsigned long long cap, unsigned long long* cursor,
                      uint32_t* slot_of_out, int sm_count, cudaStream_t st);
}

namespace {

// The live-flow count is exactly `live` and no launch is in flight (counters just read back, or the table emptied).
void set_live_known(fa_engine* e, uint64_t live) {
    e->live_known = live;
    e->unsynced_records = 0;
    e->ring_head = e->ring_tail;
}

int sync_counters(fa_engine* e) {
    CU(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(fa::Counters), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    set_live_known(e, e->h_ctr->live);
    return FA_OK;
}

// Retire launches whose live-count read-back has landed (never blocks).
void retire_completed(fa_engine* e) {
    while (e->ring_head != e->ring_tail) {
        const uint32_t s = e->ring_head % fa_engine::kLiveRing;
        if (cudaEventQuery(e->ev_live[s]) != cudaSuccess) { cudaGetLastError(); break; }
        e->live_known = e->h_live_ring[s];
        e->unsynced_records -= e->ring_n[s];
        e->ring_head++;
    }
}

// Book-keeping after the launches of one chunk: asynchronous read-back of the live-flow count.  In ACCOUNTER mode the
// chunk was one K1 launch, whose last CTA writes the count into ring entry ring_tail % kLiveRing itself (every K1 launch
// comes through here once, so the device's Counters::live_seq and ring_tail stay equal).  A KERNEL_MAP batch counts its
// inserts in one or two resolve kernels of nine and has no ticket that ends after all of them, so the count is copied
// after the batch.
int note_launch(fa_engine* e, uint32_t n) {
    e->unsynced_records += n;
    e->st.records_ingested += n;
    if (e->ring_tail - e->ring_head == fa_engine::kLiveRing) {
        CU(cudaEventSynchronize(e->ev_live[e->ring_head % fa_engine::kLiveRing]));
        retire_completed(e);
    }
    const uint32_t s = e->ring_tail % fa_engine::kLiveRing;
    if (e->cfg.mode == FA_MODE_KERNEL_MAP)
        CU(cudaMemcpyAsync(&e->h_live_ring[s], &e->d_ctr->live, 8, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaEventRecord(e->ev_live[s], e->stream));
    e->ring_n[s] = n;
    e->ring_tail++;
    return FA_OK;
}

// Launch K1 on a device-resident chunk (n <= max_batch).
int launch_chunk(fa_engine* e, const uint8_t* d_recs, uint32_t n) {
    fa::AggLaunch a{};
    a.recs = reinterpret_cast<const uint4*>(d_recs);
    a.n = n;
    a.table = e->table;
    a.epoch = ++e->epoch;
    a.ctr = e->d_ctr;
    a.spill_idx = e->d_spill_idx;
    a.sk = (e->cfg.flags & FA_F_ENABLE_SKETCH) ? e->sk : fa::SketchParams{};
    a.scratch = e->d_scratch;
    a.scratch_slots = e->scratch_slots;
    a.sm_count = e->sm_count;
    a.prof = e->d_prof;
    a.opt = e->k1_opt;
    e->st.kernel_launches += fa::launch_aggregate(a, e->stream);
    CU(cudaGetLastError());
    return note_launch(e, n);
}

// Pre-pass of a chunk that may fill the table: *cut = the index of the first of the n records whose key is new while
// live_known (exact) flows fill max_entries, or n.  Waits for the 4-byte read-back.
int find_cut(fa_engine* e, const uint8_t* d_recs, uint32_t n, uint32_t* cut) {
    e->st.kernel_launches += fa::launch_full_cut(reinterpret_cast<const uint4*>(d_recs), n, e->table, e->live_known,
                                                 e->cfg.max_entries, e->d_cut_set, e->cut_set_slots, e->d_cut_bitmap,
                                                 e->d_cut_out, e->sm_count, e->stream);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(e->h_cut_out, e->d_cut_out, 4, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    *cut = *e->h_cut_out;
    return FA_OK;
}

// ACCOUNTER mode: fold a device-resident chunk honouring max_entries.
// Returns FA_OK (all folded) or FA_FULL with *consumed < n.
int ingest_chunk_accounter(fa_engine* e, const uint8_t* d_recs, uint32_t n, uint32_t* consumed) {
    *consumed = 0;
    const uint64_t M = e->cfg.max_entries;
    retire_completed(e);
    if (e->cfg.flags & FA_F_NO_FULL_CUT) {              // max_entries only sizes the table
        int rc = launch_chunk(e, d_recs, n);
        if (rc) return rc;
        *consumed = n;
        return FA_OK;
    }
    // Launches still in flight may add up to unsynced_records flows.  When that bound does not leave room for this
    // chunk, wait for the OLDEST launch's live-count read-back only (the stream keeps working on the younger ones),
    // and drain the stream only when nothing is left in flight.
    while (e->live_known + e->unsynced_records + n > M && e->ring_head != e->ring_tail) {
        CU(cudaEventSynchronize(e->ev_live[e->ring_head % fa_engine::kLiveRing]));
        retire_completed(e);
    }
    if (e->live_known + e->unsynced_records + n > M && e->unsynced_records) {
        int rc = sync_counters(e);                     // exact live count (feature folds do not use the ring)
        if (rc) return rc;
    }
    if (e->live_known + e->unsynced_records + n <= M) { // cannot overflow: fast path
        int rc = launch_chunk(e, d_recs, n);
        if (rc) return rc;
        *consumed = n;
        return FA_OK;
    }
    // slow path: find the first record whose key is new while the cache is full.  The cut cannot come before `room`
    // new keys have been seen, so it is looked for inside a window proportional to the room that is left: the pre-pass
    // work stays linear in the records consumed however small the cache is.  A window without a cut is folded and the
    // caller goes on with the rest of its chunk.
    const uint64_t room = M > e->live_known ? M - e->live_known : 0;      // exact: the counters were just read
    const uint32_t win = (uint32_t)std::min<uint64_t>(n, std::max<uint64_t>(4096, 4 * room));
    uint32_t cut = 0;
    if (int rc = find_cut(e, d_recs, win, &cut)) return rc;
    if (cut > 0) {
        int rc = launch_chunk(e, d_recs, cut);
        if (rc) return rc;
        rc = sync_counters(e);
        if (rc) return rc;
    }
    *consumed = cut;
    if (cut < win) { e->st.full_cuts++; return FA_FULL; }
    return FA_OK;
}

// KERNEL_MAP mode: the map update of flow_monitor (bpf/flows.c:222-288) for a device-resident chunk.  The map
// never "fills and flushes": once max_entries flows are live, packets of unknown flows go to the fallback ring
// (or only count), so the whole chunk is always consumed.
int ingest_chunk_kmap(fa_engine* e, const uint8_t* d_recs, uint32_t n, uint32_t* consumed) {
    *consumed = 0;
    const uint64_t M = e->cfg.max_entries;
    retire_completed(e);
    if (e->live_known + e->unsynced_records + n > M) {
        int rc = sync_counters(e);                     // exact live count
        if (rc) return rc;
    }
    uint32_t cut = n;                                  // records [cut, n) find the map full
    if (e->live_known + e->unsynced_records + n > M) {
        if (int rc = find_cut(e, d_recs, n, &cut)) return rc;
        if (cut < n) e->st.full_cuts++;
    }
    fa::KmParams P{};
    P.recs = d_recs; P.n = n;
    P.ringbuf = (e->cfg.flags & FA_F_RINGBUF_FALLBACK) ? 1 : 0;
    P.t = e->table; P.met = e->table.met;
    P.epoch = ++e->epoch;
    P.slot_of = e->km_slot_of;
    P.live = &e->d_ctr->live;
    P.c = e->d_km_ctr;
    P.spill = e->km_spill; P.spill_cap = e->km_spill_cap;
    P.bset = e->km_bset; P.bset_mask = e->km_bset_slots - 1; P.blist = e->km_blist;
    P.touched = e->km_touched; P.deferred = e->km_deferred; P.brec = e->km_brec;
    e->st.kernel_launches += e->km_impl == 1 ? fa::launch_kmap_batch(P, cut, e->sm_count, e->stream)
                                             : fa::launch_kmap_batch_v2(P, cut, e->sm_count, e->stream);
    CU(cudaGetLastError());
    *consumed = n;
    return note_launch(e, n);
}

int ingest_chunk(fa_engine* e, const uint8_t* d_recs, uint32_t n, uint32_t* consumed) {
    return e->cfg.mode == FA_MODE_KERNEL_MAP ? ingest_chunk_kmap(e, d_recs, n, consumed)
                                             : ingest_chunk_accounter(e, d_recs, n, consumed);
}

// Fold n device-resident records in launches of at most max_batch; a launch may fold only a window of its records
// ("full" cuts).  Returns FA_OK or the first error / FA_FULL, with *consumed the records folded.
int ingest_device(fa_engine* e, const uint8_t* d_recs, size_t n, size_t* consumed) {
    size_t done = 0;
    int rc = FA_OK;
    while (rc == FA_OK && done < n) {
        const uint32_t c = (uint32_t)std::min<size_t>(n - done, e->max_batch);
        uint32_t took = 0;
        rc = ingest_chunk(e, d_recs + done * fa::kRecBytes, c, &took);
        done += took;
    }
    *consumed = done;
    return rc;
}

// Host data reaches the device through two staging buffers of stage_records() records: the copy of chunk k+1 (copy
// stream) overlaps the kernels of chunk k (engine stream).  The staging grain is independent of max_batch, the K1
// launch size for device-resident input: a large launch amortises K1's start-up, a small stage keeps the pipeline fine.
static uint64_t stage_records(const fa_engine* e) { return std::min<uint64_t>(e->max_batch, 1ull << 20); }   // 151 MB of records per copy

// ACCOUNTER mode: a cache that is about to fill cuts the chunk after roughly `room` new keys.  A chunk of c items is
// bounded by a window proportional to the room left, so that a "full" return does not leave most of a copied or
// expanded chunk unused (the caller hands the rest in again after its eviction).
static uint64_t room_window(fa_engine* e, uint64_t c) {
    if (e->cfg.mode != FA_MODE_ACCOUNTER || (e->cfg.flags & FA_F_NO_FULL_CUT)) return c;
    retire_completed(e);
    const uint64_t used = e->live_known + e->unsynced_records;
    const uint64_t room = e->cfg.max_entries > used ? e->cfg.max_entries - used : 0;
    return room < c ? std::min<uint64_t>(c, std::max<uint64_t>(4096, 4 * room)) : c;
}

enum RoomWindow { WINDOW_NONE, WINDOW_HOST, WINDOW_ALL };   // which input room_window() bounds

// The input of an fa_ingest* call: n items of `width` bytes in caller memory, handed to the kernels in chunks of at most
// dev_chunk items (device input, read in place) or host_chunk items (host input, copied into a staging buffer).  Per
// chunk: next(), release() right after the last kernel that reads the chunk is enqueued, advance() by the items
// consumed.  finish() once at the end.
struct Input {
    fa_engine* e;
    const uint8_t* src;
    size_t n, width;
    uint64_t dev_chunk, host_chunk;
    RoomWindow window;
    PtrKind kind;
    size_t done = 0;
    int sidx = -1;                                             // staging buffer of the current chunk (host input)

    Input(fa_engine* e_, const void* p, size_t n_, size_t width_, uint64_t dev_chunk_, uint64_t host_chunk_, RoomWindow window_)
        : e(e_), src(static_cast<const uint8_t*>(p)), n(n_), width(width_), dev_chunk(dev_chunk_), host_chunk(host_chunk_),
          window(window_), kind(classify(p)) {}

    bool misaligned(uintptr_t align) const { return kind == PTR_DEVICE && (reinterpret_cast<uintptr_t>(src) & (align - 1)); }
    bool more() const { return done < n; }
    void advance(size_t k) { done += k; }

    uint64_t chunk() const {                                   // items in the next chunk
        const uint64_t c = std::min<uint64_t>(n - done, kind == PTR_DEVICE ? dev_chunk : host_chunk);
        return window == WINDOW_ALL || (window == WINDOW_HOST && kind != PTR_DEVICE) ? room_window(e, c) : c;
    }

    // -> the next chunk on the device and its item count.  Host input is copied into the next staging buffer on the
    // copy stream (pageable input through a pinned buffer first); the engine stream waits for the copy.
    int next(const uint8_t** d_in, uint64_t* c) {
        *c = chunk();
        const uint8_t* p = src + done * width;
        *d_in = p;
        if (kind == PTR_DEVICE) return FA_OK;
        const size_t bytes = *c * width, stage_bytes = stage_records(e) * fa::kRecBytes;
        for (int i = 0; i < 2; i++) {
            if (!e->d_stage[i]) CU(cudaMalloc(&e->d_stage[i], stage_bytes));
            if (kind == PTR_PAGEABLE && !e->h_stage[i]) CU(cudaHostAlloc(&e->h_stage[i], stage_bytes, cudaHostAllocDefault));
        }
        sidx = e->stage_cur; e->stage_cur ^= 1;
        CU(cudaEventSynchronize(e->ev_stage_free[sidx]));            // the previous reader of this stage is done
        if (kind == PTR_PAGEABLE) { memcpy(e->h_stage[sidx], p, bytes); p = e->h_stage[sidx]; }
        CU(cudaMemcpyAsync(e->d_stage[sidx], p, bytes, cudaMemcpyHostToDevice, e->copy_stream));
        CU(cudaEventRecord(e->ev_copied[sidx], e->copy_stream));
        CU(cudaStreamWaitEvent(e->stream, e->ev_copied[sidx], 0));
        e->st.h2d_bytes += bytes;
        *d_in = e->d_stage[sidx];
        return FA_OK;
    }

    int release() {                                            // the kernels enqueued so far were the chunk's last readers
        if (sidx >= 0) CU(cudaEventRecord(e->ev_stage_free[sidx], e->stream));
        return FA_OK;
    }

    int finish(int rc, size_t* consumed) {
        if (kind != PTR_DEVICE) CU(cudaStreamSynchronize(e->copy_stream));   // the caller's buffer is not referenced after return
        if (consumed) *consumed = done;
        return rc;
    }
};

}  // namespace

// Everything fa_evict swaps (FA_F_NONBLOCKING_EVICT): identity lines, occupancy bitmap, the mode's metric lines (hot
// lines / KERNEL_MAP flow_metrics lines) and the enabled feature lines — zeroed on the engine stream.
static int alloc_table(fa_engine* e, fa::Table* t) {
    const uint64_t slots = e->slots;
    const uint32_t f = e->cfg.flags;
    auto zeroed = [e](auto** p, size_t bytes) -> int {
        CU(cudaMalloc(p, bytes));
        CU(cudaMemsetAsync(*p, 0, bytes, e->stream));
        return FA_OK;
    };
    t->mask = slots - 1;
    if (int rc = zeroed(&t->ident, slots * fa::kIdentBytes)) return rc;
    if (int rc = e->cfg.mode == FA_MODE_KERNEL_MAP ? zeroed(&t->met, slots * fa::kMetLineBytes) : zeroed(&t->hot, slots * fa::kHotBytes)) return rc;
    if (int rc = zeroed(&t->occ, slots / 8)) return rc;
    if (f & FA_F_ENABLE_RTT) { if (int rc = zeroed(&t->feat_add, slots * 80)) return rc; }
    if (f & FA_F_ENABLE_DNS) { if (int rc = zeroed(&t->feat_dns, slots * 128)) return rc; }
    if (f & FA_F_ENABLE_PKT_DROP) { if (int rc = zeroed(&t->feat_drop, slots * 96)) return rc; }
    return FA_OK;
}

static void free_staging(fa_engine::Staging* s) {
    cudaFree(s->rec); cudaFree(s->dns); cudaFree(s->add); cudaFree(s->drop); cudaFree(s->present);
    cudaFree(s->rttmin); cudaFree(s->slot_of);
    *s = fa_engine::Staging{};
}

static void free_table(fa::Table* t) {
    cudaFree(t->ident); cudaFree(t->hot); cudaFree(t->met); cudaFree(t->occ);
    cudaFree(t->feat_add); cudaFree(t->feat_dns); cudaFree(t->feat_drop);
    *t = fa::Table{};
}

extern "C" {

uint32_t fa_abi_version(void) { return FA_ABI_VERSION; }
const char* fa_last_error(void) { return g_err.c_str(); }

int fa_create(const fa_config* cfg, fa_engine** out) {
    if (!cfg || !out) return fail(FA_E_INVAL, "fa_create: null argument");
    if (cfg->abi_version != FA_ABI_VERSION) return fail(FA_E_INVAL, "fa_create: abi_version %u != %u", cfg->abi_version, FA_ABI_VERSION);
    if (cfg->max_entries == 0) return fail(FA_E_INVAL, "fa_create: max_entries must be >= 1");
    if (cfg->mode != FA_MODE_ACCOUNTER && cfg->mode != FA_MODE_KERNEL_MAP) return fail(FA_E_INVAL, "fa_create: unknown mode %u", cfg->mode);
    const bool kmap = cfg->mode == FA_MODE_KERNEL_MAP;
    if (kmap) {
        if (cfg->flags & (FA_F_ENABLE_SKETCH | FA_F_NO_FULL_CUT))
            return fail(FA_E_INVAL, "fa_create: mode KERNEL_MAP does not take FA_F_ENABLE_SKETCH / FA_F_NO_FULL_CUT (flags 0x%x)", cfg->flags);
    } else if (cfg->flags & FA_F_RINGBUF_FALLBACK) {
        return fail(FA_E_INVAL, "fa_create: FA_F_RINGBUF_FALLBACK needs mode KERNEL_MAP");
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(FA_E_NODEV, "fa_create: no CUDA device; this engine has no CPU fallback");
    }
    if (cfg->device < 0 || cfg->device >= ndev) return fail(FA_E_INVAL, "fa_create: device %d out of range (%d devices)", cfg->device, ndev);
    CU(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, cfg->device));
    // sm_90a code loads on compute capability 9.0 only (the "a" features are not forward-compatible)
    if (prop.major != 9 || prop.minor != 0)
        return fail(FA_E_NODEV, "fa_create: device sm_%d%d is not Hopper sm_90 (sm_90a kernels only)", prop.major, prop.minor);

    fa_engine* e = new (std::nothrow) fa_engine();
    if (!e) return fail(FA_E_NOMEM, "fa_create: out of memory");
    struct Guard { fa_engine* e; ~Guard() { if (e) fa_destroy(e); } } guard{e};   // releases everything on any early return
    e->cfg = *cfg;
    e->device = cfg->device;
    e->sm_count = prop.multiProcessorCount;
    e->max_batch = cfg->max_batch ? cfg->max_batch : (1ull << 22);
    if (e->max_batch > (1ull << 28)) e->max_batch = 1ull << 28;
    if (cfg->cuda_stream) { e->stream = (cudaStream_t)cfg->cuda_stream; }
    else { CU(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)); e->own_stream = true; }
    CU(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));

    // table: load factor <= 0.75 at max_entries
    uint64_t want = (4 * cfg->max_entries + 2) / 3;          // 0.75 x 2^k entries get exactly 2^k slots
    uint64_t slots = 1024; while (slots < want) slots <<= 1;
    e->slots = slots;
    if (kmap && slots > (1ull << 30)) return fail(FA_E_INVAL, "fa_create: KERNEL_MAP mode supports at most 2^30 slots");
    const uint32_t feat_flags = FA_F_ENABLE_RTT | FA_F_ENABLE_DNS | FA_F_ENABLE_PKT_DROP;
    if ((cfg->flags & FA_F_NONBLOCKING_EVICT) && !kmap && (cfg->flags & feat_flags))
        return fail(FA_E_INVAL, "fa_create: FA_F_NONBLOCKING_EVICT with feature folds needs mode KERNEL_MAP");
    if (int rc = alloc_table(e, &e->table)) return rc;
    if (cfg->flags & FA_F_NONBLOCKING_EVICT) {
        if (int rc = alloc_table(e, &e->table_spare)) return rc;
        CU(cudaStreamCreateWithFlags(&e->evict_stream, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&e->ev_swap, cudaEventDisableTiming));
        CU(cudaMalloc(&e->d_ctr_ev, sizeof(fa::Counters)));
        CU(cudaMemsetAsync(e->d_ctr_ev, 0, sizeof(fa::Counters), e->stream));
        CU(cudaHostAlloc(&e->h_ev_out, 8, cudaHostAllocDefault));
        e->double_buffered = true;
    }
    if (kmap) {
        CU(cudaMalloc(&e->km_slot_of, e->max_batch * 4));
        uint32_t bs = 1024; while ((uint64_t)bs < 2 * e->max_batch) bs <<= 1;
        e->km_bset_slots = bs;
        CU(cudaMalloc(&e->km_bset, (size_t)bs * sizeof(fa::KmBEntry)));
        CU(cudaMemsetAsync(e->km_bset, 0, (size_t)bs * sizeof(fa::KmBEntry), e->stream));
        CU(cudaMalloc(&e->km_blist, e->max_batch * 4));
        CU(cudaMalloc(&e->km_touched, e->max_batch * 4));
        CU(cudaMalloc(&e->km_deferred, e->max_batch * 4));
        CU(cudaMalloc(&e->km_brec, e->max_batch * 4));
        if (const char* ki = getenv("FA_KMAP_IMPL")) e->km_impl = ki[0] == '1' ? 1 : 2;
        if (cfg->flags & FA_F_RINGBUF_FALLBACK) {
            e->km_spill_cap = 131072;                   // >= the 16 MiB direct_flows ring (bpf/maps_definition.h:7-11)
            CU(cudaMalloc(&e->km_spill, e->km_spill_cap * fa::kRecBytes));
        }
        CU(cudaMalloc(&e->d_km_ctr, sizeof(fa::KmCounters)));
        CU(cudaMemsetAsync(e->d_km_ctr, 0, sizeof(fa::KmCounters), e->stream));
        CU(cudaHostAlloc(&e->h_km_ctr, sizeof(fa::KmCounters), cudaHostAllocDefault));
        memset(e->h_km_ctr, 0, sizeof(fa::KmCounters));
    }
    if (cfg->flags & feat_flags) CU(cudaMalloc(&e->d_slot_of, e->max_batch * 4));
    CU(cudaMalloc(&e->d_ctr, sizeof(fa::Counters)));
    CU(cudaMemsetAsync(e->d_ctr, 0, sizeof(fa::Counters), e->stream));
    CU(cudaHostAlloc(&e->h_ctr, sizeof(fa::Counters), cudaHostAllocDefault));
    memset(e->h_ctr, 0, sizeof(fa::Counters));
    CU(cudaHostAlloc(&e->h_live_ring, fa_engine::kLiveRing * 8, cudaHostAllocMapped));
    if (cfg->mode != FA_MODE_KERNEL_MAP) {
        // with unified addressing (every 64-bit process on sm_90) a mapped pinned buffer has the same address on the device
        unsigned long long* ring = e->h_live_ring;
        CU(cudaMemcpyAsync(&e->d_ctr->live_ring, &ring, sizeof ring, cudaMemcpyHostToDevice, e->stream));
        CU(cudaStreamSynchronize(e->stream));
    }
    for (int i = 0; i < fa_engine::kLiveRing; i++) CU(cudaEventCreateWithFlags(&e->ev_live[i], cudaEventDisableTiming));

    for (int i = 0; i < 2; i++) {
        CU(cudaEventCreateWithFlags(&e->ev_stage_free[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&e->ev_copied[i], cudaEventDisableTiming));
    }
    {
        // one entry per flow that needs the ordered re-fold in a launch: at most one per record, and never more than the
        // table has slots (entries are keyed by table slot)
        uint32_t ss = 1024; while ((uint64_t)ss < 2 * std::min<uint64_t>(e->max_batch, e->slots)) ss <<= 1;
        e->scratch_slots = ss;
        CU(cudaMalloc(&e->d_scratch, (size_t)ss * sizeof(fa::FixupScratch)));
        CU(cudaMemsetAsync(e->d_scratch, 0, (size_t)ss * sizeof(fa::FixupScratch), e->stream));
        CU(cudaStreamSynchronize(e->stream));
    }
    CU(cudaMalloc(&e->d_spill_idx, e->max_batch * sizeof(uint32_t)));
    uint32_t cs = 1024; while ((uint64_t)cs < 2 * e->max_batch) cs <<= 1;
    e->cut_set_slots = cs;
    CU(cudaMalloc(&e->d_cut_set, (size_t)cs * 4));
    CU(cudaMalloc(&e->d_cut_bitmap, (e->max_batch + 31) / 32 * 4 + 4));
    CU(cudaMalloc(&e->d_cut_out, 4));
    CU(cudaHostAlloc(&e->h_cut_out, 4, cudaHostAllocDefault));

    // sketches
    e->sk.log2w = cfg->cms_log2_width ? cfg->cms_log2_width : 20;
    e->sk.depth = cfg->cms_depth ? cfg->cms_depth : 4;
    e->sk.p = cfg->hll_precision ? cfg->hll_precision : 14;
    e->sk.seed = cfg->sketch_seed;
    if (e->sk.depth > 8 || e->sk.log2w < 4 || e->sk.log2w > 30 || e->sk.p < 4 || e->sk.p > 18)
        return fail(FA_E_INVAL, "fa_create: sketch parameters out of range");
    if (cfg->flags & FA_F_ENABLE_SKETCH) {
        const size_t cms_bytes = ((size_t)e->sk.depth << e->sk.log2w) * 8;
        CU(cudaMalloc(&e->sk.cms, cms_bytes));
        CU(cudaMemsetAsync(e->sk.cms, 0, cms_bytes, e->stream));
        CU(cudaMalloc(&e->sk.hll, ((size_t)1 << e->sk.p) * 4));
        CU(cudaMemsetAsync(e->sk.hll, 0, ((size_t)1 << e->sk.p) * 4, e->stream));
    }
    if (const char* ko = getenv("FA_K1_OPT")) e->k1_opt = (uint32_t)strtoul(ko, nullptr, 0);
    if (const char* pp = getenv("FA_PHASE_PROFILE")) {
        if (pp[0] == '1') { CU(cudaMalloc(&e->d_prof, 16 * 8)); CU(cudaMemsetAsync(e->d_prof, 0, 128, e->stream)); }
    }
    CU(cudaStreamSynchronize(e->stream));
    guard.e = nullptr;
    *out = e;
    return FA_OK;
}

void fa_destroy(fa_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->d_prof) {
        unsigned long long p[16];
        if (cudaMemcpy(p, e->d_prof, 128, cudaMemcpyDeviceToHost) == cudaSuccess) {
            static const char* names[8] = {"tile wait", "hash+elect+fold", "S1 barrier", "pipelined probe", "general probe",
                                           "totals", "S2 barrier", "reductions"};
            double tot = 0; for (int i = 0; i < 8; i++) tot += (double)p[i];
            fprintf(stderr, "[flowagg] K1 phase profile (warp-cycles):");
            for (int i = 0; i < 8; i++) fprintf(stderr, " %s %.1f%%;", names[i], tot > 0 ? 100.0 * p[i] / tot : 0.0);
            fprintf(stderr, " total %.3g\n", tot);
            fprintf(stderr, "[flowagg] K1 records %llu: cache hits %.1f%%, representatives %.1f%% (general-loop %.2f%%), cache installs %llu\n",
                    (unsigned long long)e->st.records_ingested, 100.0 * p[8] / (double)std::max<uint64_t>(1, e->st.records_ingested),
                    100.0 * p[9] / (double)std::max<uint64_t>(1, e->st.records_ingested),
                    100.0 * p[10] / (double)std::max<uint64_t>(1, e->st.records_ingested), p[11]);
            fprintf(stderr, "[flowagg] K1 probes: home-slot collisions %llu, resolved one slot on %llu, unsettled at first probe %llu\n", p[12], p[13], p[14]);
        }
        cudaFree(e->d_prof);
    }
    if (e->copy_stream) { cudaStreamSynchronize(e->copy_stream); cudaStreamDestroy(e->copy_stream); }
    { std::lock_guard<std::mutex> elk(e->evict_mu); }      // an fa_evict still scanning a retired table returns first
    if (e->evict_stream) { cudaStreamSynchronize(e->evict_stream); cudaStreamDestroy(e->evict_stream); }
    if (e->ev_swap) cudaEventDestroy(e->ev_swap);
    free_table(&e->table_spare); cudaFree(e->d_ctr_ev);
    if (e->h_ev_out) cudaFreeHost(e->h_ev_out);
    free_table(&e->table);
    cudaFree(e->d_ctr); if (e->h_ctr) cudaFreeHost(e->h_ctr);
    if (e->h_live_ring) cudaFreeHost(e->h_live_ring);
    for (int i = 0; i < fa_engine::kLiveRing; i++) if (e->ev_live[i]) cudaEventDestroy(e->ev_live[i]);
    for (int i = 0; i < 2; i++) {
        cudaFree(e->d_stage[i]); if (e->h_stage[i]) cudaFreeHost(e->h_stage[i]);
        if (e->ev_stage_free[i]) cudaEventDestroy(e->ev_stage_free[i]);
        if (e->ev_copied[i]) cudaEventDestroy(e->ev_copied[i]);
    }
    cudaFree(e->d_scratch); cudaFree(e->d_spill_idx); cudaFree(e->d_cut_set); cudaFree(e->d_cut_bitmap); cudaFree(e->d_cut_out);
    if (e->h_cut_out) cudaFreeHost(e->h_cut_out);
    cudaFree(e->d_route_tmp); cudaFree(e->d_route_counts); cudaFree(e->d_expanded);
    cudaFree(e->d_sroute_hist); cudaFree(e->d_sroute_tot);
    cudaFree(e->d_snap_src); cudaFree(e->d_snap_cnt); cudaFree(e->d_snap_verdict);
    free_staging(&e->evict_stage); free_staging(&e->top_stage); cudaFree(e->d_slot_of);
    cudaFree(e->top.state); cudaFree(e->top.hist); cudaFree(e->top.ents); if (e->h_top_state) cudaFreeHost(e->h_top_state);
    free_staging(&e->lookup_stage); cudaFree(e->d_lookup_slot); cudaFree(e->d_lookup_found); cudaFree(e->d_lookup_hits);
    if (e->h_lookup_hits) cudaFreeHost(e->h_lookup_hits);
    free_staging(&e->expire_stage); cudaFree(e->expire.bm); cudaFree(e->expire.list); cudaFree(e->expire.ctr);
    if (e->h_expire_ctr) cudaFreeHost(e->h_expire_ctr);
    cudaFree(e->group.tab); cudaFree(e->group.list); cudaFree(e->group.ctr); cudaFree(e->d_group_out);
    if (e->h_group_ctr) cudaFreeHost(e->h_group_ctr);
    cudaFree(e->d_hist_row_of); cudaFree(e->d_hist_out);
    cudaFree(e->distinct.tab); cudaFree(e->distinct.list); cudaFree(e->distinct.ctr); cudaFree(e->d_distinct_out);
    if (e->h_distinct_ctr) cudaFreeHost(e->h_distinct_ctr);
    cudaFree(e->sk.cms); cudaFree(e->sk.hll);
    cudaFree(e->dnsc.tab); cudaFree(e->dnsc_spare); cudaFree(e->dnsc.ctr); cudaFreeHost(e->h_dnsc_ctr);
    cudaFree(e->d_dnsc_state); cudaFree(e->d_dnsc_samples); cudaFree(e->d_dnsc_out); cudaFree(e->d_dnsc_warps);
    cudaFree(e->km_slot_of); cudaFree(e->km_bset); cudaFree(e->km_blist); cudaFree(e->km_spill);
    cudaFree(e->km_touched); cudaFree(e->km_deferred); cudaFree(e->km_brec);
    cudaFree(e->d_km_ctr); if (e->h_km_ctr) cudaFreeHost(e->h_km_ctr);
    cudaFree(e->d_pb_sizes); cudaFree(e->d_pb_offsets); cudaFree(e->d_pb_sums); cudaFree(e->d_pb_ifaces);
    if (e->own_stream && e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

int fa_ingest(fa_engine* e, const void* recs, size_t n, size_t* consumed) {
    if (consumed) *consumed = 0;
    if (!e) return fail(FA_E_INVAL, "fa_ingest: null engine");
    if (n == 0) return FA_OK;
    if (!recs) return fail(FA_E_INVAL, "fa_ingest: null records");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    // device records are folded in one go (ingest_device launches by max_batch); host records stage by stage
    Input in(e, recs, n, fa::kRecBytes, SIZE_MAX, stage_records(e), WINDOW_HOST);
    if (in.misaligned(16)) return fail(FA_E_INVAL, "fa_ingest: device records must be 16-byte aligned");
    int rc = FA_OK;
    while (rc == FA_OK && in.more()) {
        const uint8_t* d_recs = nullptr;
        uint64_t c = 0;
        size_t took = 0;
        if (int src_rc = in.next(&d_recs, &c)) return src_rc;
        rc = ingest_device(e, d_recs, c, &took);
        if (int rel_rc = in.release()) return rel_rc;
        in.advance(took);
    }
    return in.finish(rc, consumed);
}

int fa_ingest_events(fa_engine* e, const void* events, size_t n, size_t* consumed) {
    if (consumed) *consumed = 0;
    if (!e) return fail(FA_E_INVAL, "fa_ingest_events: null engine");
    if (n == 0) return FA_OK;
    if (!events) return fail(FA_E_INVAL, "fa_ingest_events: null events");
    static_assert(sizeof(fa_packet_event) == 64, "fa_packet_event ABI");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    Input in(e, events, n, 64, e->max_batch, stage_records(e), WINDOW_ALL);
    if (in.misaligned(16)) return fail(FA_E_INVAL, "fa_ingest_events: device events must be 16-byte aligned");
    if (!e->d_expanded) CU(cudaMalloc(&e->d_expanded, e->max_batch * fa::kRecBytes));
    // the expansion and K1 of successive chunks are ordered on the engine's stream, so one d_expanded is enough
    int rc = FA_OK;
    while (rc == FA_OK && in.more()) {
        const uint8_t* d_ev = nullptr;
        uint64_t c = 0;
        size_t took = 0;
        if (int src_rc = in.next(&d_ev, &c)) return src_rc;
        e->st.kernel_launches += fa::launch_expand_events(reinterpret_cast<const uint4*>(d_ev), c, reinterpret_cast<uint4*>(e->d_expanded), e->stream);
        CU(cudaGetLastError());
        if (int rel_rc = in.release()) return rel_rc;
        rc = ingest_device(e, e->d_expanded, c, &took);
        in.advance(took);
    }
    return in.finish(rc, consumed);
}

int fa_ingest_snaps(fa_engine* e, const void* snaps, size_t n, uint32_t stride, size_t* consumed) {
    if (consumed) *consumed = 0;
    if (!e) return fail(FA_E_INVAL, "fa_ingest_snaps: null engine");
    if (stride < 40 || stride > 152 || (stride & 7)) return fail(FA_E_INVAL, "fa_ingest_snaps: stride %u must be a multiple of 8 in 40..152", stride);
    if (n == 0) return FA_OK;
    if (!snaps) return fail(FA_E_INVAL, "fa_ingest_snaps: null snapshots");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    // host chunks are bounded by the staging buffers (stage_records() x 144 bytes), device chunks by max_batch records
    Input in(e, snaps, n, stride, e->max_batch, std::min<uint64_t>(e->max_batch, stage_records(e) * fa::kRecBytes / stride), WINDOW_NONE);
    if (in.misaligned(8)) return fail(FA_E_INVAL, "fa_ingest_snaps: device snapshots must be 8-byte aligned");
    if (!e->d_expanded) CU(cudaMalloc(&e->d_expanded, e->max_batch * fa::kRecBytes));
    if (!e->d_snap_src) CU(cudaMalloc(&e->d_snap_src, e->max_batch * sizeof(uint32_t)));
    if (!e->d_snap_cnt) CU(cudaMalloc(&e->d_snap_cnt, (fa::kSnapMaxCtas + 8) * sizeof(uint32_t)));
    if (e->filter.n_rules && !e->d_snap_verdict) CU(cudaMalloc(&e->d_snap_verdict, e->max_batch));
    unsigned long long* d_total = reinterpret_cast<unsigned long long*>(e->d_snap_cnt + fa::kSnapMaxCtas);
    int rc = FA_OK;
    while (in.more()) {
        const uint8_t* d_sn = nullptr;
        uint64_t c = 0;
        if (int src_rc = in.next(&d_sn, &c)) return src_rc;
        CU(cudaMemsetAsync(d_total + 1, 0, 24, e->stream));             // the filter's three counters of this chunk
        e->st.kernel_launches += fa::launch_parse_snaps(d_sn, c, stride, &e->filter, e->d_snap_cnt, e->d_snap_verdict,
                                                        reinterpret_cast<uint4*>(e->d_expanded), e->d_snap_src, d_total, d_total + 1,
                                                        e->sm_count, e->stream);
        CU(cudaGetLastError());
        if (int rel_rc = in.release()) return rel_rc;
        // how many packets were submitted decides the launch sizes of the fold: one 8-byte read-back per chunk
        unsigned long long back[4] = {0, 0, 0, 0};                      // submitted + kept | filter accept / reject / no match
        CU(cudaMemcpyAsync(back, d_total, 32, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        const uint32_t m = (uint32_t)back[0];
        e->st.filter_accept += back[1]; e->st.filter_reject += back[2]; e->st.filter_nomatch += back[3];
        // every submitted packet bumps exactly one of the three counters: what the filter skipped = submitted - kept
        const uint64_t filtered_out = e->filter.n_rules ? back[1] + back[2] + back[3] - (uint64_t)m : 0;
        size_t off = 0;
        rc = ingest_device(e, e->d_expanded, m, &off);
        if (rc == FA_FULL && off < m) {
            // the cut is reported in snapshots: everything before the first record that was not folded, discarded ones included
            uint32_t first_left = 0;
            CU(cudaMemcpyAsync(&first_left, e->d_snap_src + off, 4, cudaMemcpyDeviceToHost, e->stream));
            CU(cudaStreamSynchronize(e->stream));
            // discarded snapshots before the cut: first_left - off
            // (with a filter the discarded / filtered split of a partially consumed chunk is not known: both count as discarded)
            e->st.snaps_ingested += first_left;
            e->st.snaps_discarded += first_left - off;
            in.advance(first_left);
            break;
        }
        if (rc != FA_OK) break;
        e->st.snaps_ingested += c;
        e->st.snaps_discarded += c - m - filtered_out;                  // fill_ethhdr's DISCARDs; the filter's skips are in its counters
        in.advance(c);
    }
    return in.finish(rc, consumed);
}

int fa_set_flow_filter(fa_engine* e, const fa_filter_rule* rules, size_t n_rules, const fa_filter_cidr* peers, size_t n_peers) {
    if (!e) return fail(FA_E_INVAL, "fa_set_flow_filter: null engine");
    static_assert(sizeof(fa_filter_rule) == 64 && sizeof(fa_filter_cidr) == 20, "filter ABI");
    if (n_rules > (size_t)fa::kMaxFilterEntries || n_peers > (size_t)fa::kMaxFilterEntries)
        return fail(FA_E_INVAL, "fa_set_flow_filter: at most %d rules and %d peer CIDRs (MAX_FILTER_ENTRIES)", fa::kMaxFilterEntries, fa::kMaxFilterEntries);
    if ((n_rules && !rules) || (n_peers && !peers)) return fail(FA_E_INVAL, "fa_set_flow_filter: null table");
    std::lock_guard<std::mutex> lk(e->mu);
    fa::FilterSet F{};
    auto words = [](const uint8_t ip[16], uint32_t w[4]) {
        for (int i = 0; i < 4; i++) w[i] = ((uint32_t)ip[4 * i] << 24) | ((uint32_t)ip[4 * i + 1] << 16) | ((uint32_t)ip[4 * i + 2] << 8) | ip[4 * i + 3];
    };
    for (size_t i = 0; i < n_rules; i++) {
        const fa_filter_rule& r = rules[i];
        if (r.prefix_len > 128 || r.direction > 2 || r.action > 2) return fail(FA_E_INVAL, "fa_set_flow_filter: rule %zu out of range", i);
        fa::FilterRuleDev& d = F.rules[i];
        words(r.ip, d.ipw); d.prefix = r.prefix_len; d.sample = r.sample;
        d.dps = r.dst_port_start; d.dpe = r.dst_port_end; d.dp1 = r.dst_port1; d.dp2 = r.dst_port2;
        d.sps = r.src_port_start; d.spe = r.src_port_end; d.sp1 = r.src_port1; d.sp2 = r.src_port2;
        d.ps = r.port_start; d.pe = r.port_end; d.p1 = r.port1; d.p2 = r.port2; d.tcp_flags = r.tcp_flags;
        d.proto = r.protocol; d.icmp_type = r.icmp_type; d.icmp_code = r.icmp_code; d.direction = r.direction; d.action = r.action;
        d.filter_drops = r.filter_drops; d.peer = r.do_peer_cidr_lookup;
    }
    for (size_t i = 0; i < n_peers; i++) {
        if (peers[i].prefix_len > 128) return fail(FA_E_INVAL, "fa_set_flow_filter: peer CIDR %zu out of range", i);
        words(peers[i].ip, F.peers[i].ipw); F.peers[i].prefix = peers[i].prefix_len;
    }
    F.n_rules = (uint32_t)n_rules; F.n_peers = (uint32_t)n_peers;
    e->filter = F;
    return FA_OK;
}

// Feature samples may create flows: refuse n more (`what`: samples or packets) when they could take the table past 7/8
// of its slots.
static int check_sample_room(fa_engine* e, size_t n, const char* who, const char* what) {
    if (int rc = sync_counters(e)) return rc;
    if (e->live_known + n > e->slots - e->slots / 8)
        return fail(FA_E_2BIG, "%s: %zu %s could overfill the flow table (%llu live of %llu slots): evict first", who, n, what,
                    (unsigned long long)e->live_known, (unsigned long long)e->slots);
    return FA_OK;
}

// Fold m device-resident feature samples of `kind` (0 additional, 1 DNS, 2 packet drops) into the table.
static int fold_samples(fa_engine* e, int kind, const uint8_t* d_samples, uint32_t m) {
    e->st.kernel_launches += fa::launch_feature_fold(kind, d_samples, m, e->table, ++e->epoch, e->feat_seq[kind], e->d_slot_of,
                                                     e->d_ctr, e->sm_count, e->stream);
    CU(cudaGetLastError());
    e->feat_seq[kind] += m;
    e->unsynced_records += m;
    (kind == 0 ? e->st.additional_ingested : kind == 1 ? e->st.dns_ingested : e->st.pkt_drops_ingested) += m;
    return FA_OK;
}

static int ingest_feature(fa_engine* e, int kind, const void* recs, size_t n, const char* who) {
    const uint32_t flag = kind == 0 ? FA_F_ENABLE_RTT : kind == 1 ? FA_F_ENABLE_DNS : FA_F_ENABLE_PKT_DROP;
    if (!e) return fail(FA_E_INVAL, "%s: null engine", who);
    if (!(e->cfg.flags & flag)) return fail(FA_E_INVAL, "%s: engine was created without %s", who, kind == 0 ? "FA_F_ENABLE_RTT" : kind == 1 ? "FA_F_ENABLE_DNS" : "FA_F_ENABLE_PKT_DROP");
    if (n == 0) return FA_OK;
    if (!recs) return fail(FA_E_INVAL, "%s: null records", who);
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const size_t rec_bytes = kind == 1 ? fa::kDnsRecBytes : fa::kAddRecBytes;      // additional and packet-drop samples: 72 B
    Input in(e, recs, n, rec_bytes, e->max_batch, stage_records(e), WINDOW_NONE);
    if (in.misaligned(8)) return fail(FA_E_INVAL, "%s: device records must be 8-byte aligned", who);
    if (int rc = check_sample_room(e, n, who, "samples")) return rc;
    while (in.more()) {
        const uint8_t* d = nullptr;
        uint64_t c = 0;
        if (int rc = in.next(&d, &c)) return rc;
        if (int rc = fold_samples(e, kind, d, c)) return rc;
        if (int rc = in.release()) return rc;
        in.advance(c);
    }
    return in.finish(FA_OK, nullptr);
}

int fa_ingest_additional(fa_engine* e, const void* recs, size_t n) { return ingest_feature(e, 0, recs, n, "fa_ingest_additional"); }
int fa_ingest_dns(fa_engine* e, const void* recs, size_t n) { return ingest_feature(e, 1, recs, n, "fa_ingest_dns"); }
int fa_ingest_pkt_drops(fa_engine* e, const void* recs, size_t n) { return ingest_feature(e, 2, recs, n, "fa_ingest_pkt_drops"); }

int fa_live_flows(fa_engine* e, size_t* n) {
    if (!e || !n) return fail(FA_E_INVAL, "fa_live_flows: null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    int rc = sync_counters(e);
    if (rc) return rc;
    *n = (size_t)e->live_known;
    return FA_OK;
}

// Device staging of the host-bound blocks of fa_evict_ex / fa_top_flows and the slot list of the feature pass, grown
// on demand to hold n rows.  Eviction and fa_top_flows each have their own, never touched by fa_ingest*.
static int grow_staging(fa_engine* e, fa_engine::Staging* s, uint64_t n, bool records, bool feats) {
    const uint64_t want = std::max<uint64_t>(n, std::min<uint64_t>(e->cfg.max_entries, n * 2));
    if (records && s->cap < n) {
        cudaFree(s->rec); s->rec = nullptr; s->cap = 0;
        CU(cudaMalloc(&s->rec, want * fa::kRecBytes));
        s->cap = want;
    }
    if (feats && s->feat_cap < n) {
        cudaFree(s->dns); cudaFree(s->add); cudaFree(s->present); cudaFree(s->slot_of); cudaFree(s->drop); cudaFree(s->rttmin);
        s->dns = s->add = s->present = s->drop = nullptr; s->rttmin = nullptr; s->slot_of = nullptr; s->feat_cap = 0;
        CU(cudaMalloc(&s->dns, want * 64)); CU(cudaMalloc(&s->add, want * 32));
        CU(cudaMalloc(&s->drop, want * 32)); CU(cudaMalloc(&s->rttmin, want * 8));
        CU(cudaMalloc(&s->present, want)); CU(cudaMalloc(&s->slot_of, want * 4));
        s->feat_cap = want;
    }
    return FA_OK;
}

// Where the kernels write the n rows of each block of `o` for table `t`: device blocks in place, host blocks in the
// staging `s` (grown by grow_staging).  Every requested block the table does not produce is zeroed where it lives.
struct Blocks { uint8_t *rec, *dns, *add, *drop, *rmin, *pres; uint32_t* slot_of; };
static int place_blocks(const fa::Table& t, const fa_evict_out* o, uint64_t n, const fa_engine::Staging& s, cudaStream_t st,
                        Blocks* d) {
    const bool feats = t.feat_add || t.feat_dns || t.feat_drop;
    auto dev = [](void* p, void* staging) -> uint8_t* {          // where the kernels write a block
        return static_cast<uint8_t*>(p && classify(p) != PTR_DEVICE ? staging : p);
    };
    *d = Blocks{};
    d->rec = dev(o->records, s.rec);
    if (feats) {
        d->dns = dev(o->dns, s.dns); d->add = dev(o->additional, s.add); d->drop = dev(o->pkt_drops, s.drop);
        d->rmin = dev(o->rtt_min, s.rttmin); d->pres = dev(o->present, s.present);
        d->slot_of = s.slot_of;
        // the block of a feature this engine does not fold is zeroed where the kernels write (the feature pass does not
        // write it) and copied like the others
        if (d->dns && !t.feat_dns) CU(cudaMemsetAsync(d->dns, 0, n * 64, st));
        if (d->add && !t.feat_add) CU(cudaMemsetAsync(d->add, 0, n * 32, st));
        if (d->drop && !t.feat_drop) CU(cudaMemsetAsync(d->drop, 0, n * 32, st));
    } else {
        // no feature pass: every feature block is zeroed where it is
        const struct { void* p; size_t width; } unmade[5] = {
            {o->dns, 64}, {o->additional, 32}, {o->pkt_drops, 32}, {o->rtt_min, 8}, {o->present, 1}};
        for (const auto& b : unmade) {
            if (!b.p) continue;
            if (classify(b.p) == PTR_DEVICE) CU(cudaMemsetAsync(b.p, 0, n * b.width, st));
            else memset(b.p, 0, n * b.width);
        }
    }
    return FA_OK;
}

// After the kernels: the feature pass over the n rows (when `t` has feature lines; clear = false leaves them as they
// are), then the copies of the blocks that are host memory.  Adds the kernels launched and the bytes copied.
static int finish_blocks(fa_engine* e, const fa::Table& t, const fa_evict_out* o, uint64_t n, const Blocks& d, bool clear,
                         cudaStream_t st, uint64_t* launches, uint64_t* d2h) {
    if (t.feat_add || t.feat_dns || t.feat_drop)
        *launches += (clear ? fa::launch_evict_features : fa::launch_peek_features)(
            t, d.slot_of, n, d.rec, d.dns, d.add, d.drop, reinterpret_cast<unsigned long long*>(d.rmin), d.pres, e->sm_count, st);
    CU(cudaGetLastError());
    const struct { void* host; const uint8_t* src; size_t width; } blocks[6] = {
        {o->records, d.rec, fa::kRecBytes}, {o->dns, d.dns, 64}, {o->additional, d.add, 32}, {o->pkt_drops, d.drop, 32},
        {o->rtt_min, d.rmin, 8}, {o->present, d.pres, 1}};
    for (const auto& b : blocks) {
        if (!b.host || !b.src || b.src == b.host) continue;        // not asked for, not produced, or written in place
        CU(cudaMemcpyAsync(b.host, b.src, n * b.width, cudaMemcpyDeviceToHost, st));
        *d2h += n * b.width;
    }
    return FA_OK;
}

// Lookup-and-delete the `live` flows of `t` into the blocks of `o`, on stream `st`: the table scan (K2, or the
// KERNEL_MAP scan) with ctr->evict_out as its cursor, the feature pass when `t` has feature lines, then the copies of
// the blocks that are host memory.  Adds the kernels launched and the bytes copied.
static int evict_scan(fa_engine* e, const fa::Table& t, const fa_evict_out* o, uint64_t live, fa::Counters* ctr,
                      cudaStream_t st, uint64_t* launches, uint64_t* d2h) {
    Blocks d;
    if (int rc = place_blocks(t, o, live, e->evict_stage, st, &d)) return rc;
    if (e->cfg.mode == FA_MODE_KERNEL_MAP)
        *launches += fa::launch_kmap_evict(t, t.met, d.rec, live, &ctr->evict_out, d.slot_of, e->sm_count, st);
    else
        *launches += fa::launch_evict(t, reinterpret_cast<uint4*>(d.rec), d.slot_of, live, ctr, e->sm_count, st);
    return finish_blocks(e, t, o, live, d, /*clear=*/true, st, launches, d2h);
}

// Lookup-and-delete every flow.  Blocking: the live table is scanned on the engine stream under `mu`.
// FA_F_NONBLOCKING_EVICT: the tables are swapped under `mu` (fa_ingest* goes on at once, into the empty one), then the
// retired table is scanned on the eviction stream, with its own cursor and staging, under `evict_mu` alone; only the
// launches queued before the swap are waited for.  Not swapped: the DNS correlation table, the fallback ring, the
// KERNEL_MAP counters.
int fa_evict_ex(fa_engine* e, const fa_evict_out* o, size_t cap, size_t* n_out) {
    if (n_out) *n_out = 0;
    if (!e || !n_out || !o) return fail(FA_E_INVAL, "fa_evict: null argument");
    const bool swap = e->double_buffered;
    std::unique_lock<std::mutex> elk(e->evict_mu, std::defer_lock);   // one eviction at a time
    if (swap) elk.lock();
    std::unique_lock<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    if (int rc = sync_counters(e)) return rc;          // the queued folds finish; exact live count
    const uint64_t live = e->live_known;
    e->st.evictions++;
    if (live == 0) return FA_OK;
    if (!o->records) return fail(FA_E_INVAL, "fa_evict: null out_records");
    if (cap < live) return fail(FA_E_2BIG, "fa_evict: capacity %zu < %llu live flows", cap, (unsigned long long)live);
    const fa::Table t = e->table;
    fa::Counters* ctr = e->d_ctr;
    cudaStream_t st = e->stream;
    if (swap) {
        std::swap(e->table, e->table_spare);           // the spare is empty: the previous eviction deleted every flow in place
        CU(cudaMemsetAsync(&e->d_ctr->live, 0, sizeof(unsigned long long), e->stream));
        CU(cudaEventRecord(e->ev_swap, e->stream));
        set_live_known(e, 0);
        e->st.flows_evicted += live;
        lk.unlock();                                   // from here on fa_ingest* runs concurrently, into the new table
        ctr = e->d_ctr_ev;
        st = e->evict_stream;
    }
    const bool feats = t.feat_add || t.feat_dns || t.feat_drop;
    if (int rc = grow_staging(e, &e->evict_stage, live, classify(o->records) != PTR_DEVICE, feats)) return rc;
    if (swap) CU(cudaStreamWaitEvent(st, e->ev_swap, 0));
    CU(cudaMemsetAsync(&ctr->evict_out, 0, sizeof(unsigned long long), st));
    uint64_t launched = 0, d2h = 0;
    if (int rc = evict_scan(e, t, o, live, ctr, st, &launched, &d2h)) return rc;
    const unsigned long long* found = e->h_ev_out;
    if (swap) {
        CU(cudaMemcpyAsync(e->h_ev_out, &ctr->evict_out, 8, cudaMemcpyDeviceToHost, st));
    } else {
        CU(cudaMemsetAsync(&e->d_ctr->live, 0, sizeof(unsigned long long), st));
        CU(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(fa::Counters), cudaMemcpyDeviceToHost, st));
        found = &e->h_ctr->evict_out;
    }
    CU(cudaStreamSynchronize(st));
    if (*found != live)
        return fail(FA_E_CUDA, "fa_evict: table scan found %llu flows, counter says %llu", *found, (unsigned long long)live);
    if (swap) {
        lk.lock();
    } else {
        set_live_known(e, 0);
        e->st.flows_evicted += live;
    }
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    *n_out = (size_t)live;
    return FA_OK;
}

int fa_evict(fa_engine* e, void* out_records, void* out_dns, void* out_additional, uint8_t* out_present,
             size_t cap, size_t* n_out) {
    fa_evict_out o{};
    o.records = out_records; o.dns = out_dns; o.additional = out_additional; o.present = out_present;
    return fa_evict_ex(e, &o, cap, n_out);
}

// The exact top-k live flows by bytes or packets, read in place (evict.cu: launch_top_flows).  The select, the
// compaction, the sort and the gather run on the engine stream after the queued folds; the feature pass runs with
// clear = false.  Nothing of the table or the counters is written.
int fa_top_flows(fa_engine* e, uint32_t by, size_t k, const fa_evict_out* o, size_t* n_out) {
    if (n_out) *n_out = 0;
    if (!e || !o || !o->records || !n_out) return fail(FA_E_INVAL, "fa_top_flows: null argument");
    if (by != FA_TOP_BYTES && by != FA_TOP_PACKETS) return fail(FA_E_INVAL, "fa_top_flows: unknown metric %u", by);
    if (k == 0 || k > FA_TOP_MAX_K) return fail(FA_E_INVAL, "fa_top_flows: k = %zu not in [1, %u]", k, FA_TOP_MAX_K);
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    if (int rc = sync_counters(e)) return rc;          // the queued folds finish; exact live count
    const uint64_t live = e->live_known;
    const uint64_t n = std::min<uint64_t>(k, live);
    if (n == 0) return FA_OK;
    const fa::Table t = e->table;
    const bool kmap = e->cfg.mode == FA_MODE_KERNEL_MAP;
    const bool feats = t.feat_add || t.feat_dns || t.feat_drop;
    cudaStream_t st = e->stream;
    // FA_TOP_SLACK (diagnostics, tests): the room beyond k; a small one makes small tables run the digit passes
    uint64_t slack = fa::kTopSlack;
    if (const char* ts = getenv("FA_TOP_SLACK")) slack = strtoull(ts, nullptr, 0);
    uint64_t cap = fa::kTopSortTile;
    while (cap < n + slack) cap <<= 1;
    if (e->top.cap < cap) {
        cudaFree(e->top.ents); e->top.ents = nullptr; e->top.cap = 0;
        CU(cudaMalloc(&e->top.ents, cap * sizeof(fa::TopEnt)));
        e->top.cap = cap;
    }
    if (!e->top.state) {
        CU(cudaMalloc(&e->top.state, sizeof(fa::TopState)));
        CU(cudaMalloc(&e->top.hist, fa::kTopPasses * 256 * sizeof(unsigned)));
        CU(cudaHostAlloc(&e->h_top_state, sizeof(fa::TopState), cudaHostAllocDefault));
    }
    fa::TopScratch s = e->top;
    s.cap = cap;                                       // a larger scratch from an earlier call: sort only what is needed
    if (int rc = grow_staging(e, &e->top_stage, n, classify(o->records) != PTR_DEVICE, feats)) return rc;
    Blocks d;
    if (int rc = place_blocks(t, o, n, e->top_stage, st, &d)) return rc;
    CU(cudaMemsetAsync(s.state, 0, sizeof(fa::TopState), st));
    CU(cudaMemsetAsync(s.hist, 0, fa::kTopPasses * 256 * sizeof(unsigned), st));
    uint64_t launched = 0, d2h = 0;
    launched += fa::launch_top_flows(t, kmap, by == FA_TOP_BYTES, n, live, s, d.rec, d.slot_of, e->sm_count, st);
    if (int rc = finish_blocks(e, t, o, n, d, /*clear=*/false, st, &launched, &d2h)) return rc;
    CU(cudaMemcpyAsync(e->h_top_state, s.state, sizeof(fa::TopState), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (e->h_top_state->overflow || e->h_top_state->count < n)
        return fail(FA_E_CUDA, "fa_top_flows: %llu candidates for %llu rows in a scratch of %llu (more than %llu flows tie with the "
                    "k-th in metric and key premix)", e->h_top_state->count, (unsigned long long)n, (unsigned long long)cap,
                    (unsigned long long)(cap - n));
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    *n_out = (size_t)n;
    return FA_OK;
}

// Exact point lookups of live flows by key, read in place (evict.cu: launch_lookup_flows).  Chunk by chunk on the engine
// stream after the queued folds: the keys reach the device through Input, the probe writes each key's slot (or kNoSlot)
// and counts the hits on the device, the gather and the feature pass (clear = false) fill the chunk's rows of every
// block.  Device scratch and staging hold one chunk; one wait at the end.  Nothing of the table or the counters is written.
int fa_lookup_flows(fa_engine* e, const void* keys, size_t n, const fa_evict_out* o, uint8_t* found, size_t* n_found) {
    if (!e || !o || !o->records || !n_found || (!keys && n)) return fail(FA_E_INVAL, "fa_lookup_flows: null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const uint64_t chunk = stage_records(e);
    Input in(e, keys, n, fa::kKeyBytes, chunk, chunk, WINDOW_NONE);
    if (n && in.misaligned(8)) return fail(FA_E_INVAL, "fa_lookup_flows: device keys must be 8-byte aligned");
    *n_found = 0;
    if (n == 0) return FA_OK;
    const fa::Table t = e->table;
    const bool kmap = e->cfg.mode == FA_MODE_KERNEL_MAP;
    const bool feats = t.feat_add || t.feat_dns || t.feat_drop;
    const bool found_dev = found && classify(found) == PTR_DEVICE;
    cudaStream_t st = e->stream;
    const uint64_t rows = std::min<uint64_t>(n, chunk);
    if (int rc = grow_staging(e, &e->lookup_stage, rows, classify(o->records) != PTR_DEVICE, feats)) return rc;
    if (e->lookup_cap < rows) {
        cudaFree(e->d_lookup_slot); cudaFree(e->d_lookup_found);
        e->d_lookup_slot = nullptr; e->d_lookup_found = nullptr; e->lookup_cap = 0;
        CU(cudaMalloc(&e->d_lookup_slot, rows * 4)); CU(cudaMalloc(&e->d_lookup_found, rows));
        e->lookup_cap = rows;
    }
    if (!e->d_lookup_hits) {
        CU(cudaMalloc(&e->d_lookup_hits, 8));
        CU(cudaHostAlloc(&e->h_lookup_hits, 8, cudaHostAllocDefault));
    }
    CU(cudaMemsetAsync(e->d_lookup_hits, 0, 8, st));
    uint64_t launched = 0, d2h = 0;
    while (in.more()) {
        const uint8_t* d_keys = nullptr;
        uint64_t c = 0;
        if (int rc = in.next(&d_keys, &c)) return rc;
        const size_t at = in.done;
        auto row = [at](void* p, size_t width) { return p ? static_cast<uint8_t*>(p) + at * width : nullptr; };
        fa_evict_out oc{};                             // the chunk's rows of every block
        oc.records = row(o->records, fa::kRecBytes); oc.dns = row(o->dns, 64); oc.additional = row(o->additional, 32);
        oc.pkt_drops = row(o->pkt_drops, 32); oc.rtt_min = reinterpret_cast<uint64_t*>(row(o->rtt_min, 8));
        oc.present = row(o->present, 1);
        Blocks d;
        if (int rc = place_blocks(t, &oc, c, e->lookup_stage, st, &d)) return rc;
        d.slot_of = e->d_lookup_slot;                  // the feature pass reads the probe's slots (kNoSlot: zero rows)
        uint8_t* d_found = found_dev ? found + at : found ? e->d_lookup_found : nullptr;
        launched += fa::launch_lookup_flows(t, kmap, reinterpret_cast<const uint64_t*>(d_keys), c, e->d_lookup_slot, d_found,
                                            e->d_lookup_hits, d.rec, e->sm_count, st);
        if (int rc = in.release()) return rc;
        if (int rc = finish_blocks(e, t, &oc, c, d, /*clear=*/false, st, &launched, &d2h)) return rc;
        if (found && !found_dev) {
            CU(cudaMemcpyAsync(found + at, d_found, c, cudaMemcpyDeviceToHost, st));
            d2h += c;
        }
        in.advance(c);
    }
    CU(cudaMemcpyAsync(e->h_lookup_hits, e->d_lookup_hits, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (int rc = in.finish(FA_OK, nullptr)) return rc;
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    *n_found = (size_t)*e->h_lookup_hits;
    return FA_OK;
}

// Remove only the live flows past an idle or active timeout (evict.cu: launch_expire_*), on the engine stream after the
// queued folds: the mark writes the expire bitmap and slot list and counts them (one wait, to check cap), the gather and
// the clearing feature pass emit their rows, then the delete pass removes them and compacts their clusters in place.
// Every other flow stays live, bit for bit.  FA_F_NONBLOCKING_EVICT: the live table only; the spare stays empty.
int fa_expire_flows(fa_engine* e, uint64_t mono_now_ns, uint64_t idle_timeout_ns, uint64_t active_timeout_ns,
                    const fa_evict_out* o, size_t cap, size_t* n_out) {
    if (n_out) *n_out = 0;
    if (!e || !o || !o->records || !n_out) return fail(FA_E_INVAL, "fa_expire_flows: null argument");
    if (!idle_timeout_ns && !active_timeout_ns) return fail(FA_E_INVAL, "fa_expire_flows: both timeouts are zero");
    if (idle_timeout_ns > (uint64_t)INT64_MAX || active_timeout_ns > (uint64_t)INT64_MAX)
        return fail(FA_E_INVAL, "fa_expire_flows: a timeout above INT64_MAX");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    if (int rc = sync_counters(e)) return rc;          // the queued folds finish; exact live count
    const uint64_t live = e->live_known;
    if (live == 0) { e->st.evictions++; return FA_OK; }
    const fa::Table t = e->table;
    const bool kmap = e->cfg.mode == FA_MODE_KERNEL_MAP;
    const bool feats = t.feat_add || t.feat_dns || t.feat_drop;
    cudaStream_t st = e->stream;
    if (!e->expire.bm) {
        CU(cudaMalloc(&e->expire.bm, e->slots / 8));
        CU(cudaMalloc(&e->expire.ctr, sizeof(fa::ExpireCtr)));
        CU(cudaHostAlloc(&e->h_expire_ctr, sizeof(fa::ExpireCtr), cudaHostAllocDefault));
    }
    if (e->expire.cap < live) {                        // room for every live flow: the list never overflows
        cudaFree(e->expire.list); e->expire.list = nullptr; e->expire.cap = 0;
        const uint64_t want = std::max<uint64_t>(live, std::min<uint64_t>(e->slots, 2 * live));
        CU(cudaMalloc(&e->expire.list, want * 4));
        e->expire.cap = want;
    }
    const fa::ExpireScratch s = e->expire;
    CU(cudaMemsetAsync(s.ctr, 0, sizeof(fa::ExpireCtr), st));
    uint64_t launched = fa::launch_expire_mark(t, mono_now_ns, idle_timeout_ns, active_timeout_ns, s, e->sm_count, st);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(e->h_expire_ctr, s.ctr, sizeof(fa::ExpireCtr), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint64_t n = e->h_expire_ctr->n;
    if (n > live) return fail(FA_E_CUDA, "fa_expire_flows: the mark found %llu flows, counter says %llu live", (unsigned long long)n,
                              (unsigned long long)live);
    if (n > cap) {
        *n_out = (size_t)n;
        return fail(FA_E_2BIG, "fa_expire_flows: capacity %zu < %llu expiring flows", cap, (unsigned long long)n);
    }
    uint64_t d2h = 0;
    if (n) {
        if (int rc = grow_staging(e, &e->expire_stage, n, classify(o->records) != PTR_DEVICE, feats)) return rc;
        Blocks d;
        if (int rc = place_blocks(t, o, n, e->expire_stage, st, &d)) return rc;
        launched += fa::launch_gather(t, kmap, s.list, 1u, n, false, d.rec, d.slot_of, e->sm_count, st);
        if (int rc = finish_blocks(e, t, o, n, d, /*clear=*/true, st, &launched, &d2h)) return rc;
        launched += fa::launch_expire_delete(t, s, n, live == e->slots, e->d_ctr, e->sm_count, st);
        CU(cudaGetLastError());
        CU(cudaStreamSynchronize(st));
        set_live_known(e, live - n);
    }
    e->st.evictions++;
    e->st.flows_evicted += n;
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    *n_out = (size_t)n;
    return FA_OK;
}

// Device staging of host-bound rows (the group rows, the histogram rows): *buf grown to hold n rows of row_bytes, with
// room for twice that up to one row per flow-table slot.  On failure no buffer and no pending CUDA error are left, so
// the caller still clears the group table.
static int grow_group_out(uint8_t** buf, uint64_t* have_bytes, uint64_t n, uint64_t row_bytes, uint64_t slots, const char* who) {
    if (*have_bytes >= n * row_bytes) return FA_OK;
    cudaFree(*buf); *buf = nullptr; *have_bytes = 0;
    const uint64_t want = std::max<uint64_t>(n, std::min<uint64_t>(slots, 2 * n)) * row_bytes;
    if (cudaMalloc(buf, want) != cudaSuccess) {
        (void)cudaGetLastError();
        *buf = nullptr;
        return fail(FA_E_CUDA, "%s: no device memory for %llu B of staging", who, (unsigned long long)want);
    }
    *have_bytes = want;
    return FA_OK;
}

// A group table (all zero between calls), its list and counters for up to n groups, allocated on first use and grown
// with n, and its pinned host counter.  *grown: the table was (re)allocated.
static int grow_groups(fa::GroupScratch* g, fa::GroupCtr** h_ctr, uint64_t n, cudaStream_t st, bool* grown) {
    uint64_t slots = 1024;                             // load factor <= 3/4: groups never outnumber n
    while (slots < (4 * n + 2) / 3) slots <<= 1;
    *grown = !g->tab || g->mask + 1 < slots;
    if (*grown) {
        cudaFree(g->tab); cudaFree(g->list);
        g->tab = nullptr; g->list = nullptr; g->mask = 0;
        CU(cudaMalloc(&g->tab, slots * fa::kGroupSlotWords * 8));
        CU(cudaMalloc(&g->list, slots * 4));
        CU(cudaMemsetAsync(g->tab, 0, slots * fa::kGroupSlotWords * 8, st));
        g->mask = slots - 1;
    }
    if (!g->ctr) CU(cudaMalloc(&g->ctr, sizeof(fa::GroupCtr)));
    if (!*h_ctr) CU(cudaHostAlloc(h_ctr, sizeof(fa::GroupCtr), cudaHostAllocDefault));
    return FA_OK;
}

// The group table of fa_group_flows for `live` flows; with_row_of: also fa_histogram_flows' row index, one u32 per slot,
// grown with the table.
static int grow_group_table(fa_engine* e, uint64_t live, bool with_row_of) {
    bool grown = false;
    if (int rc = grow_groups(&e->group, &e->h_group_ctr, live, e->stream, &grown)) return rc;
    if (grown) { cudaFree(e->d_hist_row_of); e->d_hist_row_of = nullptr; }
    if (with_row_of && !e->d_hist_row_of) CU(cudaMalloc(&e->d_hist_row_of, (e->group.mask + 1) * 4));
    return FA_OK;
}

// The group scan fa_group_flows and fa_histogram_flows start with, on the engine stream after the queued folds: the
// masked key (byte 39, padding, is ignored), the group table for `live` flows, the scan, and the group count (the one
// wait).  A non-zero return ends the call at once.  Otherwise g->rc is FA_OK, FA_E_CUDA (more groups than live flows,
// or folds without a slot) or FA_E_2BIG (more groups than cap), and in every case the caller clears the g->n listed
// groups.
struct GroupScan { fa::GroupMask m; uint64_t n, launched; int rc; };
static int scan_groups(fa_engine* e, const char* who, const uint8_t key_mask[40], uint64_t live, size_t cap, bool with_row_of,
                       GroupScan* g) {
    memcpy(g->m.w, key_mask, fa::kKeyBytes);
    g->m.w[4] &= 0x00FFFFFFFFFFFFFFull;
    if (int rc = grow_group_table(e, live, with_row_of)) return rc;
    const fa::GroupScratch s = e->group;
    CU(cudaMemsetAsync(s.ctr, 0, sizeof(fa::GroupCtr), e->stream));
    g->launched = fa::launch_group_scan(e->table, g->m, s, e->sm_count, e->stream);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(e->h_group_ctr, s.ctr, sizeof(fa::GroupCtr), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    g->n = e->h_group_ctr->n;
    g->rc = FA_OK;
    if (e->h_group_ctr->lost || g->n > live)
        g->rc = fail(FA_E_CUDA, "%s: %llu groups of %llu live flows, %llu folds without a slot", who, (unsigned long long)g->n,
                     (unsigned long long)live, e->h_group_ctr->lost);
    else if (g->n > cap)
        g->rc = fail(FA_E_2BIG, "%s: capacity %zu < %llu groups", who, cap, (unsigned long long)g->n);
    return FA_OK;
}

// Exact roll-ups of the live flows by a key mask, read in place (evict.cu: launch_group_*): the group scan, then one
// pass writes the listed groups' rows (device `out` in place, host `out` through the group staging) and zeroes their
// slots, or only zeroes them when the rows are not wanted (FA_E_2BIG).  Either way the group table is all zero again for
// the next call.  Nothing of the flow table or the counters is written.
int fa_group_flows(fa_engine* e, const uint8_t key_mask[40], fa_flow_group* out, size_t cap, size_t* n_groups) {
    if (n_groups) *n_groups = 0;
    if (!e || !key_mask || !n_groups || (!out && cap)) return fail(FA_E_INVAL, "fa_group_flows: null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const bool out_dev = out && classify(out) == PTR_DEVICE;
    if (out_dev && (reinterpret_cast<uintptr_t>(out) & 7))
        return fail(FA_E_INVAL, "fa_group_flows: device out must be 8-byte aligned");
    if (int rc = sync_counters(e)) return rc;          // the queued folds finish; exact live count
    const uint64_t live = e->live_known;
    if (live == 0) return FA_OK;
    cudaStream_t st = e->stream;
    GroupScan g;
    if (int rc = scan_groups(e, "fa_group_flows", key_mask, live, cap, false, &g)) return rc;
    const fa::GroupScratch s = e->group;
    const uint64_t n = g.n;
    uint64_t launched = g.launched;
    int rc = g.rc;
    uint64_t* rows = nullptr;
    if (rc == FA_OK) {
        if (out_dev) rows = reinterpret_cast<uint64_t*>(out);
        else if ((rc = grow_group_out(&e->d_group_out, &e->group_out_bytes, n, fa::kGroupRowBytes, e->slots, "fa_group_flows")) == FA_OK)
            rows = reinterpret_cast<uint64_t*>(e->d_group_out);
    }
    launched += fa::launch_group_emit(s, std::min<uint64_t>(n, s.mask + 1), rows, e->sm_count, st);   // rows == nullptr: clear only
    CU(cudaGetLastError());
    uint64_t d2h = 0;
    if (rows && !out_dev) {
        CU(cudaMemcpyAsync(out, rows, n * fa::kGroupRowBytes, cudaMemcpyDeviceToHost, st));
        d2h = n * fa::kGroupRowBytes;
    }
    CU(cudaStreamSynchronize(st));
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    if (rc == FA_OK || rc == FA_E_2BIG) *n_groups = (size_t)n;
    return rc;
}

// Per-group histograms of one per-flow value (evict.cu: launch_hist_*), on the groups of fa_group_flows: the group scan
// builds the groups and their flow counts, then the rows are zeroed (device `out` in place, host `out` through the
// histogram staging), indexed by group, binned by a second scan of the live flows and completed from the group table,
// which is zeroed after (FA_E_2BIG: only zeroed).  Nothing of the flow table or the counters is written.
static_assert(FA_HIST_BYTES == fa::kHistBytes && FA_HIST_PACKETS == fa::kHistPackets && FA_HIST_DURATION == fa::kHistDuration &&
              FA_HIST_RTT == fa::kHistRtt && FA_HIST_DNS_LATENCY == fa::kHistDnsLatency, "FA_HIST_* values");
static_assert(FA_HIST_MAX_BOUNDS == fa::kHistMaxBounds && sizeof(fa_hist_row) == fa::kHistHeadWords * 8 &&
              FA_HIST_ROW_BYTES(0) == fa::kHistHeadWords * 8 + 8 && offsetof(fa_hist_row, max) == 72, "fa_hist_row ABI");

int fa_histogram_flows(fa_engine* e, const uint8_t key_mask[40], uint32_t value, const uint64_t* bounds, uint32_t n_bounds,
                       void* out, size_t cap, size_t* n_groups) {
    if (n_groups) *n_groups = 0;
    if (!e || !key_mask || !bounds || !n_groups || (!out && cap)) return fail(FA_E_INVAL, "fa_histogram_flows: null argument");
    if (value > FA_HIST_DNS_LATENCY) return fail(FA_E_INVAL, "fa_histogram_flows: unknown value %u", value);
    if (n_bounds == 0 || n_bounds > FA_HIST_MAX_BOUNDS)
        return fail(FA_E_INVAL, "fa_histogram_flows: n_bounds %u not in [1, %u]", n_bounds, FA_HIST_MAX_BOUNDS);
    for (uint32_t i = 1; i < n_bounds; i++)
        if (bounds[i] <= bounds[i - 1]) return fail(FA_E_INVAL, "fa_histogram_flows: bounds not strictly increasing at %u", i);
    if (value == FA_HIST_RTT && !(e->cfg.flags & FA_F_ENABLE_RTT))
        return fail(FA_E_INVAL, "fa_histogram_flows: FA_HIST_RTT needs an engine created with FA_F_ENABLE_RTT");
    if (value == FA_HIST_DNS_LATENCY && !(e->cfg.flags & FA_F_ENABLE_DNS))
        return fail(FA_E_INVAL, "fa_histogram_flows: FA_HIST_DNS_LATENCY needs an engine created with FA_F_ENABLE_DNS");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const bool out_dev = out && classify(out) == PTR_DEVICE;
    if (out_dev && (reinterpret_cast<uintptr_t>(out) & 7))
        return fail(FA_E_INVAL, "fa_histogram_flows: device out must be 8-byte aligned");
    if (int rc = sync_counters(e)) return rc;          // the queued folds finish; exact live count
    const uint64_t live = e->live_known;
    if (live == 0) return FA_OK;
    cudaStream_t st = e->stream;
    fa::HistParams h{};
    memcpy(h.bounds, bounds, n_bounds * sizeof(uint64_t));
    h.n_bounds = n_bounds;
    h.value = value;
    const uint64_t row_bytes = FA_HIST_ROW_BYTES(n_bounds);
    GroupScan g;
    if (int rc = scan_groups(e, "fa_histogram_flows", key_mask, live, cap, true, &g)) return rc;
    const fa::GroupScratch s = e->group;
    const uint64_t n = g.n;
    uint64_t launched = g.launched;
    int rc = g.rc;
    uint64_t* rows = nullptr;
    if (rc == FA_OK) {
        if (out_dev) rows = reinterpret_cast<uint64_t*>(out);
        else if ((rc = grow_group_out(&e->d_hist_out, &e->hist_out_bytes, n, row_bytes, e->slots, "fa_histogram_flows")) == FA_OK)
            rows = reinterpret_cast<uint64_t*>(e->d_hist_out);
    }
    if (rows) {
        CU(cudaMemsetAsync(rows, 0, n * row_bytes, st));
        launched += fa::launch_hist_index(s, n, e->d_hist_row_of, e->sm_count, st);
        launched += fa::launch_hist_scan(e->table, g.m, s, e->d_hist_row_of, h, rows, e->sm_count, st);
        launched += fa::launch_hist_emit(s, n, n_bounds, rows, e->sm_count, st);
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(e->h_group_ctr, s.ctr, sizeof(fa::GroupCtr), cudaMemcpyDeviceToHost, st));
    }
    launched += fa::launch_group_emit(s, std::min<uint64_t>(n, s.mask + 1), nullptr, e->sm_count, st);   // clear the groups
    CU(cudaGetLastError());
    uint64_t d2h = 0;
    if (rows && !out_dev) {
        CU(cudaMemcpyAsync(out, rows, n * row_bytes, cudaMemcpyDeviceToHost, st));
        d2h = n * row_bytes;
    }
    CU(cudaStreamSynchronize(st));
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    if (rows && e->h_group_ctr->lost)
        rc = fail(FA_E_CUDA, "fa_histogram_flows: %llu flows did not find their group", e->h_group_ctr->lost);
    if (rc == FA_OK || rc == FA_E_2BIG) *n_groups = (size_t)n;
    return rc;
}

// Per-group distinct counts of a second key mask (evict.cu: launch_distinct_*), in two levels of the group table.  Level
// 1 is the group scan with U = G | D (cap = live: never FA_E_2BIG): one group per distinct (key & G, key & D) pair,
// because key & U is that pair and (key & U) & G == key & G.  Level 2 folds the listed pairs by & G into the second group
// table (flows summed, pairs counted), then level 1 is cleared and its list, free again, receives the slots of the
// level-2 groups that pass min_distinct; their count is the second wait.  Then their rows are written (device `out` in
// place, host `out` through the distinct staging) and the second table is cleared, or only cleared (FA_E_2BIG, errors).
// Both group tables are all zero again for the next call.  Nothing of the flow table or the counters is written.
static_assert(sizeof(fa_distinct_group) == fa::kDistinctRowBytes && offsetof(fa_distinct_group, flows) == 40 &&
              offsetof(fa_distinct_group, distinct) == 48, "fa_distinct_group ABI");

int fa_distinct_flows(fa_engine* e, const uint8_t group_mask[40], const uint8_t distinct_mask[40], uint64_t min_distinct,
                      fa_distinct_group* out, size_t cap, size_t* n_groups) {
    if (n_groups) *n_groups = 0;
    if (!e || !group_mask || !distinct_mask || !n_groups || (!out && cap))
        return fail(FA_E_INVAL, "fa_distinct_flows: null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const bool out_dev = out && classify(out) == PTR_DEVICE;
    if (out_dev && (reinterpret_cast<uintptr_t>(out) & 7))
        return fail(FA_E_INVAL, "fa_distinct_flows: device out must be 8-byte aligned");
    if (int rc = sync_counters(e)) return rc;          // the queued folds finish; exact live count
    const uint64_t live = e->live_known;
    if (live == 0) return FA_OK;
    cudaStream_t st = e->stream;
    uint8_t u[fa::kKeyBytes];
    for (int i = 0; i < fa::kKeyBytes; i++) u[i] = group_mask[i] | distinct_mask[i];
    fa::GroupMask gm;
    memcpy(gm.w, group_mask, fa::kKeyBytes);
    gm.w[4] &= 0x00FFFFFFFFFFFFFFull;
    GroupScan g;
    if (int rc = scan_groups(e, "fa_distinct_flows", u, live, live, false, &g)) return rc;
    const fa::GroupScratch s1 = e->group;
    const uint64_t n1 = g.n;
    uint64_t launched = g.launched;
    int rc = g.rc;
    bool grown = false;
    if (rc == FA_OK && (rc = grow_groups(&e->distinct, &e->h_distinct_ctr, n1, st, &grown)) != FA_OK)
        (void)cudaGetLastError();                      // no pending error: level 1 is still cleared below
    const fa::GroupScratch s2 = e->distinct;
    const bool second = rc == FA_OK;
    if (second) {
        CU(cudaMemsetAsync(s2.ctr, 0, sizeof(fa::GroupCtr), st));
        launched += fa::launch_distinct_fold(s1, n1, gm, s2, e->sm_count, st);
    }
    launched += fa::launch_group_emit(s1, std::min<uint64_t>(n1, s1.mask + 1), nullptr, e->sm_count, st);   // clear level 1
    if (second) {
        CU(cudaMemsetAsync(s1.ctr, 0, sizeof(fa::GroupCtr), st));
        launched += fa::launch_distinct_select(s2, n1, min_distinct, s1.list, &s1.ctr->n, e->sm_count, st);
        CU(cudaMemcpyAsync(e->h_group_ctr, s1.ctr, sizeof(fa::GroupCtr), cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(e->h_distinct_ctr, s2.ctr, sizeof(fa::GroupCtr), cudaMemcpyDeviceToHost, st));
    }
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    uint64_t n2 = 0, n = 0;                            // level-2 groups, passing groups
    if (second) {
        n2 = e->h_distinct_ctr->n;
        n = e->h_group_ctr->n;
        if (e->h_distinct_ctr->lost || n2 > n1 || n > n2)
            rc = fail(FA_E_CUDA, "fa_distinct_flows: %llu groups of %llu pairs, %llu passing, %llu folds without a slot",
                      (unsigned long long)n2, (unsigned long long)n1, (unsigned long long)n, e->h_distinct_ctr->lost);
        else if (n > cap)
            rc = fail(FA_E_2BIG, "fa_distinct_flows: capacity %zu < %llu groups", cap, (unsigned long long)n);
    }
    uint64_t* rows = nullptr;
    if (rc == FA_OK && n) {
        if (out_dev) rows = reinterpret_cast<uint64_t*>(out);
        else if ((rc = grow_group_out(&e->d_distinct_out, &e->distinct_out_bytes, n, fa::kDistinctRowBytes, e->slots,
                                      "fa_distinct_flows")) == FA_OK)
            rows = reinterpret_cast<uint64_t*>(e->d_distinct_out);
    }
    if (rows) launched += fa::launch_distinct_emit(s2, s1.list, n, rows, e->sm_count, st);
    if (second) launched += fa::launch_group_emit(s2, std::min<uint64_t>(n2, s2.mask + 1), nullptr, e->sm_count, st);   // clear level 2
    CU(cudaGetLastError());
    uint64_t d2h = 0;
    if (rows && !out_dev) {
        CU(cudaMemcpyAsync(out, rows, n * fa::kDistinctRowBytes, cudaMemcpyDeviceToHost, st));
        d2h = n * fa::kDistinctRowBytes;
    }
    CU(cudaStreamSynchronize(st));
    e->st.kernel_launches += launched;
    e->st.d2h_bytes += d2h;
    if (rc == FA_OK || rc == FA_E_2BIG) *n_groups = (size_t)n;
    return rc;
}

// Emit and reset the flows touched since the last drain into out_records_dev.  The count goes to *n_dev_out (device
// memory, nothing waited for) when it is given, else to *n_out after a wait.
static int drain_active(fa_engine* e, void* out_records_dev, size_t cap, const char* who, size_t* n_out, uint64_t* n_dev_out) {
    if (e->table.feat_add || e->table.feat_dns || e->table.feat_drop) return fail(FA_E_INVAL, "%s: not available with feature folds enabled", who);
    if (e->cfg.mode != FA_MODE_ACCOUNTER) return fail(FA_E_INVAL, "%s: ACCOUNTER mode only", who);
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    CU(cudaMemsetAsync(&e->d_ctr->evict_out, 0, sizeof(unsigned long long), e->stream));
    e->st.kernel_launches += fa::launch_evict(e->table, static_cast<uint4*>(out_records_dev), nullptr, cap, e->d_ctr,
                                              e->sm_count, e->stream, /*drain=*/true);
    CU(cudaGetLastError());
    if (n_dev_out) {
        CU(cudaMemcpyAsync(n_dev_out, &e->d_ctr->evict_out, 8, cudaMemcpyDeviceToDevice, e->stream));
        return FA_OK;
    }
    if (int rc = sync_counters(e)) return rc;
    if (e->h_ctr->evict_out > cap)
        return fail(FA_E_2BIG, "%s: %llu active flows > capacity %zu (flows beyond it were reset but not written)", who,
                    (unsigned long long)e->h_ctr->evict_out, cap);
    *n_out = (size_t)e->h_ctr->evict_out;
    return FA_OK;
}

int fa_drain_active(fa_engine* e, void* out_records_dev, size_t cap, size_t* n_out) {
    if (n_out) *n_out = 0;
    if (!e || !n_out || !out_records_dev) return fail(FA_E_INVAL, "fa_drain_active: null argument");
    if (classify(out_records_dev) != PTR_DEVICE) return fail(FA_E_INVAL, "fa_drain_active: out_records must be device memory");
    return drain_active(e, out_records_dev, cap, "fa_drain_active", n_out, nullptr);
}

int fa_drain_active_counted(fa_engine* e, void* out_records_dev, size_t cap, uint64_t* n_dev_out) {
    if (!e || !out_records_dev || !n_dev_out) return fail(FA_E_INVAL, "fa_drain_active_counted: null argument");
    return drain_active(e, out_records_dev, cap, "fa_drain_active_counted", nullptr, n_dev_out);
}

int fa_route_peer(fa_engine* e, const void* recs, const uint64_t* n_dev, size_t max_n, uint32_t n_shards, uint32_t self_shard,
                  void* const* peer_bufs, uint64_t* const* peer_counts, size_t cap, uint64_t* overflow_dev) {
    if (!e || !recs || !peer_bufs || !peer_counts || !overflow_dev) return fail(FA_E_INVAL, "fa_route_peer: null argument");
    if (n_shards == 0 || n_shards > 16) return fail(FA_E_INVAL, "fa_route_peer: n_shards must be 1..16");
    if (max_n > 0xFFFFFFFFull) return fail(FA_E_INVAL, "fa_route_peer: max_n too large");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    fa::PeerTargets pt{};
    for (uint32_t i = 0; i < n_shards; i++) {
        pt.buf[i] = static_cast<uint4*>(peer_bufs[i]);
        pt.count[i] = reinterpret_cast<unsigned long long*>(peer_counts[i]);
    }
    e->st.kernel_launches += fa::launch_route_peer(static_cast<const uint4*>(recs), reinterpret_cast<const unsigned long long*>(n_dev),
                                                   (uint32_t)max_n, n_shards, self_shard, pt, cap, reinterpret_cast<unsigned long long*>(overflow_dev), e->sm_count, e->stream);
    CU(cudaGetLastError());
    return FA_OK;
}

int fa_ingest_counted(fa_engine* e, const void* recs, uint64_t* n_dev, size_t max_n, int reset_count) {
    if (!e || !recs || !n_dev) return fail(FA_E_INVAL, "fa_ingest_counted: null argument");
    if (!(e->cfg.flags & FA_F_NO_FULL_CUT)) return fail(FA_E_INVAL, "fa_ingest_counted: engine needs FA_F_NO_FULL_CUT");
    if (e->cfg.mode != FA_MODE_ACCOUNTER) return fail(FA_E_INVAL, "fa_ingest_counted: ACCOUNTER mode only");
    if (max_n == 0 || max_n > e->max_batch) return fail(FA_E_INVAL, "fa_ingest_counted: max_n must be 1..max_batch");
    if (reinterpret_cast<uintptr_t>(recs) & 15) return fail(FA_E_INVAL, "fa_ingest_counted: records must be 16-byte aligned");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    CU(cudaMemcpyAsync(&e->d_ctr->launch_n, n_dev, 8, cudaMemcpyDeviceToDevice, e->stream));
    const uint32_t saved = e->k1_opt;
    e->k1_opt |= 16u;
    int rc = launch_chunk(e, static_cast<const uint8_t*>(recs), (uint32_t)max_n);
    e->k1_opt = saved;
    if (rc) return rc;
    if (reset_count) CU(cudaMemsetAsync(n_dev, 0, 8, e->stream));
    return FA_OK;
}

static const char* sample_kind_name(uint32_t kind) { return kind == 0 ? "FA_F_ENABLE_RTT" : kind == 1 ? "FA_F_ENABLE_DNS" : "FA_F_ENABLE_PKT_DROP"; }
static uint32_t sample_kind_flag(uint32_t kind) { return kind == 0 ? FA_F_ENABLE_RTT : kind == 1 ? FA_F_ENABLE_DNS : FA_F_ENABLE_PKT_DROP; }

int fa_route_peer_samples(fa_engine* e, uint32_t kind, const void* samples_dev, const uint64_t* n_dev, size_t max_n, uint32_t n_shards,
                          uint32_t self_shard, void* const* peer_segs, uint64_t* const* peer_seg_counts, size_t seg_cap, uint64_t* overflow_dev) {
    if (!e || !samples_dev || !peer_segs || !peer_seg_counts || !overflow_dev) return fail(FA_E_INVAL, "fa_route_peer_samples: null argument");
    if (kind > FA_SAMPLES_PKT_DROPS) return fail(FA_E_INVAL, "fa_route_peer_samples: unknown sample kind %u", kind);
    if (n_shards == 0 || n_shards > 16 || self_shard >= n_shards) return fail(FA_E_INVAL, "fa_route_peer_samples: n_shards must be 1..16, self_shard below it");
    if (max_n > 0xFFFFFFFFull) return fail(FA_E_INVAL, "fa_route_peer_samples: max_n too large");
    if (reinterpret_cast<uintptr_t>(samples_dev) & 7) return fail(FA_E_INVAL, "fa_route_peer_samples: samples must be 8-byte aligned");
    for (uint32_t i = 0; i < n_shards; i++)
        if (!peer_segs[i] || !peer_seg_counts[i] || (reinterpret_cast<uintptr_t>(peer_segs[i]) & 7))
            return fail(FA_E_INVAL, "fa_route_peer_samples: segment %u missing or not 8-byte aligned", i);
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const uint64_t tiles = (max_n + 255) / 256;
    if (tiles > e->sroute_tiles) {                                   // scratch of the count pass, grown on demand
        CU(cudaFree(e->d_sroute_hist)); e->d_sroute_hist = nullptr; e->sroute_tiles = 0;
        CU(cudaMalloc(&e->d_sroute_hist, tiles * 16 * 4));
        e->sroute_tiles = tiles;
        if (!e->d_sroute_tot) CU(cudaMalloc(&e->d_sroute_tot, 16 * 8));
    }
    fa::PeerTargets pt{};
    for (uint32_t i = 0; i < n_shards; i++) {
        pt.buf[i] = static_cast<uint4*>(peer_segs[i]);
        pt.count[i] = reinterpret_cast<unsigned long long*>(peer_seg_counts[i]);
    }
    e->st.kernel_launches += fa::launch_route_samples((int)kind, static_cast<const uint8_t*>(samples_dev), reinterpret_cast<const unsigned long long*>(n_dev),
                                                      (uint32_t)max_n, n_shards, pt, seg_cap, e->d_sroute_hist, e->d_sroute_tot,
                                                      reinterpret_cast<unsigned long long*>(overflow_dev), e->sm_count, e->stream);
    CU(cudaGetLastError());
    return FA_OK;
}

int fa_ingest_samples_counted(fa_engine* e, uint32_t kind, const void* samples_dev, uint64_t* n_dev, size_t max_n, int reset_count) {
    if (!e || !samples_dev || !n_dev) return fail(FA_E_INVAL, "fa_ingest_samples_counted: null argument");
    if (kind > FA_SAMPLES_PKT_DROPS) return fail(FA_E_INVAL, "fa_ingest_samples_counted: unknown sample kind %u", kind);
    if (!(e->cfg.flags & sample_kind_flag(kind))) return fail(FA_E_INVAL, "fa_ingest_samples_counted: engine was created without %s", sample_kind_name(kind));
    if (!(e->cfg.flags & FA_F_NO_FULL_CUT)) return fail(FA_E_INVAL, "fa_ingest_samples_counted: engine needs FA_F_NO_FULL_CUT");
    if (e->cfg.mode != FA_MODE_ACCOUNTER) return fail(FA_E_INVAL, "fa_ingest_samples_counted: ACCOUNTER mode only");
    if (max_n == 0 || max_n > e->max_batch) return fail(FA_E_INVAL, "fa_ingest_samples_counted: max_n must be 1..max_batch");
    if (reinterpret_cast<uintptr_t>(samples_dev) & 7) return fail(FA_E_INVAL, "fa_ingest_samples_counted: samples must be 8-byte aligned");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    // sample numbers feat_seq .. feat_seq + max_n - 1 are reserved for this segment; the unused ones are a harmless gap
    e->st.kernel_launches += fa::launch_feature_fold_counted((int)kind, static_cast<const uint8_t*>(samples_dev), reinterpret_cast<const unsigned long long*>(n_dev),
                                                             (uint32_t)max_n, e->table, ++e->epoch, e->feat_seq[kind], e->d_slot_of,
                                                             e->d_ctr, e->sm_count, e->stream);
    CU(cudaGetLastError());
    e->feat_seq[kind] += max_n;
    e->unsynced_records += max_n;
    if (reset_count) CU(cudaMemsetAsync(n_dev, 0, 8, e->stream));
    return FA_OK;
}

int fa_ipc_export(fa_engine* e, void* dev_ptr, uint8_t handle_out[FA_IPC_HANDLE_BYTES]) {
    if (!e || !dev_ptr || !handle_out) return fail(FA_E_INVAL, "fa_ipc_export: null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == FA_IPC_HANDLE_BYTES, "IPC handle size");
    CU(cudaSetDevice(e->device));
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, dev_ptr));
    memcpy(handle_out, &h, sizeof h);
    return FA_OK;
}
int fa_ipc_open(fa_engine* e, const uint8_t handle[FA_IPC_HANDLE_BYTES], void** out) {
    if (!e || !handle || !out) return fail(FA_E_INVAL, "fa_ipc_open: null argument");
    CU(cudaSetDevice(e->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    CU(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
    return FA_OK;
}
int fa_ipc_close(fa_engine* e, void* mapped) {
    if (!e) return fail(FA_E_INVAL, "fa_ipc_close: null engine");
    CU(cudaSetDevice(e->device));
    CU(cudaIpcCloseMemHandle(mapped));
    return FA_OK;
}

// ---------------------------------------------------------------- K7: DNS query -> response correlation (dnscorr.cu)
static constexpr uint64_t kDnsMaxEntries = 1ull << 20;        // dns_flows max_entries (bpf/maps_definition.h:84); FA_DNS_MAX_ENTRIES overrides (tests)

static int dnsc_sync(fa_engine* e) {                          // device counters -> pinned mirror
    CU(cudaMemcpyAsync(e->h_dnsc_ctr, e->dnsc.ctr, fa::DNSC_N * 8, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    e->st.dns_queries_pending = e->h_dnsc_ctr[fa::DNSC_PRESENT];
    e->st.dns_map_full = e->h_dnsc_ctr[fa::DNSC_FULL];
    e->st.dns_queries_purged = e->h_dnsc_ctr[fa::DNSC_PURGED];
    return FA_OK;
}

static int dnsc_init(fa_engine* e) {
    if (e->dnsc.tab) return FA_OK;
    e->dnsc_chunk = std::min<uint64_t>(e->max_batch, 1ull << 20);
    uint64_t max_entries = kDnsMaxEntries;
    if (const char* me = getenv("FA_DNS_MAX_ENTRIES")) max_entries = std::max<uint64_t>(1, strtoull(me, nullptr, 0));
    uint64_t kDnsSlots = 64; while (kDnsSlots < 4 * max_entries) kDnsSlots <<= 1;
    e->dnsc_slots = kDnsSlots;
    fa::DnsEntry* tab = nullptr;
    CU(cudaMalloc(&tab, kDnsSlots * sizeof(fa::DnsEntry)));
    CU(cudaMemsetAsync(tab, 0, kDnsSlots * sizeof(fa::DnsEntry), e->stream));
    CU(cudaMalloc(&e->dnsc.ctr, fa::DNSC_N * 8));
    CU(cudaMemsetAsync(e->dnsc.ctr, 0, fa::DNSC_N * 8, e->stream));
    CU(cudaHostAlloc(&e->h_dnsc_ctr, fa::DNSC_N * 8, cudaHostAllocDefault));
    CU(cudaMalloc(&e->d_dnsc_state, e->dnsc_chunk * 4));
    CU(cudaMalloc(&e->d_dnsc_samples, e->dnsc_chunk * fa::kDnsRecBytes));
    CU(cudaMalloc(&e->d_dnsc_out, e->dnsc_chunk * fa::kDnsRecBytes));
    CU(cudaMalloc(&e->d_dnsc_warps, (e->dnsc_chunk + 31) / 32 * 4));
    e->dnsc.mask = kDnsSlots - 1; e->dnsc.max_entries = max_entries;
    e->dnsc.tab = tab;
    return FA_OK;
}

// move the pending queries into an empty table: the entries of answered queries are dropped
static int dnsc_rebuild(fa_engine* e) {
    if (!e->dnsc_spare) CU(cudaMalloc(&e->dnsc_spare, e->dnsc_slots * sizeof(fa::DnsEntry)));
    CU(cudaMemsetAsync(e->dnsc_spare, 0, e->dnsc_slots * sizeof(fa::DnsEntry), e->stream));
    CU(cudaMemsetAsync(&e->dnsc.ctr[fa::DNSC_CREATED], 0, 8, e->stream));
    fa::DnsCorr to = e->dnsc;
    to.tab = e->dnsc_spare;
    e->st.kernel_launches += fa::launch_dns_rebuild(e->dnsc, to, e->sm_count, e->stream);
    CU(cudaGetLastError());
    std::swap(e->dnsc.tab, e->dnsc_spare);
    if (int rc = dnsc_sync(e)) return rc;
    e->dnsc_used = e->h_dnsc_ctr[fa::DNSC_CREATED];
    return FA_OK;
}

int fa_ingest_dns_packets(fa_engine* e, const void* pkts, size_t n) {
    const char* who = "fa_ingest_dns_packets";
    if (!e) return fail(FA_E_INVAL, "%s: null engine", who);
    if (!(e->cfg.flags & FA_F_ENABLE_DNS)) return fail(FA_E_INVAL, "%s: engine was created without FA_F_ENABLE_DNS", who);
    if (n == 0) return FA_OK;
    if (!pkts) return fail(FA_E_INVAL, "%s: null packets", who);
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    if (int rc = dnsc_init(e)) return rc;
    // a chunk never takes more than a quarter of the table: with at most max_entries = slots / 4 present keys after a
    // rebuild the table stays at most half full.  That bounds the fill, not the length of a run: every packet takes an
    // entry, and keys can share a home slot, so one run can hold every entry in use.  The walk of dns_find_or_create is
    // therefore bounded by the table size, and always ends at the key or at an empty slot.
    const uint64_t cmax = std::min<uint64_t>(e->dnsc_chunk, e->dnsc_slots / 4);
    Input in(e, pkts, n, fa::kDnsRecBytes, cmax, std::min<uint64_t>(cmax, stage_records(e)), WINDOW_NONE);
    if (in.misaligned(8)) return fail(FA_E_INVAL, "%s: device packets must be 8-byte aligned", who);
    if (int rc = check_sample_room(e, n, who, "packets")) return rc;     // every packet may add a sample for a new flow
    while (in.more()) {
        if (e->dnsc_used + in.chunk() > e->dnsc_slots / 2) { if (int rc = dnsc_rebuild(e)) return rc; }
        const uint8_t* d = nullptr;
        uint64_t c = 0;
        if (int rc = in.next(&d, &c)) return rc;
        e->st.kernel_launches += fa::launch_dns_correlate(d, c, e->dnsc, e->d_dnsc_state, e->d_dnsc_samples, e->d_dnsc_warps, e->d_dnsc_out,
                                                          e->sm_count, e->stream);
        CU(cudaGetLastError());
        if (int rc = in.release()) return rc;
        if (int rc = dnsc_sync(e)) return rc;                 // how many samples the chunk produced (sizes the fold)
        e->dnsc_used += c;
        const uint32_t m = (uint32_t)e->h_dnsc_ctr[fa::DNSC_EMITTED];
        if (m) { if (int rc = fold_samples(e, 1, e->d_dnsc_out, m)) return rc; }
        e->st.dns_packets_ingested += c;
        in.advance(c);
    }
    return in.finish(FA_OK, nullptr);
}

int fa_purge_stale_dns(fa_engine* e, uint64_t mono_now_ns, uint64_t timeout_ns) {
    if (!e) return fail(FA_E_INVAL, "fa_purge_stale_dns: null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    if (!e->dnsc.tab) return FA_OK;   // no packet stream was correlated (pre-computed-latency contract, SURVEY.md §8 a12'): nothing to purge
    CU(cudaSetDevice(e->device));
    e->st.kernel_launches += fa::launch_dns_purge(e->dnsc, mono_now_ns, timeout_ns, e->sm_count, e->stream);
    CU(cudaGetLastError());
    return dnsc_sync(e);
}

int fa_cms_query(fa_engine* e, const void* keys, size_t n, uint64_t* est) {
    if (!e || (!keys && n) || (!est && n)) return fail(FA_E_INVAL, "fa_cms_query: null argument");
    if (!(e->cfg.flags & FA_F_ENABLE_SKETCH)) return fail(FA_E_INVAL, "fa_cms_query: engine was created without FA_F_ENABLE_SKETCH");
    if (n == 0) return FA_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    struct DevBuf { void* p = nullptr; ~DevBuf() { if (p) cudaFree(p); } } keys_buf, est_buf;   // freed on every return path
    CU(cudaMalloc(&keys_buf.p, n * 40 + 16));
    CU(cudaMalloc(&est_buf.p, n * 8));
    uint8_t* d_keys = static_cast<uint8_t*>(keys_buf.p);
    unsigned long long* d_est = static_cast<unsigned long long*>(est_buf.p);
    CU(cudaMemcpyAsync(d_keys, keys, n * 40, cudaMemcpyDefault, e->stream));
    e->st.kernel_launches += fa::launch_cms_query(e->sk, reinterpret_cast<const uint4*>(d_keys), (uint32_t)n, d_est, e->stream);
    CU(cudaMemcpyAsync(est, d_est, n * 8, cudaMemcpyDefault, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return FA_OK;
}

int fa_sketch_export(fa_engine* e, uint64_t* cms_out, size_t cms_words, uint8_t* hll_out, size_t hll_regs) {
    if (!e) return fail(FA_E_INVAL, "fa_sketch_export: null engine");
    if (!(e->cfg.flags & FA_F_ENABLE_SKETCH)) return fail(FA_E_INVAL, "fa_sketch_export: engine was created without FA_F_ENABLE_SKETCH");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    const size_t words = (size_t)e->sk.depth << e->sk.log2w, regs = (size_t)1 << e->sk.p;
    if (cms_out) {
        if (cms_words < words) return fail(FA_E_2BIG, "fa_sketch_export: cms buffer too small");
        CU(cudaMemcpyAsync(cms_out, e->sk.cms, words * 8, cudaMemcpyDeviceToHost, e->stream));
    }
    if (hll_out) {
        if (hll_regs < regs) return fail(FA_E_2BIG, "fa_sketch_export: hll buffer too small");
        uint8_t* d_regs = nullptr;
        CU(cudaMalloc(&d_regs, regs));
        e->st.kernel_launches += fa::launch_hll_pack(e->sk, d_regs, e->stream);
        CU(cudaMemcpyAsync(hll_out, d_regs, regs, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        cudaFree(d_regs);
    }
    CU(cudaStreamSynchronize(e->stream));
    return FA_OK;
}

int fa_sketch_reset(fa_engine* e) {
    if (!e) return fail(FA_E_INVAL, "fa_sketch_reset: null engine");
    if (!(e->cfg.flags & FA_F_ENABLE_SKETCH)) return FA_OK;
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    CU(cudaMemsetAsync(e->sk.cms, 0, ((size_t)e->sk.depth << e->sk.log2w) * 8, e->stream));
    CU(cudaMemsetAsync(e->sk.hll, 0, ((size_t)1 << e->sk.p) * 4, e->stream));
    return FA_OK;
}

int fa_hll_estimate(fa_engine* e, double* estimate) {
    if (!e || !estimate) return fail(FA_E_INVAL, "fa_hll_estimate: null argument");
    const size_t m = (size_t)1 << e->sk.p;
    std::vector<uint8_t> regs(m);
    int rc = fa_sketch_export(e, nullptr, 0, regs.data(), m);
    if (rc) return rc;
    double sum = 0.0; size_t zeros = 0;
    for (size_t i = 0; i < m; i++) { sum += std::ldexp(1.0, -(int)regs[i]); if (!regs[i]) zeros++; }
    const double alpha = m >= 128 ? 0.7213 / (1.0 + 1.079 / (double)m) : (m == 64 ? 0.709 : (m == 32 ? 0.697 : 0.673));
    double est = alpha * (double)m * (double)m / sum;
    if (est <= 2.5 * (double)m && zeros) est = (double)m * std::log((double)m / (double)zeros);
    *estimate = est;
    return FA_OK;
}

int fa_get_stats(fa_engine* e, fa_stats* out) {
    if (!e || !out) return fail(FA_E_INVAL, "fa_get_stats: null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    int rc = sync_counters(e);
    if (rc) return rc;
    e->st.live_flows = e->h_ctr->live;
    e->st.spills = e->h_ctr->spills;
    e->st.order_fixups = e->h_ctr->fixups_total;
    if (e->d_km_ctr) {
        CU(cudaMemcpyAsync(e->h_km_ctr, e->d_km_ctr, sizeof(fa::KmCounters), cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        e->st.observed_intf_missed = e->h_km_ctr->intf_missed;
        e->st.hashmap_fail_create = e->h_km_ctr->fail_create;
        e->st.ringbuf_dropped = e->h_km_ctr->spill_dropped;
        e->st.ringbuf_spilled = e->km_spilled_total + std::min<uint64_t>(e->h_km_ctr->spill_cursor, e->km_spill_cap);
        e->st.spills = e->h_km_ctr->table_full;
    }
    *out = e->st;
    return FA_OK;
}

int fa_read_spilled(fa_engine* e, void* out_records, size_t cap, size_t* n_out) {
    if (n_out) *n_out = 0;
    if (!e || !n_out) return fail(FA_E_INVAL, "fa_read_spilled: null argument");
    if (e->cfg.mode != FA_MODE_KERNEL_MAP || !(e->cfg.flags & FA_F_RINGBUF_FALLBACK))
        return fail(FA_E_INVAL, "fa_read_spilled: needs mode KERNEL_MAP with FA_F_RINGBUF_FALLBACK");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    CU(cudaMemcpyAsync(e->h_km_ctr, e->d_km_ctr, sizeof(fa::KmCounters), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    const uint64_t n = std::min<uint64_t>(e->h_km_ctr->spill_cursor, e->km_spill_cap);
    if (n == 0) return FA_OK;
    if (!out_records) return fail(FA_E_INVAL, "fa_read_spilled: null out_records");
    if (cap < n) return fail(FA_E_2BIG, "fa_read_spilled: capacity %zu < %llu spilled records", cap, (unsigned long long)n);
    CU(cudaMemcpyAsync(out_records, e->km_spill, n * fa::kRecBytes, cudaMemcpyDefault, e->stream));
    CU(cudaMemsetAsync(&e->d_km_ctr->spill_cursor, 0, sizeof(unsigned long long), e->stream));
    CU(cudaStreamSynchronize(e->stream));
    if (classify(out_records) != PTR_DEVICE) e->st.d2h_bytes += n * fa::kRecBytes;
    e->km_spilled_total += n;
    *n_out = (size_t)n;
    return FA_OK;
}

// ------------------------------------------------------------------ K8: protobuf batch encode
static_assert(sizeof(fa_iface_name) == sizeof(fa::PbIface) && offsetof(fa_iface_name, name) == offsetof(fa::PbIface, name) &&
              offsetof(fa_iface_name, udn) == offsetof(fa::PbIface, udn), "fa_iface_name layout");

int fa_pb_encode(fa_engine* e, const void* records, const void* dns, const void* additional, const void* pkt_drops,
                 const uint8_t* present, size_t n, const fa_pb_params* p, void* out_bytes, size_t out_cap, uint64_t* offsets,
                 void* keys_out, size_t* out_len) {
    if (out_len) *out_len = 0;
    if (!e || !p || !out_len) return fail(FA_E_INVAL, "fa_pb_encode: null argument");
    if (n == 0) return FA_OK;
    if (!records) return fail(FA_E_INVAL, "fa_pb_encode: null records");
    if (n > 0xFFFFFFFFull) return fail(FA_E_INVAL, "fa_pb_encode: n too large");
    if (p->n_ifaces && !p->ifaces) return fail(FA_E_INVAL, "fa_pb_encode: n_ifaces without ifaces");
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    struct DevBuf { void* p = nullptr; ~DevBuf() { if (p) cudaFree(p); } };
    // inputs: device pointers are used in place, host buffers are staged
    DevBuf in_bufs[5], out_buf, keys_buf;
    const void* src[5] = {records, dns, additional, present, pkt_drops};
    const size_t width[5] = {fa::kRecBytes, 64, 32, 1, 32};
    const uint8_t* d_in[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    for (int i = 0; i < 5; i++) {
        if (!src[i]) continue;
        if (classify(src[i]) == PTR_DEVICE) { d_in[i] = static_cast<const uint8_t*>(src[i]); continue; }
        CU(cudaMalloc(&in_bufs[i].p, n * width[i]));
        CU(cudaMemcpyAsync(in_bufs[i].p, src[i], n * width[i], cudaMemcpyHostToDevice, e->stream));
        e->st.h2d_bytes += n * width[i];
        d_in[i] = static_cast<const uint8_t*>(in_bufs[i].p);
    }
    if (e->pb_cap < n) {
        cudaFree(e->d_pb_sizes); cudaFree(e->d_pb_offsets); cudaFree(e->d_pb_sums);
        e->d_pb_sizes = nullptr; e->d_pb_offsets = nullptr; e->d_pb_sums = nullptr; e->pb_cap = 0;
        CU(cudaMalloc(&e->d_pb_sizes, n * 4));
        CU(cudaMalloc(&e->d_pb_offsets, (n + 1) * 8));
        CU(cudaMalloc(&e->d_pb_sums, ((n + 1023) / 1024 + 1) * 8));
        e->pb_cap = n;
    }
    if (p->n_ifaces > e->pb_ifaces_cap) {
        cudaFree(e->d_pb_ifaces); e->d_pb_ifaces = nullptr; e->pb_ifaces_cap = 0;
        CU(cudaMalloc(&e->d_pb_ifaces, (size_t)p->n_ifaces * sizeof(fa::PbIface)));
        e->pb_ifaces_cap = p->n_ifaces;
    }
    if (p->n_ifaces) CU(cudaMemcpyAsync(e->d_pb_ifaces, p->ifaces, (size_t)p->n_ifaces * sizeof(fa::PbIface), cudaMemcpyHostToDevice, e->stream));
    fa::PbParams P{};
    P.now_unix_ns = p->now_unix_ns; P.mono_now_ns = p->mono_now_ns;
    memcpy(P.agent_ip, p->agent_ip, 16);
    P.agent_is_v4 = p->agent_ip_is_v4 ? 1u : 0u;
    P.wrap = (p->flags & FA_PB_WRAP_ENTRIES) ? 1u : 0u;
    P.ifaces = e->d_pb_ifaces; P.n_ifaces = p->n_ifaces;
    fa::PbInputs in{d_in[0], d_in[1], d_in[2], d_in[4], d_in[3]};
    e->st.kernel_launches += fa::launch_pb_sizes(in, (uint32_t)n, P, e->d_pb_sizes, e->d_pb_offsets, e->d_pb_sums, e->sm_count, e->stream);
    CU(cudaGetLastError());
    unsigned long long total = 0;
    CU(cudaMemcpyAsync(&total, e->d_pb_offsets + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    *out_len = (size_t)total;
    if (total > out_cap) return fail(FA_E_2BIG, "fa_pb_encode: %llu bytes needed, capacity %zu", total, out_cap);
    if (!out_bytes && total) return fail(FA_E_INVAL, "fa_pb_encode: null out_bytes");   // total 0: every record dropped
    uint8_t* d_out = static_cast<uint8_t*>(out_bytes);
    const bool out_dev = classify(out_bytes) == PTR_DEVICE;
    if (!out_dev) { CU(cudaMalloc(&out_buf.p, total ? total : 16)); d_out = static_cast<uint8_t*>(out_buf.p); }
    uint8_t* d_keys = static_cast<uint8_t*>(keys_out);
    const bool keys_dev = keys_out && classify(keys_out) == PTR_DEVICE;
    if (keys_out && !keys_dev) { CU(cudaMalloc(&keys_buf.p, n * 32)); d_keys = static_cast<uint8_t*>(keys_buf.p); }
    e->st.kernel_launches += fa::launch_pb_write(in, (uint32_t)n, P, e->d_pb_offsets, e->d_pb_sizes, d_out, d_keys, e->stream);
    CU(cudaGetLastError());
    if (!out_dev && total) { CU(cudaMemcpyAsync(out_bytes, d_out, total, cudaMemcpyDeviceToHost, e->stream)); e->st.d2h_bytes += total; }
    if (keys_out && !keys_dev) { CU(cudaMemcpyAsync(keys_out, d_keys, n * 32, cudaMemcpyDeviceToHost, e->stream)); e->st.d2h_bytes += n * 32; }
    if (offsets) CU(cudaMemcpyAsync(offsets, e->d_pb_offsets, (n + 1) * 8, cudaMemcpyDefault, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return FA_OK;
}

int fa_sync(fa_engine* e) {
    if (!e) return fail(FA_E_INVAL, "fa_sync: null engine");
    CU(cudaSetDevice(e->device));
    CU(cudaStreamSynchronize(e->copy_stream));
    CU(cudaStreamSynchronize(e->stream));
    return FA_OK;
}

// ------------------------------------------------------------------ routing
uint64_t fa_owner_hash(const fa_flow_id* key) {
    uint64_t w[5];
    memcpy(w, key, 40);
    return fa::owner_hash(fa::key_premix(w[0], w[1], w[2], w[3], w[4]));
}

int fa_route(fa_engine* e, const void* recs, size_t n, uint32_t n_shards, void* out, uint64_t* counts_host) {
    if (!e || !counts_host || (n && (!recs || !out))) return fail(FA_E_INVAL, "fa_route: null argument");
    if (n_shards == 0 || n_shards > 16) return fail(FA_E_INVAL, "fa_route: n_shards must be 1..16");
    if (n > e->max_batch) return fail(FA_E_INVAL, "fa_route: n %zu > max_batch %llu", n, (unsigned long long)e->max_batch);
    std::lock_guard<std::mutex> lk(e->mu);
    CU(cudaSetDevice(e->device));
    if (!e->d_route_tmp) {
        const size_t ctas = (e->max_batch + 2047) / 2048;
        CU(cudaMalloc(&e->d_route_tmp, (e->max_batch + 16 * ctas + 16) * 4));
        CU(cudaMalloc(&e->d_route_counts, 16 * 8));
    }
    e->st.kernel_launches += fa::launch_route(reinterpret_cast<const uint4*>(recs), (uint32_t)n, n_shards,
                                              reinterpret_cast<uint4*>(out), e->d_route_counts, e->d_route_tmp, e->sm_count, e->stream);
    CU(cudaGetLastError());
    unsigned long long h[16];
    CU(cudaMemcpyAsync(h, e->d_route_counts, n_shards * 8, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    for (uint32_t i = 0; i < n_shards; i++) counts_host[i] = h[i];
    return FA_OK;
}

// ------------------------------------------------------------------ memory + generator
int fa_device_alloc(fa_engine* e, size_t bytes, void** out) {
    if (!e || !out) return fail(FA_E_INVAL, "fa_device_alloc: null argument");
    CU(cudaSetDevice(e->device));
    CU(cudaMalloc(out, bytes ? bytes : 16));
    CU(cudaMemset(*out, 0, bytes ? bytes : 16));       // zero-initialised (counters, receive buffers)
    return FA_OK;
}
int fa_device_free(fa_engine* e, void* p) {
    if (!e) return fail(FA_E_INVAL, "fa_device_free: null engine");
    CU(cudaSetDevice(e->device));
    CU(cudaFree(p));
    return FA_OK;
}
int fa_host_alloc(size_t bytes, void** out) {
    if (!out) return fail(FA_E_INVAL, "fa_host_alloc: null argument");
    CU(cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocDefault));
    return FA_OK;
}
int fa_host_free(void* p) { CU(cudaFreeHost(p)); return FA_OK; }

static int gen_params(const fa_gen_params* p, int device, fa::GenDeviceParams* g) {
    if (!p || p->n_keys == 0 || p->n_keys > (1ull << 32)) return fail(FA_E_INVAL, "fa_gen: n_keys must be 1..2^32");
    g->seed = p->seed; g->n_keys = p->n_keys; g->t0_ns = p->t0_ns; g->dist = p->dist; g->varying_desc = p->varying_desc;
    g->thresholds = nullptr; g->bucket_first = nullptr; g->bucket_size = nullptr; g->n_buckets = 0; g->reserved = 0;
    if (p->dist == FA_GEN_ZIPF) {
        ZipfTable* z = zipf_table(p->n_keys, p->zipf_s_milli ? p->zipf_s_milli : 1100);
        g->n_buckets = (uint32_t)z->thresholds.size();
        if (device < 0) {
            g->thresholds = z->thresholds.data(); g->bucket_first = z->first.data(); g->bucket_size = z->size.data();
        } else {
            std::lock_guard<std::mutex> lk(g_zipf_mu);
            if (z->device != device) {
                if (z->d_thresholds) { cudaFree(z->d_thresholds); cudaFree(z->d_first); cudaFree(z->d_size); }
                CU(cudaMalloc(&z->d_thresholds, z->thresholds.size() * 8));
                CU(cudaMalloc(&z->d_first, z->first.size() * 4));
                CU(cudaMalloc(&z->d_size, z->size.size() * 4));
                CU(cudaMemcpy(z->d_thresholds, z->thresholds.data(), z->thresholds.size() * 8, cudaMemcpyHostToDevice));
                CU(cudaMemcpy(z->d_first, z->first.data(), z->first.size() * 4, cudaMemcpyHostToDevice));
                CU(cudaMemcpy(z->d_size, z->size.data(), z->size.size() * 4, cudaMemcpyHostToDevice));
                z->device = device;
            }
            g->thresholds = z->d_thresholds; g->bucket_first = z->d_first; g->bucket_size = z->d_size;
        }
    }
    return FA_OK;
}

int fa_gen_records(fa_engine* e, const fa_gen_params* p, uint64_t first_index, size_t n, void* dst) {
    if (!dst && n) return fail(FA_E_INVAL, "fa_gen_records: null dst");
    const PtrKind k = e ? classify(dst) : PTR_PAGEABLE;
    fa::GenDeviceParams g;
    if (k == PTR_DEVICE) {
        CU(cudaSetDevice(e->device));
        int rc = gen_params(p, e->device, &g);
        if (rc) return rc;
        std::lock_guard<std::mutex> lk(e->mu);
        size_t done = 0;
        while (done < n) {
            const uint32_t c = (uint32_t)std::min<size_t>(n - done, 1u << 24);
            e->st.kernel_launches += fa::launch_generate(g, first_index + done, c, reinterpret_cast<uint4*>(static_cast<uint8_t*>(dst) + done * fa::kRecBytes), e->stream);
            done += c;
        }
        CU(cudaGetLastError());
        return FA_OK;
    }
    int rc = gen_params(p, -1, &g);
    if (rc) return rc;
    uint8_t* o = static_cast<uint8_t*>(dst);
    for (size_t i = 0; i < n; i++) {
        uint32_t w[36];
        fa::gen_record_words(g, first_index + i, w);
        memcpy(o + i * fa::kRecBytes, w, fa::kRecBytes);
    }
    return FA_OK;
}

int fa_gen_key(const fa_gen_params* p, uint64_t rank, fa_flow_id* out) {
    if (!p || !out) return fail(FA_E_INVAL, "fa_gen_key: null argument");
    uint32_t w[10];
    fa::gen_key_words(p->seed, rank, w);
    memcpy(out, w, 40);
    return FA_OK;
}

}  // extern "C"
