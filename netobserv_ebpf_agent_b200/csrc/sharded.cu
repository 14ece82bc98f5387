// sharded.cu — fa_sharded_*: one process drives N GPUs of one box behind the C ABI (include/flowagg.h).
//
// Flows are independent, so the path shards: owner = fa_owner_hash(flow_id) % N.  Every GPU is at once a SOURCE (it
// receives a slice of each host batch over its own PCIe link) and an OWNER (it keeps the flows that hash to it).
// Per round and source GPU, all enqueued on that GPU's stream, nothing waits on the host:
//   H2D copy of the slice -> local combine (K1 into a scratch table, K2 in lookup-and-reset mode: partial flow
//   records of the flows the slice touched; the reference folds its per-CPU maps the same way,
//   pkg/tracer/tracer.go:1159-1187) -> K3 fused with the exchange (fa_route_peer: the partials are partitioned by
//   owner and stored straight into the owners' receive buffers over NVLink; peer access, no NCCL, no IPC)
// then every owner waits for the N route events (cudaStreamWaitEvent: the only synchronisation, device side) and
// folds what it received (fa_ingest_counted: the record count is read from its own memory).  Receive buffers are
// double-buffered; a source only re-uses a buffer after the owners' fold events of two rounds ago.
// No collective at eviction: the owners' key sets are disjoint and are simply concatenated.
//
// Feature samples (RTT / IPsec, DNS, packet drops) take the same rounds, buffers and events, without the combiner: K6's
// folds depend on the order of a flow's samples, so the route is the stable one (fa_route_peer_samples: source i stores
// into segment i of every owner's buffer, in slice order) and every owner folds segment 0, 1, .., N-1 in that order
// (fa_ingest_samples_counted, one launch pair per segment, the count read from its own memory).  A flow's samples then
// reach its owner's fold in stream order whatever GPUs they crossed: the result is bit-identical to one engine.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "../../include/flowagg.h"

namespace {
constexpr size_t kRec = 144;
constexpr size_t kSample = 72, kDnsSample = 104;     // additional / packet-drop samples, DNS samples
const uint32_t kFeatFlag[3] = {FA_F_ENABLE_RTT, FA_F_ENABLE_DNS, FA_F_ENABLE_PKT_DROP};
const char* const kFeatFlagName[3] = {"FA_F_ENABLE_RTT", "FA_F_ENABLE_DNS", "FA_F_ENABLE_PKT_DROP"};
int sfail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
std::string& serr() { static thread_local std::string s; return s; }
int sfail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    serr() = buf;
    return code;
}
#define SCU(call)                                                                                              \
    do {                                                                                                       \
        cudaError_t e_ = (call);                                                                               \
        if (e_ != cudaSuccess) return sfail(FA_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)
#define SFA(call)                                                                                              \
    do {                                                                                                       \
        int rc_ = (call);                                                                                      \
        if (rc_ < 0) return sfail(rc_, "%s: %s", #call, fa_last_error());                                      \
    } while (0)
}  // namespace

struct fa_sharded {
    uint32_t n = 0;
    uint64_t round_cap = 0;                       // records per source GPU and round
    uint64_t recv_cap = 0;                        // records a receive buffer holds
    bool combine = true;
    std::mutex mu;
    struct Gpu {
        int device = 0;
        cudaStream_t stream = nullptr;
        fa_engine* owner = nullptr;               // the flows that hash to this GPU
        fa_engine* local = nullptr;               // scratch table of the per-round combiner
        uint8_t* d_in = nullptr;                  // staged slice of the host batch
        uint8_t* h_pin = nullptr;                 // pinned bounce buffer for pageable input
        uint8_t* d_part = nullptr; uint64_t* d_part_n = nullptr;      // partial flow records of a round + their count
        uint8_t* recv[2] = {nullptr, nullptr}; uint64_t* recv_n[2] = {nullptr, nullptr};   // what the peers deliver
        uint64_t* seg_n[2] = {nullptr, nullptr};  // sample rounds: the samples of segment i (source i) of recv[b] in seg_n[b][i]
        uint64_t* d_over = nullptr;               // [0] records that did not fit a receive buffer, [1] records sent to other GPUs
        cudaEvent_t ev_routed[2] = {nullptr, nullptr}, ev_folded[2] = {nullptr, nullptr}, ev_in_free = nullptr;
    };
    std::vector<Gpu> g;
    uint64_t rounds = 0, records = 0;
    uint64_t samples[3] = {0, 0, 0};              // additional, DNS, packet-drop samples passed in
    uint32_t feat_flags = 0;                      // FA_F_ENABLE_RTT / _DNS / _PKT_DROP of the owners
};

extern "C" {

const char* fa_sharded_last_error(void) { return serr().empty() ? fa_last_error() : serr().c_str(); }

void fa_sharded_destroy(fa_sharded* s) {
    if (!s) return;
    for (auto& G : s->g) {
        cudaSetDevice(G.device);
        if (G.stream) cudaStreamSynchronize(G.stream);
    }
    for (auto& G : s->g) {
        cudaSetDevice(G.device);
        if (G.owner) fa_destroy(G.owner);
        if (G.local) fa_destroy(G.local);
        cudaFree(G.d_in); cudaFree(G.d_part); cudaFree(G.d_part_n); cudaFree(G.d_over);
        for (int b = 0; b < 2; b++) {
            cudaFree(G.recv[b]); cudaFree(G.recv_n[b]); cudaFree(G.seg_n[b]);
            if (G.ev_routed[b]) cudaEventDestroy(G.ev_routed[b]);
            if (G.ev_folded[b]) cudaEventDestroy(G.ev_folded[b]);
        }
        if (G.ev_in_free) cudaEventDestroy(G.ev_in_free);
        if (G.h_pin) cudaFreeHost(G.h_pin);
        if (G.stream) cudaStreamDestroy(G.stream);
    }
    delete s;
}

int fa_sharded_create(const fa_config* cfg, const int32_t* devices, uint32_t n_devices, fa_sharded** out) {
    if (!cfg || !devices || !out || n_devices == 0 || n_devices > 16) return sfail(FA_E_INVAL, "fa_sharded_create: bad argument (1..16 devices)");
    if (cfg->mode != FA_MODE_ACCOUNTER) return sfail(FA_E_INVAL, "fa_sharded_create: ACCOUNTER mode only");
    if (cfg->flags & FA_F_ENABLE_SKETCH)
        return sfail(FA_E_INVAL, "fa_sharded_create: FA_F_ENABLE_SKETCH is per-engine (sketches of sharded flows are not merged)");
    fa_sharded* s = new (std::nothrow) fa_sharded();
    if (!s) return sfail(FA_E_NOMEM, "fa_sharded_create: out of memory");
    struct Guard { fa_sharded* s; ~Guard() { if (s) fa_sharded_destroy(s); } } guard{s};
    s->n = n_devices;
    s->round_cap = cfg->max_batch ? cfg->max_batch : (1ull << 22);
    s->combine = (cfg->reserved0 & 1u) == 0;              // reserved0 bit 0: route raw records, no local combiner
    s->recv_cap = s->round_cap * n_devices;               // worst case: every source's whole round lands on one owner
    s->feat_flags = cfg->flags & (FA_F_ENABLE_RTT | FA_F_ENABLE_DNS | FA_F_ENABLE_PKT_DROP);
    s->g.resize(n_devices);
    for (uint32_t i = 0; i < n_devices; i++) {
        auto& G = s->g[i];
        G.device = devices[i];
        SCU(cudaSetDevice(G.device));
        for (uint32_t j = 0; j < n_devices; j++) {
            if (devices[j] == G.device) continue;
            int can = 0;
            SCU(cudaDeviceCanAccessPeer(&can, G.device, devices[j]));
            if (!can) return sfail(FA_E_NODEV, "fa_sharded_create: device %d cannot access device %d (NVLink / P2P needed)", G.device, devices[j]);
            cudaError_t pe = cudaDeviceEnablePeerAccess(devices[j], 0);
            if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) return sfail(FA_E_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(pe));
            cudaGetLastError();
        }
        SCU(cudaStreamCreateWithFlags(&G.stream, cudaStreamNonBlocking));
        fa_config oc = *cfg;
        oc.device = G.device; oc.flags = FA_F_NO_FULL_CUT | s->feat_flags; oc.cuda_stream = G.stream; oc.reserved0 = 0;
        oc.max_batch = s->recv_cap;                       // an owner folds a whole receive buffer in one launch
        oc.max_entries = std::max<uint64_t>(1024, (cfg->max_entries + n_devices - 1) / n_devices * 5 / 4);   // owners hold ~1/N of the flows
        SFA(fa_create(&oc, &G.owner));
        if (s->combine) {
            fa_config lc = oc;
            lc.flags = FA_F_NO_FULL_CUT;                  // samples bypass the combiner
            lc.max_batch = s->round_cap;
            lc.max_entries = std::max<uint64_t>(2 * s->round_cap, std::min<uint64_t>(cfg->max_entries, 1ull << 26));
            SFA(fa_create(&lc, &G.local));
        }
        SCU(cudaMalloc(&G.d_in, s->round_cap * kRec));
        SCU(cudaMalloc(&G.d_part, s->round_cap * kRec));
        SCU(cudaMalloc(&G.d_part_n, 8));
        SCU(cudaMalloc(&G.d_over, 16));
        SCU(cudaMemset(G.d_over, 0, 16));
        for (int b = 0; b < 2; b++) {
            SCU(cudaMalloc(&G.recv[b], s->recv_cap * kRec));
            SCU(cudaMalloc(&G.recv_n[b], 8));
            SCU(cudaMemset(G.recv_n[b], 0, 8));
            if (s->feat_flags) {                          // N segments of round_cap samples (<= 104 B) fit the 144-byte rows
                SCU(cudaMalloc(&G.seg_n[b], 8 * n_devices));
                SCU(cudaMemset(G.seg_n[b], 0, 8 * n_devices));
            }
            SCU(cudaEventCreateWithFlags(&G.ev_routed[b], cudaEventDisableTiming));
            SCU(cudaEventCreateWithFlags(&G.ev_folded[b], cudaEventDisableTiming));
            SCU(cudaEventRecord(G.ev_folded[b], G.stream));
        }
        SCU(cudaEventCreateWithFlags(&G.ev_in_free, cudaEventDisableTiming));
        SCU(cudaEventRecord(G.ev_in_free, G.stream));
    }
    guard.s = nullptr;
    *out = s;
    return FA_OK;
}

// One round: source i holds cnt[i] items in its d_in (already enqueued on its stream): 144-byte flow records
// (kind < 0) or feature samples of `kind` (0 additional, 1 DNS, 2 packet drops).
static int sharded_round(fa_sharded* s, const size_t* cnt, int kind) {
    const int b = (int)(s->rounds & 1);
    const uint32_t N = s->n;
    const size_t seg_bytes = s->round_cap * (kind == 1 ? kDnsSample : kSample);   // sample rounds: segment i of recv[b] is source i's
    void* bufs[16]; uint64_t* cnts[16];
    for (uint32_t j = 0; j < N; j++) { bufs[j] = s->g[j].recv[b]; cnts[j] = s->g[j].recv_n[b]; }
    for (uint32_t i = 0; i < N; i++) {
        auto& G = s->g[i];
        SCU(cudaSetDevice(G.device));
        // the owners folded what round-2 delivered into these buffers
        for (uint32_t j = 0; j < N; j++) SCU(cudaStreamWaitEvent(G.stream, s->g[j].ev_folded[b], 0));
        if (cnt[i] && kind >= 0) {
            void* segs[16]; uint64_t* seg_n[16];
            for (uint32_t j = 0; j < N; j++) { segs[j] = s->g[j].recv[b] + i * seg_bytes; seg_n[j] = s->g[j].seg_n[b] + i; }
            SFA(fa_route_peer_samples(G.owner, (uint32_t)kind, G.d_in, nullptr, cnt[i], N, i, segs, seg_n, s->round_cap, G.d_over));
        } else if (cnt[i]) {
            const void* src = G.d_in; const uint64_t* src_n = nullptr; size_t max_n = cnt[i];
            if (s->combine) {
                size_t took = 0;
                SFA(fa_ingest(G.local, G.d_in, cnt[i], &took));
                SFA(fa_drain_active_counted(G.local, G.d_part, s->round_cap, G.d_part_n));
                src = G.d_part; src_n = G.d_part_n; max_n = std::min<size_t>(s->round_cap, cnt[i]);
            }
            SFA(fa_route_peer(G.owner, src, src_n, max_n, N, i, bufs, cnts, s->recv_cap, G.d_over));
        }
        SCU(cudaEventRecord(G.ev_routed[b], G.stream));
        SCU(cudaEventRecord(G.ev_in_free, G.stream));
    }
    for (uint32_t j = 0; j < N; j++) {
        auto& G = s->g[j];
        SCU(cudaSetDevice(G.device));
        for (uint32_t i = 0; i < N; i++) SCU(cudaStreamWaitEvent(G.stream, s->g[i].ev_routed[b], 0));
        if (kind < 0) SFA(fa_ingest_counted(G.owner, G.recv[b], G.recv_n[b], s->recv_cap, 1));
        else {
            // segments in source order = the samples in stream order; a source without samples left its count at 0
            for (uint32_t i = 0; i < N; i++)
                if (cnt[i]) SFA(fa_ingest_samples_counted(G.owner, (uint32_t)kind, G.recv[b] + i * seg_bytes, G.seg_n[b] + i, cnt[i], 1));
        }
        SCU(cudaEventRecord(G.ev_folded[b], G.stream));
    }
    s->rounds++;
    return FA_OK;
}

// Host items (records, kind < 0, or samples of `kind`) in rounds of N x round_cap, dealt to the sources by position.
static int sharded_ingest_host(fa_sharded* s, int kind, const void* items, size_t n, const char* who) {
    if (!s) return sfail(FA_E_INVAL, "%s: null engine", who);
    if (kind >= 0 && !(s->feat_flags & kFeatFlag[kind])) return sfail(FA_E_INVAL, "%s: engine was created without %s", who, kFeatFlagName[kind]);
    if (n == 0) return FA_OK;
    if (!items) return sfail(FA_E_INVAL, "%s: null %s", who, kind < 0 ? "records" : "samples");
    const size_t rb = kind < 0 ? kRec : kind == 1 ? kDnsSample : kSample;
    std::lock_guard<std::mutex> lk(s->mu);
    cudaPointerAttributes a;
    bool pinned = false;
    if (cudaPointerGetAttributes(&a, items) == cudaSuccess) {
        if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)
            return sfail(FA_E_INVAL, "%s: host %s expected%s", who, kind < 0 ? "records" : "samples", kind < 0 ? " (device batches: fa_sharded_ingest_device)" : "");
        pinned = a.type == cudaMemoryTypeHost;
    } else cudaGetLastError();
    const uint8_t* src = static_cast<const uint8_t*>(items);
    const uint32_t N = s->n;
    size_t done = 0;
    while (done < n) {
        // the next N x round_cap items, dealt to the sources by position
        const size_t chunk = std::min<size_t>(n - done, (size_t)N * s->round_cap);
        size_t cnt[16];
        for (uint32_t i = 0; i < N; i++) {
            const size_t lo = chunk * i / N, hi = chunk * (i + 1) / N;
            cnt[i] = hi - lo;
            auto& G = s->g[i];
            if (!cnt[i]) continue;
            SCU(cudaSetDevice(G.device));
            const uint8_t* p = src + (done + lo) * rb;
            if (!pinned) {
                if (!G.h_pin) SCU(cudaHostAlloc(&G.h_pin, s->round_cap * kRec, cudaHostAllocDefault));
                SCU(cudaEventSynchronize(G.ev_in_free));                  // the bounce buffer's previous copy has been consumed
                memcpy(G.h_pin, p, cnt[i] * rb);
                p = G.h_pin;
            }
            SCU(cudaMemcpyAsync(G.d_in, p, cnt[i] * rb, cudaMemcpyHostToDevice, G.stream));
        }
        int rc = sharded_round(s, cnt, kind);
        if (rc) return rc;
        done += chunk;
    }
    // the caller's buffer must not be referenced after return
    for (auto& G : s->g) { SCU(cudaSetDevice(G.device)); SCU(cudaEventSynchronize(G.ev_in_free)); }
    (kind < 0 ? s->records : s->samples[kind]) += n;
    return FA_OK;
}

int fa_sharded_ingest(fa_sharded* s, const void* flow_records, size_t n) { return sharded_ingest_host(s, -1, flow_records, n, "fa_sharded_ingest"); }
int fa_sharded_ingest_additional(fa_sharded* s, const void* samples, size_t n) { return sharded_ingest_host(s, 0, samples, n, "fa_sharded_ingest_additional"); }
int fa_sharded_ingest_dns(fa_sharded* s, const void* samples, size_t n) { return sharded_ingest_host(s, 1, samples, n, "fa_sharded_ingest_dns"); }
int fa_sharded_ingest_pkt_drops(fa_sharded* s, const void* samples, size_t n) { return sharded_ingest_host(s, 2, samples, n, "fa_sharded_ingest_pkt_drops"); }

int fa_sharded_ingest_device(fa_sharded* s, const void* const* records_dev, const size_t* n_per_gpu) {
    if (!s || !records_dev || !n_per_gpu) return sfail(FA_E_INVAL, "fa_sharded_ingest_device: null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    const uint32_t N = s->n;
    size_t off[16] = {0};
    for (;;) {
        size_t cnt[16]; bool any = false;
        for (uint32_t i = 0; i < N; i++) {
            cnt[i] = std::min<size_t>(n_per_gpu[i] - off[i], s->round_cap);
            if (!cnt[i]) continue;
            any = true;
            auto& G = s->g[i];
            SCU(cudaSetDevice(G.device));
            SCU(cudaMemcpyAsync(G.d_in, static_cast<const uint8_t*>(records_dev[i]) + off[i] * kRec, cnt[i] * kRec, cudaMemcpyDeviceToDevice, G.stream));
            off[i] += cnt[i];
            s->records += cnt[i];
        }
        if (!any) break;
        int rc = sharded_round(s, cnt, -1);
        if (rc) return rc;
    }
    return FA_OK;
}

int fa_sharded_sync(fa_sharded* s) {
    if (!s) return sfail(FA_E_INVAL, "fa_sharded_sync: null engine");
    for (auto& G : s->g) { SCU(cudaSetDevice(G.device)); SCU(cudaStreamSynchronize(G.stream)); }
    return FA_OK;
}

int fa_sharded_live_flows(fa_sharded* s, size_t* n) {
    if (!s || !n) return sfail(FA_E_INVAL, "fa_sharded_live_flows: null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    size_t tot = 0;
    for (auto& G : s->g) { size_t k = 0; SFA(fa_live_flows(G.owner, &k)); tot += k; }
    *n = tot;
    return FA_OK;
}

// fa_evict_ex over every owner: disjoint key sets, so the rows are concatenated, every block offset by the rows before
static int sharded_evict(fa_sharded* s, const fa_evict_out* out, size_t cap, size_t* n_out, const char* who) {
    if (n_out) *n_out = 0;
    if (!s || !out || !n_out) return sfail(FA_E_INVAL, "%s: null argument", who);
    std::lock_guard<std::mutex> lk(s->mu);
    size_t live[16], tot = 0;
    for (uint32_t j = 0; j < s->n; j++) { SFA(fa_live_flows(s->g[j].owner, &live[j])); tot += live[j]; }
    if (tot > cap) return sfail(FA_E_2BIG, "%s: capacity %zu < %zu live flows", who, cap, tot);
    if (tot && !out->records) return sfail(FA_E_INVAL, "%s: null out_records", who);
    size_t off = 0;
    for (uint32_t j = 0; j < s->n; j++) {
        auto at = [off](void* p, size_t bytes) { return p ? static_cast<void*>(static_cast<uint8_t*>(p) + off * bytes) : nullptr; };
        fa_evict_out o{};
        o.records = at(out->records, kRec); o.dns = at(out->dns, 64); o.additional = at(out->additional, 32);
        o.pkt_drops = at(out->pkt_drops, 32); o.rtt_min = static_cast<uint64_t*>(at(out->rtt_min, 8));
        o.present = static_cast<uint8_t*>(at(out->present, 1));
        size_t got = 0;
        SFA(fa_evict_ex(s->g[j].owner, &o, cap - off, &got));
        off += got;
    }
    // the combiners' scratch tables only cache keys (their accumulators were drained): empty them with the flows
    for (auto& G : s->g) {
        if (!G.local) continue;
        size_t k = 0;
        SFA(fa_live_flows(G.local, &k));
        for (size_t done = 0; done < k;) {
            // lookup-and-delete into the (idle) staging buffer, discarded
            size_t got = 0;
            if (k <= s->round_cap) { SFA(fa_evict(G.local, G.d_part, nullptr, nullptr, nullptr, s->round_cap, &got)); done = k; }
            else {
                SCU(cudaSetDevice(G.device));
                void* tmp = nullptr;
                SCU(cudaMalloc(&tmp, k * kRec));
                int rc = fa_evict(G.local, tmp, nullptr, nullptr, nullptr, k, &got);
                cudaFree(tmp);
                if (rc < 0) return sfail(rc, "fa_evict(local): %s", fa_last_error());
                done = k;
            }
        }
    }
    *n_out = off;
    return FA_OK;
}

int fa_sharded_evict(fa_sharded* s, void* out_records, size_t cap, size_t* n_out) {
    fa_evict_out o{};
    o.records = out_records;
    return sharded_evict(s, &o, cap, n_out, "fa_sharded_evict");
}

int fa_sharded_evict_ex(fa_sharded* s, const fa_evict_out* out, size_t cap, size_t* n_out) { return sharded_evict(s, out, cap, n_out, "fa_sharded_evict_ex"); }

int fa_sharded_get_stats(fa_sharded* s, fa_stats* sum, uint64_t* nvlink_records, uint64_t* receive_overflow) {
    if (!s || !sum) return sfail(FA_E_INVAL, "fa_sharded_get_stats: null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    memset(sum, 0, sizeof *sum);
    uint64_t nv = 0, ov = 0;
    for (auto& G : s->g) {
        fa_stats st;
        SFA(fa_get_stats(G.owner, &st));
        uint64_t* a = reinterpret_cast<uint64_t*>(sum); const uint64_t* b = reinterpret_cast<const uint64_t*>(&st);
        for (size_t k = 0; k < sizeof(fa_stats) / 8; k++) a[k] += b[k];
        if (G.local) { SFA(fa_get_stats(G.local, &st)); sum->kernel_launches += st.kernel_launches; sum->h2d_bytes += st.h2d_bytes; sum->spills += st.spills; }
        uint64_t h[2];
        SCU(cudaSetDevice(G.device));
        SCU(cudaMemcpy(h, G.d_over, 16, cudaMemcpyDeviceToHost));
        ov += h[0]; nv += h[1];
    }
    sum->records_ingested = s->records;
    sum->additional_ingested = s->samples[0]; sum->dns_ingested = s->samples[1]; sum->pkt_drops_ingested = s->samples[2];
    if (nvlink_records) *nvlink_records = nv;
    if (receive_overflow) *receive_overflow = ov;
    return FA_OK;
}

}  // extern "C"
