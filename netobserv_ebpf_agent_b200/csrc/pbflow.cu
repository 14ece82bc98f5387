// pbflow.cu — K8: evicted flows -> pbflow.Record wire bytes (protobuf), with the NewRecord decoration and the Kafka key.
//
// Replaces, for a whole eviction at once, the per-record host work that follows LookupAndDeleteMap / Accounter.evict:
//   model.NewRecord            (pkg/model/record.go:82-159): wall-clock start / end, interface list, DNS latency, RTT
//   pbflow.FlowToPB            (pkg/pbflow/proto.go:39-149) + proto.Marshal of the generated message (proto/flow.proto:31-126)
//   getFlowKey                 (pkg/exporter/kafka_proto.go:37-47): the two addresses, smaller one first
// Three kernels: size (one thread per flow, the same encoder run against a counting sink) -> exclusive scan ->
// write (one CTA per 256 flows: every thread encodes into a shared-memory image of the CTA's contiguous output range,
// which then leaves with coalesced 16-byte stores; a CTA whose range does not fit writes straight to global memory).
// Fields are written in field-number order, zero scalars are omitted, sub-messages the reference always allocates
// (timestamps, data_link, network, transport, agent_ip, time_flow_rtt) are always present — what protobuf-go emits.
// A record whose dns_name, interface name or UDN is not valid UTF-8 is emitted as zero bytes: protobuf-go refuses to
// marshal such a `string` field and the Kafka exporter drops the record (pkg/exporter/kafka_proto.go:53-57).  The size
// pass decides (its size is 0, and a real record is never empty); the write pass reads that size back.
// Not produced here (the engine has no such state): xlat, quic, network_events_metadata, `interface`, `duplicate`.
#include "kernels.cuh"

namespace fa {

static_assert(sizeof(PbIface) == 92, "fa_iface_name layout");

// CountSink also checks the string fields (ok); ByteSink only runs on records the CountSink found valid
struct CountSink { static constexpr bool kCounts = true;  uint32_t n = 0; bool ok = true; __device__ __forceinline__ void put(uint8_t) { n++; } };
struct ByteSink  { static constexpr bool kCounts = false; uint8_t* p;                      __device__ __forceinline__ void put(uint8_t b) { *p++ = b; } };

// utf8.ValidString: well-formed UTF-8 (Unicode Table 3-7) — no overlong form, surrogate, code point past U+10FFFF,
// stray continuation byte or truncated sequence
__device__ __forceinline__ bool utf8_valid(const uint8_t* s, uint32_t len) {
    uint32_t i = 0;
    while (i < len) {
        const uint32_t c = s[i];
        if (c < 0x80u) { i++; continue; }
        uint32_t more, lo = 0x80u, hi = 0xBFu;                          // continuation bytes, and the second byte's range
        if (c >= 0xC2u && c <= 0xDFu) more = 1;
        else if (c >= 0xE0u && c <= 0xEFu) { more = 2; lo = c == 0xE0u ? 0xA0u : 0x80u; hi = c == 0xEDu ? 0x9Fu : 0xBFu; }
        else if (c >= 0xF0u && c <= 0xF4u) { more = 3; lo = c == 0xF0u ? 0x90u : 0x80u; hi = c == 0xF4u ? 0x8Fu : 0xBFu; }
        else return false;
        if (len - i <= more) return false;
        if (s[i + 1] < lo || s[i + 1] > hi) return false;
        for (uint32_t k = 2; k <= more; k++)
            if ((s[i + k] & 0xC0u) != 0x80u) return false;
        i += more + 1;
    }
    return true;
}
// the interface table's strings, 4-byte aligned in their row: an all-ASCII string (the usual one) is checked a word at a
// time, any other by utf8_valid
__device__ __forceinline__ bool utf8_valid_row(const char* str, uint32_t len) {
    const uint8_t* s = reinterpret_cast<const uint8_t*>(str);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(s);
    uint32_t high = 0;
    for (uint32_t k = 0; k < len / 4u; k++) high |= w[k];
    for (uint32_t k = len & ~3u; k < len; k++) high |= s[k];
    return (high & 0x80808080u) == 0u || utf8_valid(s, len);
}

__device__ __forceinline__ uint32_t vlen(uint64_t v) { return v == 0 ? 1u : (uint32_t)(64 - __clzll((long long)v) + 6) / 7u; }
template <class S> __device__ __forceinline__ void put_varint(S& s, uint64_t v) {
    while (v >= 0x80u) { s.put((uint8_t)(v | 0x80u)); v >>= 7; }
    s.put((uint8_t)v);
}
template <class S> __device__ __forceinline__ void put_tag(S& s, uint32_t field, uint32_t wire) { put_varint(s, (field << 3) | wire); }
// scalar varint field, proto3: zero is not written
template <class S> __device__ __forceinline__ void f_varint(S& s, uint32_t field, uint64_t v) {
    if (v) { put_tag(s, field, 0); put_varint(s, v); }
}
__device__ __forceinline__ uint32_t f_varint_len(uint32_t field, uint64_t v) { return v ? vlen((uint64_t)field << 3) + vlen(v) : 0u; }
template <class S> __device__ __forceinline__ void f_bytes(S& s, uint32_t field, const uint8_t* b, uint32_t len) {
    if (len) { put_tag(s, field, 2); put_varint(s, len); for (uint32_t i = 0; i < len; i++) s.put(b[i]); }
}
__device__ __forceinline__ uint32_t f_bytes_len(uint32_t field, uint32_t len) { return len ? vlen((uint64_t)field << 3) + vlen(len) + len : 0u; }

// google.protobuf.Timestamp / Duration {1: int64 seconds, 2: int32 nanos}
__device__ __forceinline__ uint32_t secnanos_len(int64_t sec, int32_t nanos) {
    return f_varint_len(1, (uint64_t)sec) + f_varint_len(2, (uint64_t)(int64_t)nanos);
}
template <class S> __device__ __forceinline__ void f_secnanos(S& s, uint32_t field, int64_t sec, int32_t nanos) {
    put_tag(s, field, 2); put_varint(s, secnanos_len(sec, nanos));
    f_varint(s, 1, (uint64_t)sec); f_varint(s, 2, (uint64_t)(int64_t)nanos);
}
// IP {oneof: fixed32 ipv4 = 1 | bytes ipv6 = 2}; a set oneof member is written even when it is zero
template <class S> __device__ __forceinline__ void f_ip(S& s, uint32_t field, const uint8_t* ip16, bool v4) {
    put_tag(s, field, 2);
    if (v4) { put_varint(s, 5); s.put(0x0D); s.put(ip16[15]); s.put(ip16[14]); s.put(ip16[13]); s.put(ip16[12]); }   // BigEndian.Uint32, little-endian on the wire
    else { put_varint(s, 18); s.put(0x12); s.put(16); for (int i = 0; i < 16; i++) s.put(ip16[i]); }
}
__device__ __forceinline__ uint32_t f_ip_len(uint32_t field, bool v4) { return vlen((uint64_t)field << 3) + 1u + (v4 ? 5u : 18u); }

// wall clock of a monotonic timestamp: currentTime.Add(-Duration(monoNow - mono)) -> (Unix(), Nanosecond()).
// In seconds + nanoseconds, as time.Time.Add does, so that a result outside the int64 nanosecond range (before 1677 or
// after 2262) stays exact; Go's negation wraps, -Duration(MinInt64) == MinInt64, which is Duration(mono - monoNow).
__device__ __forceinline__ void wall_of(uint64_t now_unix_ns, uint64_t mono_now, uint64_t mono, int64_t& sec, int32_t& nanos) {
    const int64_t d = (int64_t)(mono - mono_now);
    int64_t s = (int64_t)(now_unix_ns / 1000000000ull) + d / 1000000000ll;
    int64_t ns = (int64_t)(now_unix_ns % 1000000000ull) + d % 1000000000ll;     // in (-1e9, 2e9)
    if (ns >= 1000000000ll) { ns -= 1000000000ll; s++; }             // Go: Unix() floors, Nanosecond() is in [0, 1e9)
    else if (ns < 0) { ns += 1000000000ll; s--; }
    sec = s; nanos = (int32_t)ns;
}
// durationpb.New(d): seconds and nanos truncate towards zero, same sign
__device__ __forceinline__ void dur_of(uint64_t ns, int64_t& sec, int32_t& nanos) {
    const int64_t d = (int64_t)ns;
    sec = d / 1000000000ll; nanos = (int32_t)(d % 1000000000ll);
}
// macToUint64 (proto.go:244-251): 11:22:33:44:55:66 -> 0x112233445566
__device__ __forceinline__ uint64_t mac_u64(const uint8_t* m) {
    return ((uint64_t)m[0] << 40) | ((uint64_t)m[1] << 32) | ((uint64_t)m[2] << 24) | ((uint64_t)m[3] << 16) | ((uint64_t)m[4] << 8) | m[5];
}
// utils.DNSRawNameToDotted (pkg/utils/dns.go:20-60): label format -> dotted, stops at NUL / compression pointer / overrun
__device__ __forceinline__ uint32_t dns_dotted(const uint8_t* raw32, uint8_t* out) {
    uint32_t blen = 0;
    while (blen < 32 && raw32[blen] != 0) blen++;
    uint32_t i = 0, o = 0;
    bool first = true;
    while (i < blen) {
        const uint32_t l = raw32[i];
        if (l == 0 || (l & 0xC0u) == 0xC0u) break;
        i++;
        if (i + l > blen) break;
        if (!first) out[o++] = '.';
        first = false;
        for (uint32_t k = 0; k < l; k++) out[o++] = raw32[i + k];
        i += l;
    }
    return o;
}
// interfaceNamer (pkg/agent/interfaces_listener.go:74-80 over ifaces.Registerer.ifaceCacheLookup, registerer.go:153-190):
// one row for the index -> that name whatever the MAC; several -> the row with this MAC, else the first; none -> "unknown"
__device__ __forceinline__ const PbIface* iface_lookup(const PbParams& P, uint32_t if_index, const uint8_t* mac) {
    const PbIface* first = nullptr; const PbIface* exact = nullptr;
    uint32_t rows = 0;
    for (uint32_t i = 0; i < P.n_ifaces; i++) {
        const PbIface* r = &P.ifaces[i];
        if (r->if_index != if_index) continue;
        if (!first) first = r;
        rows++;
        bool same = true;
        for (int b = 0; b < 6; b++) same = same && r->mac[b] == mac[b];
        if (same && !exact) exact = r;
    }
    if (rows <= 1) return first;
    return exact ? exact : first;
}
template <class S> __device__ __forceinline__ void f_dup_entry(S& s, const PbParams& P, uint32_t if_index, const uint8_t* lmac, uint32_t dir) {
    const PbIface* r = iface_lookup(P, if_index, lmac);
    const uint8_t* name = r ? reinterpret_cast<const uint8_t*>(r->name) : reinterpret_cast<const uint8_t*>("unknown");
    const uint32_t nlen = r ? min((uint32_t)r->name_len, 16u) : 7u;
    const uint8_t* udn = r ? reinterpret_cast<const uint8_t*>(r->udn) : nullptr;
    const uint32_t ulen = r ? min((uint32_t)r->udn_len, 64u) : 0u;
    if constexpr (S::kCounts) s.ok = s.ok && (!r || (utf8_valid_row(r->name, nlen) && utf8_valid_row(r->udn, ulen)));   // "unknown" is ASCII
    put_tag(s, 26, 2);
    put_varint(s, f_bytes_len(1, nlen) + f_varint_len(2, dir) + f_bytes_len(3, ulen));
    f_bytes(s, 1, name, nlen); f_varint(s, 2, dir); f_bytes(s, 3, udn, ulen);
}

// One pbflow.Record.  rec: 144-byte flow record; dns / add / drop: feature blocks or nullptr (absent).
template <class S>
__device__ void pb_encode_record(S& s, const uint8_t* rec, const uint8_t* dns, const uint8_t* add, const uint8_t* drop, const PbParams& P) {
    const uint8_t* id = rec; const uint8_t* m = rec + 40;
    const uint64_t start = *reinterpret_cast<const uint64_t*>(m + 0), end = *reinterpret_cast<const uint64_t*>(m + 8);
    const uint64_t bytes = *reinterpret_cast<const uint64_t*>(m + 16);
    const uint32_t packets = *reinterpret_cast<const uint32_t*>(m + 24);
    const uint32_t eth = *reinterpret_cast<const uint16_t*>(m + 28), flags = *reinterpret_cast<const uint16_t*>(m + 30);
    const uint32_t if_first = *reinterpret_cast<const uint32_t*>(m + 44), sampling = *reinterpret_cast<const uint32_t*>(m + 52);
    const uint32_t dir = m[56], dscp = m[58];
    uint32_t nobs = m[59]; if (nobs > 6u) nobs = 6u;
    const uint32_t ssl = *reinterpret_cast<const uint16_t*>(m + 92), cipher = *reinterpret_cast<const uint16_t*>(m + 94);
    const uint32_t keyshare = *reinterpret_cast<const uint16_t*>(m + 96), tls_types = m[98], misc = m[99];
    const bool v6 = eth == 0x86DDu;

    f_varint(s, 1, eth);
    f_varint(s, 2, dir);
    int64_t sec; int32_t nanos;
    wall_of(P.now_unix_ns, P.mono_now_ns, start, sec, nanos); f_secnanos(s, 3, sec, nanos);
    wall_of(P.now_unix_ns, P.mono_now_ns, end, sec, nanos);   f_secnanos(s, 4, sec, nanos);
    const uint64_t smac = mac_u64(m + 32), dmac = mac_u64(m + 38);
    put_tag(s, 5, 2); put_varint(s, f_varint_len(1, smac) + f_varint_len(2, dmac)); f_varint(s, 1, smac); f_varint(s, 2, dmac);
    put_tag(s, 6, 2); put_varint(s, f_ip_len(1, !v6) + f_ip_len(2, !v6) + f_varint_len(3, dscp));
    f_ip(s, 1, id, !v6); f_ip(s, 2, id + 16, !v6); f_varint(s, 3, dscp);
    const uint32_t sport = *reinterpret_cast<const uint16_t*>(id + 32), dport = *reinterpret_cast<const uint16_t*>(id + 34), proto = id[36];
    put_tag(s, 7, 2); put_varint(s, f_varint_len(1, sport) + f_varint_len(2, dport) + f_varint_len(3, proto));
    f_varint(s, 1, sport); f_varint(s, 2, dport); f_varint(s, 3, proto);
    f_varint(s, 8, bytes);
    f_varint(s, 9, packets);
    f_ip(s, 12, P.agent_ip, P.agent_is_v4 != 0);
    f_varint(s, 13, flags);
    f_varint(s, 14, id[37]);
    f_varint(s, 15, id[38]);
    if (drop) {                                                            // proto.go:86-92
        f_varint(s, 16, *reinterpret_cast<const uint16_t*>(drop + 16));
        f_varint(s, 17, *reinterpret_cast<const uint16_t*>(drop + 18));
        f_varint(s, 18, *reinterpret_cast<const uint16_t*>(drop + 24));
        f_varint(s, 19, drop[28]);
        f_varint(s, 20, *reinterpret_cast<const uint32_t*>(drop + 20));
    }
    uint8_t dname[32]; uint32_t dname_len = 0;
    if (dns) {                                                             // proto.go:73-85
        f_varint(s, 21, *reinterpret_cast<const uint16_t*>(dns + 24));
        f_varint(s, 22, *reinterpret_cast<const uint16_t*>(dns + 26));
        const uint64_t lat = *reinterpret_cast<const uint64_t*>(dns + 16);
        if (lat) { dur_of(lat, sec, nanos); f_secnanos(s, 23, sec, nanos); }
        dname_len = dns_dotted(dns + 31, dname);
        if constexpr (S::kCounts) s.ok = s.ok && utf8_valid(dname, dname_len);
    }
    dur_of(add ? *reinterpret_cast<const uint64_t*>(add + 16) : 0ull, sec, nanos);   // record.go:123-127; always a message
    f_secnanos(s, 24, sec, nanos);
    if (dns) f_varint(s, 25, dns[30]);
    const uint8_t* lmac = dir == 0 ? m + 38 : m + 32;                      // record.go:100-103
    f_dup_entry(s, P, if_first, lmac, dir);
    for (uint32_t i = 0; i < nobs; i++) f_dup_entry(s, P, *reinterpret_cast<const uint32_t*>(m + 68 + 4 * i), lmac, m[60 + i]);
    f_varint(s, 29, sampling);
    if (add) {                                                             // proto.go:100-105
        f_varint(s, 30, add[30] ? 1u : 0u);
        f_varint(s, 31, (uint64_t)(int64_t)*reinterpret_cast<const int32_t*>(add + 24));
    }
    f_bytes(s, 32, dname, dname_len);
    f_varint(s, 33, ssl);
    f_varint(s, 34, (misc & 0x01u) ? 1u : 0u);                             // HasSSLMismatch, record.go:29,255-257
    f_varint(s, 35, tls_types);
    f_varint(s, 36, cipher);
    f_varint(s, 37, keyshare);
}

__device__ __forceinline__ void pb_blocks(const PbInputs& in, size_t i, const uint8_t*& dns, const uint8_t*& add, const uint8_t*& drop) {
    const uint8_t pr = in.present ? in.present[i] : 0;
    dns = (in.dns && (pr & 1)) ? in.dns + i * 64 : nullptr;
    add = (in.add && (pr & 2)) ? in.add + i * 32 : nullptr;
    drop = (in.drop && (pr & 4)) ? in.drop + i * 32 : nullptr;
}

__global__ void pb_size_kernel(PbInputs in, uint32_t n, PbParams P, uint32_t* __restrict__ sizes) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint8_t *dns, *add, *drop;
        pb_blocks(in, i, dns, add, drop);
        CountSink c;
        pb_encode_record(c, in.recs + (size_t)i * kRecBytes, dns, add, drop, P);
        sizes[i] = c.ok ? c.n : 0u;                                        // body length (0: dropped); the wrapper is added by pb_total
    }
}

// a dropped record (body 0) gets no Records entry either
__device__ __forceinline__ uint32_t pb_total(uint32_t body, uint32_t wrap) { return wrap && body ? 1u + vlen(body) + body : body; }

// exclusive scan of n u32 into u64 offsets (n + 1 entries): per-block sums, one block over the sums, add back
constexpr int kScanBlock = 1024;
__global__ void pb_scan_block_kernel(const uint32_t* __restrict__ sizes, uint32_t n, uint32_t wrap, unsigned long long* __restrict__ offsets,
                                     unsigned long long* __restrict__ block_sums) {
    __shared__ unsigned long long sh[kScanBlock];
    const uint32_t i = blockIdx.x * kScanBlock + threadIdx.x;
    const unsigned long long v = i < n ? pb_total(sizes[i], wrap) : 0ull;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int d = 1; d < kScanBlock; d <<= 1) {
        const unsigned long long a = threadIdx.x >= (unsigned)d ? sh[threadIdx.x - d] : 0ull;
        __syncthreads();
        sh[threadIdx.x] += a;
        __syncthreads();
    }
    if (i < n) offsets[i] = sh[threadIdx.x] - v;                          // exclusive, block-local
    if (threadIdx.x == kScanBlock - 1) block_sums[blockIdx.x] = sh[threadIdx.x];
}
__global__ void pb_scan_sums_kernel(unsigned long long* block_sums, uint32_t n_blocks) {       // one CTA
    __shared__ unsigned long long carry;
    __shared__ unsigned long long sh[kScanBlock];
    if (threadIdx.x == 0) carry = 0ull;
    __syncthreads();
    for (uint32_t base = 0; base < n_blocks; base += kScanBlock) {
        const uint32_t i = base + threadIdx.x;
        const unsigned long long v = i < n_blocks ? block_sums[i] : 0ull;
        sh[threadIdx.x] = v;
        __syncthreads();
        for (int d = 1; d < kScanBlock; d <<= 1) {
            const unsigned long long a = threadIdx.x >= (unsigned)d ? sh[threadIdx.x - d] : 0ull;
            __syncthreads();
            sh[threadIdx.x] += a;
            __syncthreads();
        }
        if (i < n_blocks) block_sums[i] = carry + sh[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == kScanBlock - 1) carry += sh[threadIdx.x];
        __syncthreads();
    }
}
__global__ void pb_scan_add_kernel(unsigned long long* __restrict__ offsets, uint32_t n, const unsigned long long* __restrict__ block_sums,
                                   const uint32_t* __restrict__ sizes, uint32_t wrap) {
    const uint32_t i = blockIdx.x * kScanBlock + threadIdx.x;
    if (i < n) {
        const unsigned long long o = offsets[i] + block_sums[blockIdx.x];
        offsets[i] = o;
        if (i == n - 1) offsets[n] = o + pb_total(sizes[i], wrap);
    }
}

constexpr int kPbCta = 256;                    // flows per CTA of the write kernel
constexpr int kPbStage = 64 * 1024;            // shared-memory image of the CTA's output range
__global__ void __launch_bounds__(kPbCta)
pb_write_kernel(PbInputs in, uint32_t n, PbParams P, const unsigned long long* __restrict__ offsets, const uint32_t* __restrict__ sizes,
                uint8_t* __restrict__ out, uint8_t* __restrict__ keys_out) {
    FA_DYN_SMEM(stage);
    const uint32_t first = blockIdx.x * kPbCta;
    const uint32_t last = min(n, first + kPbCta);
    const unsigned long long base = offsets[first], total = offsets[last] - base;
    const uint32_t skew = (uint32_t)((uintptr_t)(out + base) & 15u);          // keep shared and global 16-byte phases equal
    const bool staged = total + skew <= (unsigned long long)kPbStage;
    const uint32_t i = first + threadIdx.x;
    if (i < last) {
        if (sizes[i]) {                                                        // 0: dropped by the size pass
            const uint8_t *dns, *add, *drop;
            pb_blocks(in, i, dns, add, drop);
            const unsigned long long off = offsets[i] - base;
            ByteSink w{staged ? stage + skew + off : out + base + off};
            if (P.wrap) {                                                      // Records.entries = 1, length-delimited
                w.put(0x0A); put_varint(w, sizes[i]);
            }
            pb_encode_record(w, in.recs + (size_t)i * kRecBytes, dns, add, drop, P);
        }
        if (keys_out) {                                                        // getFlowKey: the smaller address first
            const uint8_t* id = in.recs + (size_t)i * kRecBytes;
            int cmp = 0;
            for (int k = 0; k < 16 && cmp == 0; k++) cmp = (int)id[k] - (int)id[16 + k];
            const uint8_t* a = cmp <= 0 ? id : id + 16; const uint8_t* b = cmp <= 0 ? id + 16 : id;
            uint8_t* K = keys_out + (size_t)i * 32;
            for (int k = 0; k < 16; k++) { K[k] = a[k]; K[16 + k] = b[k]; }
        }
    }
    if (!staged) return;
    __syncthreads();
    uint8_t* g = out + base;
    const uint32_t tot = (uint32_t)total;
    const uint32_t head = min(tot, (16u - skew) & 15u);                        // bytes before the first 16-byte boundary
    if (threadIdx.x < head) g[threadIdx.x] = stage[skew + threadIdx.x];
    const uint32_t vec = (tot - head) / 16u;
    const uint4* sv = reinterpret_cast<const uint4*>(stage + skew + head);
    uint4* gv = reinterpret_cast<uint4*>(g + head);
    for (uint32_t k = threadIdx.x; k < vec; k += kPbCta) gv[k] = sv[k];
    const uint32_t tail0 = head + vec * 16u;
    if (tail0 + threadIdx.x < tot) g[tail0 + threadIdx.x] = stage[skew + tail0 + threadIdx.x];
}

#ifndef FA_HOST_EMUL
// sizes: n u32, offsets: n + 1 u64, block_sums: ceil(n / 1024) u64 (device scratch).  Returns kernels launched.
int launch_pb_sizes(const PbInputs& in, uint32_t n, const PbParams& P, uint32_t* sizes, unsigned long long* offsets,
                    unsigned long long* block_sums, int sm_count, cudaStream_t st) {
    if (!n) return 0;
    const uint32_t nb = (n + kScanBlock - 1) / kScanBlock;
    pb_size_kernel<<<min((uint32_t)(sm_count * 8), (n + 255u) / 256u), 256, 0, st>>>(in, n, P, sizes);
    pb_scan_block_kernel<<<nb, kScanBlock, 0, st>>>(sizes, n, P.wrap, offsets, block_sums);
    pb_scan_sums_kernel<<<1, kScanBlock, 0, st>>>(block_sums, nb);
    pb_scan_add_kernel<<<nb, kScanBlock, 0, st>>>(offsets, n, block_sums, sizes, P.wrap);
    return 4;
}
int launch_pb_write(const PbInputs& in, uint32_t n, const PbParams& P, const unsigned long long* offsets, const uint32_t* sizes,
                    uint8_t* out, uint8_t* keys_out, cudaStream_t st) {
    if (!n) return 0;
    static bool attr_done[64] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (!attr_done[dev & 63]) { cudaFuncSetAttribute(pb_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPbStage); attr_done[dev & 63] = true; }
    pb_write_kernel<<<(n + kPbCta - 1) / kPbCta, kPbCta, kPbStage, st>>>(in, n, P, offsets, sizes, out, keys_out);
    return 1;
}
#endif

}  // namespace fa
