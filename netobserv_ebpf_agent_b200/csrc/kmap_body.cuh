// kmap_body.cuh — KERNEL_MAP mode: the per-thread bodies of the kernels that reproduce the map update of
// flow_monitor (reference bpf/flows.c:222-288: lookup, update_existing_flow :98-143, add_observed_intf :76-96,
// insert with BPF_NOEXIST, ring-buffer fallback :262-279).
//
// The map update is a sequential program per flow (first-seen interface decides what counts, "last writer" fields,
// an ordered list of other interfaces).  It is made data-parallel by splitting one batch into passes whose bodies
// only use commutative atomics; the kernel boundary between two passes is the only ordering they need:
//
//   resolve   record -> table slot (find, or claim + publish while the map has room); flows born in this batch
//             elect their creating record = the smallest stream index
//   init      the creating record writes the new flow (flows.c:228-245)
//   fold      every other record, classified against the flow's first-seen interface:
//               A same interface      packets += 1, bytes += len, flags |=, tls_types |=, max of the stream index
//                                     over {all, dscp/sampling, cipher, key share}, min index with a TLS version
//               B another interface   flags |=, max index, (flow, ifindex) entered into a scratch set with the
//                                     smallest index it was seen at, chained to its flow
//               C ifindex 0 on a flow first seen elsewhere: the reference does nothing
//   bresolve  one thread per flow with B records: which of its new interfaces enter observed_intf[] (the
//             first 6 - nb by stream index), their slots, and the index at which the list filled up
//   order     the records that turned out to be "last" write end / dscp / sampling / cipher / key share; TLS
//             version + mismatch; direction merge of B records before the list filled, OBSERVED_INTF_MISSED after
//   cleanup   per-batch scratch back to zero
//
// Every body is a plain function of (record index, KmParams) so that the same text runs on the device (one
// thread per index) and in the host emulation used by tests/test_kmap_emulation.py (indices in shuffled order,
// atomics = plain operations).  The product library only ever launches the device kernels (kmap.cu).
#pragma once
#include "common.cuh"

namespace fa {

// ---- metrics offsets inside the 104-byte flow_metrics (bpf/types.h:94-126) ----------------------------------
constexpr int KM_START = 0, KM_END = 8, KM_BYTES = 16, KM_PACKETS = 24, KM_ETH = 28, KM_FLAGS = 30, KM_SRCMAC = 32,
              KM_DSTMAC = 38, KM_IFINDEX = 44, KM_SAMPLING = 52, KM_DIR = 56, KM_ERRNO = 57, KM_DSCP = 58, KM_NBOBS = 59,
              KM_OBSDIR = 60, KM_OBSINTF = 68, KM_SSLVER = 92, KM_CIPHER = 94, KM_KEYSHARE = 96, KM_TLSTYPES = 98,
              KM_MISC = 99;
constexpr int kMaxObservedIntf = 6;                 // MAX_OBSERVED_INTERFACES (bpf/types.h)
constexpr int kMetLineBytes = 128;                  // one line per slot: 104 B metrics + 24 B spare

// ---- per-batch scratch inside the identity line (bytes 48..84), all-zero between batches --------------------
constexpr int KS_NFIRST = 48;      // max ~i over the flow's records      (only read for flows born in this batch)
constexpr int KS_LAST_AB = 52;     // max i+1 over class A and B records  -> end
constexpr int KS_LAST_A = 56;      // max i+1 over class A records        -> dscp, sampling
constexpr int KS_LAST_CIPHER = 60; // max i+1 over A records with cipher > 0 in a SERVER_HELLO
constexpr int KS_LAST_KEYSHARE = 64;
constexpr int KS_NFIRST_VER = 68;  // max ~i over A records with a TLS version
constexpr int KS_BHEAD = 72;       // 1 + index of the newest (flow, ifindex) set entry of this flow
constexpr int KS_FULLAT = 76;      // 0: list never full in this batch; 1: full before it; i+2: filled by record i
constexpr int KS_END = 80;
// v2 only (per-flow finalisation): TLS versions seen on class A records, so that the mismatch flag needs no second
// look at the records
constexpr int KS_HVMAX = 80;       // max version
constexpr int KS_NHVMIN = 84;      // max ~version (low 16 bits) | 0x10000 -> min version; 0 = none seen
constexpr int KS_END2 = 88;

constexpr uint32_t kKmNone = 0xFFFFFFFFu;     // slot_of[i]: the record found no room (spilled / counted)
constexpr uint32_t kKmBorn = 0x80000000u;     // slot_of[i] bit 31: the record's flow was created in this batch

// (flow, ifindex) scratch set entry
struct KmBEntry {
    unsigned long long key;   // (slot + 1) << 32 | ifindex, 0 = empty
    uint32_t nfirst;          // max ~i
    uint32_t next;            // 1 + index of the next entry of the same flow, 0 = end
    uint32_t kind;            // 0 unassigned, 1 already in observed_intf[], 2 added in this batch
    uint32_t pos;             // its position in observed_intf[]
};
static_assert(sizeof(KmBEntry) == 24, "KmBEntry");

struct KmCounters {
    unsigned long long intf_missed;      // OBSERVED_INTF_MISSED (flows.c:134-142)
    unsigned long long fail_create;      // HASHMAP_FAIL_CREATE_FLOW (flows.c:285)
    unsigned long long spill_cursor;     // single-packet records handed to the ring buffer
    unsigned long long spill_dropped;    // ... that found the ring buffer full
    unsigned long long bset_count;       // (flow, ifindex) entries created in this batch
    unsigned long long table_full;       // records that found the table physically full (sizing error)
    // v2: per-batch work lists
    unsigned long long touched_count;    // flows that received class A / B records or were created in this batch
    unsigned long long deferred_count;   // records of flows created in this batch (folded after their creator is known)
    unsigned long long brec_count;       // class B records (direction merge / missed counter after bresolve)
};

struct KmParams {
    const uint8_t* recs;       // n x 144 B
    uint32_t n;
    uint32_t lo, hi;           // resolve: index range of this launch
    int allow_insert;          // resolve: 0 = lookup only (the map is full from `lo` on)
    int ringbuf;               // ENABLE_FLOWS_RINGBUF_FALLBACK
    Table t;                   // ident + occ + mask
    uint8_t* met;              // slots x 128 B
    uint64_t epoch;
    uint32_t* slot_of;         // n
    unsigned long long* live;
    KmCounters* c;
    uint8_t* spill; unsigned long long spill_cap;
    KmBEntry* bset; uint32_t bset_mask; uint32_t* blist;
    uint32_t* touched; uint32_t* deferred; uint32_t* brec;      // v2 work lists, n entries each
};

// ---- memory helpers ------------------------------------------------------------------------------------------
FA_HD uint64_t km_ld64(const uint8_t* p) { return *reinterpret_cast<const uint64_t*>(p); }
FA_HD uint32_t km_ld32(const uint8_t* p) { return *reinterpret_cast<const uint32_t*>(p); }
FA_HD uint16_t km_ld16(const uint8_t* p) { return *reinterpret_cast<const uint16_t*>(p); }
FA_HD void km_st64(uint8_t* p, uint64_t v) { *reinterpret_cast<uint64_t*>(p) = v; }
FA_HD void km_st32(uint8_t* p, uint32_t v) { *reinterpret_cast<uint32_t*>(p) = v; }
FA_HD void km_st16(uint8_t* p, uint16_t v) { *reinterpret_cast<uint16_t*>(p) = v; }

#if defined(__CUDA_ARCH__)
__device__ __forceinline__ uint32_t km_add32(void* p, uint32_t v) { return atomicAdd(reinterpret_cast<unsigned int*>(p), v); }
__device__ __forceinline__ unsigned long long km_add64(void* p, unsigned long long v) { return atomicAdd(reinterpret_cast<unsigned long long*>(p), v); }
__device__ __forceinline__ void km_or32(void* p, uint32_t v) { atomicOr(reinterpret_cast<unsigned int*>(p), v); }
__device__ __forceinline__ void km_max32(void* p, uint32_t v) { atomicMax(reinterpret_cast<unsigned int*>(p), v); }
__device__ __forceinline__ uint32_t km_max32_ret(void* p, uint32_t v) { return atomicMax(reinterpret_cast<unsigned int*>(p), v); }
__device__ __forceinline__ uint32_t km_exch32(void* p, uint32_t v) { return atomicExch(reinterpret_cast<unsigned int*>(p), v); }
__device__ __forceinline__ unsigned long long km_cas64(void* p, unsigned long long cmp, unsigned long long v) { return atomicCAS(reinterpret_cast<unsigned long long*>(p), cmp, v); }
__device__ __forceinline__ unsigned long long km_ld_coherent64(const void* p) { return __ldcg(reinterpret_cast<const unsigned long long*>(p)); }
__device__ __forceinline__ uint32_t km_ld_coherent32(const void* p) { return __ldcg(reinterpret_cast<const unsigned int*>(p)); }
__device__ __forceinline__ void km_fence() { __threadfence(); }
__device__ __forceinline__ void km_publish64(void* p, unsigned long long v) { *reinterpret_cast<volatile unsigned long long*>(p) = v; }
// single-writer update of the low half of a word whose high half receives atomics in the same kernel
__device__ __forceinline__ void km_set_lo16(void* word, uint16_t v) {
    atomicAnd(reinterpret_cast<unsigned int*>(word), 0xFFFF0000u);
    atomicOr(reinterpret_cast<unsigned int*>(word), (unsigned int)v);
}
#elif defined(FA_HOST_EMUL)
// SIMT emulation (tests/emul/simt.h): one OS thread per CUDA thread, so these have to be real atomics
inline uint32_t km_add32(void* p, uint32_t v) { return __atomic_fetch_add(static_cast<uint32_t*>(p), v, __ATOMIC_SEQ_CST); }
inline unsigned long long km_add64(void* p, unsigned long long v) { return __atomic_fetch_add(static_cast<unsigned long long*>(p), v, __ATOMIC_SEQ_CST); }
inline void km_or32(void* p, uint32_t v) { __atomic_fetch_or(static_cast<uint32_t*>(p), v, __ATOMIC_SEQ_CST); }
inline void km_max32(void* p, uint32_t v) {
    uint32_t* q = static_cast<uint32_t*>(p); uint32_t cur = __atomic_load_n(q, __ATOMIC_SEQ_CST);
    while (cur < v && !__atomic_compare_exchange_n(q, &cur, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
}
inline uint32_t km_max32_ret(void* p, uint32_t v) {
    uint32_t* q = static_cast<uint32_t*>(p); uint32_t cur = __atomic_load_n(q, __ATOMIC_SEQ_CST);
    while (cur < v && !__atomic_compare_exchange_n(q, &cur, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return cur;
}
inline uint32_t km_exch32(void* p, uint32_t v) { return __atomic_exchange_n(static_cast<uint32_t*>(p), v, __ATOMIC_SEQ_CST); }
inline unsigned long long km_cas64(void* p, unsigned long long cmp, unsigned long long v) {
    __atomic_compare_exchange_n(static_cast<unsigned long long*>(p), &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST); return cmp;
}
inline unsigned long long km_ld_coherent64(const void* p) { return __atomic_load_n(static_cast<const unsigned long long*>(p), __ATOMIC_SEQ_CST); }
inline uint32_t km_ld_coherent32(const void* p) { return __atomic_load_n(static_cast<const uint32_t*>(p), __ATOMIC_SEQ_CST); }
inline void km_fence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void km_publish64(void* p, unsigned long long v) { __atomic_store_n(static_cast<unsigned long long*>(p), v, __ATOMIC_SEQ_CST); }
inline void km_set_lo16(void* word, uint16_t v) {
    __atomic_fetch_and(static_cast<uint32_t*>(word), 0xFFFF0000u, __ATOMIC_SEQ_CST);
    __atomic_fetch_or(static_cast<uint32_t*>(word), (uint32_t)v, __ATOMIC_SEQ_CST);
}
#else
inline uint32_t km_add32(void* p, uint32_t v) { uint32_t* q = static_cast<uint32_t*>(p); uint32_t o = *q; *q = o + v; return o; }
inline unsigned long long km_add64(void* p, unsigned long long v) { auto* q = static_cast<unsigned long long*>(p); auto o = *q; *q = o + v; return o; }
inline void km_or32(void* p, uint32_t v) { *static_cast<uint32_t*>(p) |= v; }
inline void km_max32(void* p, uint32_t v) { uint32_t* q = static_cast<uint32_t*>(p); if (*q < v) *q = v; }
inline uint32_t km_max32_ret(void* p, uint32_t v) { uint32_t* q = static_cast<uint32_t*>(p); uint32_t o = *q; if (o < v) *q = v; return o; }
inline uint32_t km_exch32(void* p, uint32_t v) { uint32_t* q = static_cast<uint32_t*>(p); uint32_t o = *q; *q = v; return o; }
inline unsigned long long km_cas64(void* p, unsigned long long cmp, unsigned long long v) { auto* q = static_cast<unsigned long long*>(p); auto o = *q; if (o == cmp) *q = v; return o; }
inline unsigned long long km_ld_coherent64(const void* p) { return *static_cast<const unsigned long long*>(p); }
inline uint32_t km_ld_coherent32(const void* p) { return *static_cast<const uint32_t*>(p); }
inline void km_fence() {}
inline void km_publish64(void* p, unsigned long long v) { *static_cast<unsigned long long*>(p) = v; }
inline void km_set_lo16(void* word, uint16_t v) { *static_cast<uint16_t*>(word) = v; }
#endif

FA_HD uint8_t* km_ident(const KmParams& P, uint32_t slot) { return reinterpret_cast<uint8_t*>(P.t.ident) + (size_t)slot * kIdentBytes; }
FA_HD uint8_t* km_met(const KmParams& P, uint32_t slot) { return P.met + (size_t)slot * kMetLineBytes; }
FA_HD const uint8_t* km_rec(const KmParams& P, uint32_t i) { return P.recs + (size_t)i * kRecBytes; }

// new_flow of flows.c:228-245 built from a packet event (padding, lock, errno, observed_* stay zero)
FA_HD void km_new_flow(const uint8_t* ev, uint8_t* nf /*104 B, 8-byte aligned*/, uint8_t err) {
    const uint64_t ts = km_ld64(ev + KM_START);
    km_st64(nf + KM_START, ts);
    km_st64(nf + KM_END, ts);
    km_st64(nf + KM_BYTES, km_ld64(ev + KM_BYTES));
    km_st32(nf + KM_PACKETS, 1u);
    km_st32(nf + KM_ETH, km_ld32(ev + KM_ETH));                      // eth_protocol + flags
    km_st64(nf + KM_SRCMAC, km_ld64(ev + KM_SRCMAC));                // src_mac + dst_mac[0..2)
    km_st32(nf + KM_SRCMAC + 8, km_ld32(ev + KM_SRCMAC + 8));        // dst_mac[2..6)
    km_st32(nf + KM_IFINDEX, km_ld32(ev + KM_IFINDEX));
    km_st32(nf + 48, 0u);                                            // lock
    km_st32(nf + KM_SAMPLING, km_ld32(ev + KM_SAMPLING));
    km_st32(nf + KM_DIR, (uint32_t)ev[KM_DIR] | ((uint32_t)err << 8) | ((uint32_t)ev[KM_DSCP] << 16));   // nb_observed_intf = 0
    km_st32(nf + 60, 0u); km_st32(nf + 64, 0u);                      // observed_direction + padding
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 6; k++) km_st32(nf + KM_OBSINTF + 4 * k, 0u);
    km_st32(nf + KM_SSLVER, km_ld32(ev + KM_SSLVER));                // ssl_version + tls_cipher_suite
    km_st32(nf + KM_KEYSHARE, (uint32_t)km_ld16(ev + KM_KEYSHARE) | ((uint32_t)ev[KM_TLSTYPES] << 16));  // misc_flags = 0
    km_st32(nf + 100, 0u);
}

// ---- resolve -------------------------------------------------------------------------------------------------
FA_HD void km_resolve_body(const KmParams& P, uint32_t i) {
    const uint8_t* R = km_rec(P, i);
    const uint64_t k0 = km_ld64(R), k1 = km_ld64(R + 8), k2 = km_ld64(R + 16), k3 = km_ld64(R + 24),
                   k4 = km_ld64(R + 32) & 0x00FFFFFFFFFFFFFFull;
    const uint64_t h = slot_hash(key_premix(k0, k1, k2, k3, k4));
    uint64_t slot = h & P.t.mask;
    uint32_t found = kKmNone;
    bool born_now = false;
    for (uint64_t probes = 0; probes <= P.t.mask; ) {
        uint8_t* L = km_ident(P, (uint32_t)slot);
        const unsigned long long tag = km_ld_coherent64(L + 40);
        const uint32_t state = (uint32_t)(tag & TAG_STATE_MASK);
        if (state == 0) {
            if (!P.allow_insert) break;                                            // miss while the map is full
            if (km_cas64(L + 40, 0ull, TAG_CLAIMED) == 0ull) {
                km_st64(L, k0); km_st64(L + 8, k1); km_st64(L + 16, k2); km_st64(L + 24, k3); km_st64(L + 32, k4);
                km_fence();
                km_publish64(L + 40, TAG_PUBLISHED | TAG_HAS_BASE | (P.epoch << TAG_EPOCH_SHIFT));
                km_or32(&P.t.occ[slot >> 5], 1u << (slot & 31));
                km_add64(P.live, 1ull);
                found = (uint32_t)slot; born_now = true;
                break;
            }
            continue;                                                              // lost the race: look again
        }
        if (state == (uint32_t)TAG_CLAIMED) continue;                              // key being written
        km_fence();
        if (km_ld_coherent64(L) == k0 && km_ld_coherent64(L + 8) == k1 && km_ld_coherent64(L + 16) == k2 &&
            km_ld_coherent64(L + 24) == k3 && (km_ld_coherent64(L + 32) & 0x00FFFFFFFFFFFFFFull) == k4) {
            if (!(tag & TAG_HAS_BASE)) {
                // the flow exists through feature samples only (tracer.go:1179-1182: an empty base): this packet
                // creates its kernel-map entry, i.e. the flow is born in this batch.  Not while the map is full.
                if (!P.allow_insert) break;
                km_cas64(L + 40, tag, (tag & ~(~0ull << TAG_EPOCH_SHIFT)) | TAG_HAS_BASE | (P.epoch << TAG_EPOCH_SHIFT));
                continue;                                                          // re-read the tag: ours or a peer's claim
            }
            found = (uint32_t)slot;
            born_now = (tag >> TAG_EPOCH_SHIFT) == P.epoch;
            break;
        }
        slot = (slot + 1) & P.t.mask;
        probes++;
        if (probes > P.t.mask) km_add64(&P.c->table_full, 1ull);
    }
    if (found != kKmNone) {
        P.slot_of[i] = found | (born_now ? kKmBorn : 0u);        // slots <= 2^30 (checked by fa_create)
        if (born_now) km_max32(km_ident(P, found) + KS_NFIRST, ~i);
        return;
    }
    P.slot_of[i] = kKmNone;
    // flows.c:262-286: the insert failed for a reason other than EEXIST
    if (P.ringbuf) {
        const unsigned long long at = km_add64(&P.c->spill_cursor, 1ull);
        if (at < P.spill_cap) {
            uint8_t* O = P.spill + (size_t)at * kRecBytes;
            km_st64(O, k0); km_st64(O + 8, k1); km_st64(O + 16, k2); km_st64(O + 24, k3); km_st64(O + 32, k4);
            km_new_flow(R + kKeyBytes, O + kKeyBytes, /*E2BIG*/ 7);
        } else {
            km_add64(&P.c->spill_dropped, 1ull);
        }
    } else {
        km_add64(&P.c->fail_create, 1ull);
    }
}

// true when record i created its flow in this batch (so = slot_of[i]: only flows born now look at the election)
FA_HD bool km_is_creator(const KmParams& P, uint32_t so, uint32_t i) {
    return (so & kKmBorn) && km_ld32(km_ident(P, so & ~kKmBorn) + KS_NFIRST) == ~i;
}

// ---- init ----------------------------------------------------------------------------------------------------
FA_HD void km_init_body(const KmParams& P, uint32_t i) {
    const uint32_t so = P.slot_of[i];
    if (so == kKmNone || !km_is_creator(P, so, i)) return;
    uint8_t* M = km_met(P, so & ~kKmBorn);
    km_new_flow(km_rec(P, i) + kKeyBytes, M, 0);
    km_st64(M + 104, 0ull); km_st64(M + 112, 0ull); km_st64(M + 120, 0ull);
}

// 0 = C (ignored), 1 = A (first-seen interface), 2 = B (another interface)
FA_HD int km_class(const uint8_t* M, uint32_t ifindex) {
    if (km_ld32(M + KM_IFINDEX) == ifindex) return 1;
    return ifindex != 0 ? 2 : 0;
}
FA_HD uint64_t km_bkey(uint32_t slot, uint32_t ifindex) { return ((uint64_t)(slot + 1) << 32) | ifindex; }
FA_HD uint32_t km_bhash(uint64_t key, uint32_t mask) { return (uint32_t)(fmix64(key) >> 20) & mask; }

// ---- fold ----------------------------------------------------------------------------------------------------
FA_HD void km_fold_body(const KmParams& P, uint32_t i) {
    const uint32_t so = P.slot_of[i];
    if (so == kKmNone || km_is_creator(P, so, i)) return;
    const uint32_t slot = so & ~kKmBorn;
    const uint8_t* ev = km_rec(P, i) + kKeyBytes;
    uint8_t* M = km_met(P, slot);
    uint8_t* L = km_ident(P, slot);
    const uint32_t ifindex = km_ld32(ev + KM_IFINDEX);
    const int cls = km_class(M, ifindex);
    if (cls == 0) return;
    const uint32_t flags = km_ld16(ev + KM_FLAGS);
    if (flags) km_or32(M + KM_ETH, flags << 16);
    km_max32(L + KS_LAST_AB, i + 1);
    if (cls == 1) {
        km_add32(M + KM_PACKETS, 1u);
        km_add64(M + KM_BYTES, km_ld64(ev + KM_BYTES));
        km_max32(L + KS_LAST_A, i + 1);
        const uint32_t ty = ev[KM_TLSTYPES];
        if (ty) km_or32(M + KM_KEYSHARE, ty << 16);
        if (ty == 0x02) {                                   // SERVER_HELLO (flows.c:119-124)
            if (km_ld16(ev + KM_CIPHER) > 0) km_max32(L + KS_LAST_CIPHER, i + 1);
            if (km_ld16(ev + KM_KEYSHARE) > 0) km_max32(L + KS_LAST_KEYSHARE, i + 1);
        }
        if (km_ld16(ev + KM_SSLVER) > 0) km_max32(L + KS_NFIRST_VER, ~i);
        return;
    }
    // class B: remember (flow, ifindex) with the first index it was seen at
    const uint64_t key = km_bkey(slot, ifindex);
    uint32_t s = km_bhash(key, P.bset_mask);
    for (;;) {
        KmBEntry* e = &P.bset[s];
        unsigned long long cur = km_ld_coherent64(&e->key);
        if (cur == 0ull) {
            cur = km_cas64(&e->key, 0ull, key);
            if (cur == 0ull) {                              // created: chain it to the flow, list it for cleanup
                e->next = km_exch32(L + KS_BHEAD, s + 1);
                P.blist[km_add64(&P.c->bset_count, 1ull)] = s;
                cur = key;
            }
        }
        if (cur == key) { km_max32(&e->nfirst, ~i); return; }
        s = (s + 1) & P.bset_mask;
    }
}

// ---- bresolve: one call per created (flow, ifindex) entry; the entry at the head of a flow's chain works ------
FA_HD void km_bresolve_body(const KmParams& P, uint32_t j) {
    const uint32_t s0 = P.blist[j];
    const uint32_t slot = (uint32_t)(P.bset[s0].key >> 32) - 1u;
    uint8_t* L = km_ident(P, slot);
    if (km_ld32(L + KS_BHEAD) != s0 + 1) return;
    uint8_t* M = km_met(P, slot);
    uint32_t nb = M[KM_NBOBS];
    if (nb >= (uint32_t)kMaxObservedIntf) { km_st32(L + KS_FULLAT, 1u); return; }   // add_observed_intf returns 1 at once
    // interfaces already listed keep their position
    for (uint32_t x = s0 + 1; x != 0; x = P.bset[x - 1].next) {
        KmBEntry* e = &P.bset[x - 1];
        const uint32_t ifindex = (uint32_t)e->key;
        for (uint32_t k = 0; k < nb; k++)
            if (km_ld32(M + KM_OBSINTF + 4 * k) == ifindex) { e->kind = 1; e->pos = k; break; }
    }
    // new interfaces enter in the order of their first record while there is room (flows.c:90-94)
    long long last = -1;
    uint32_t full_at = 0;
    while (nb < (uint32_t)kMaxObservedIntf) {
        KmBEntry* best = nullptr; long long best_first = 0;
        for (uint32_t x = s0 + 1; x != 0; x = P.bset[x - 1].next) {
            KmBEntry* e = &P.bset[x - 1];
            if (e->kind != 0) continue;
            const long long first = (long long)(uint32_t)~e->nfirst;
            if (first > last && (!best || first < best_first)) { best = e; best_first = first; }
        }
        if (!best) break;
        km_st32(M + KM_OBSINTF + 4 * nb, (uint32_t)best->key);
        M[KM_OBSDIR + nb] = km_rec(P, (uint32_t)best_first)[kKeyBytes + KM_DIR];
        best->kind = 2; best->pos = nb;
        last = best_first;
        nb++;
        if (nb == (uint32_t)kMaxObservedIntf) full_at = (uint32_t)best_first + 2u;
    }
    M[KM_NBOBS] = (uint8_t)nb;
    km_st32(L + KS_FULLAT, full_at);
}

// ---- order ---------------------------------------------------------------------------------------------------
FA_HD void km_order_body(const KmParams& P, uint32_t i) {
    const uint32_t so = P.slot_of[i];
    if (so == kKmNone || km_is_creator(P, so, i)) return;
    const uint32_t slot = so & ~kKmBorn;
    const uint8_t* R = km_rec(P, i);
    const uint8_t* ev = R + kKeyBytes;
    uint8_t* M = km_met(P, slot);
    const uint8_t* L = km_ident(P, slot);
    const uint32_t ifindex = km_ld32(ev + KM_IFINDEX);
    const int cls = km_class(M, ifindex);
    if (cls == 0) return;
    if (km_ld32(L + KS_LAST_AB) == i + 1) km_st64(M + KM_END, km_ld64(ev + KM_START));       // last writer (flows.c:107,128)
    if (cls == 1) {
        if (km_ld32(L + KS_LAST_A) == i + 1) {                                               // flows.c:109-110
            M[KM_DSCP] = ev[KM_DSCP];
            km_st32(M + KM_SAMPLING, km_ld32(ev + KM_SAMPLING));
        }
        if (km_ld32(L + KS_LAST_CIPHER) == i + 1) km_st16(M + KM_CIPHER, km_ld16(ev + KM_CIPHER));
        if (km_ld32(L + KS_LAST_KEYSHARE) == i + 1) km_set_lo16(M + KM_KEYSHARE, km_ld16(ev + KM_KEYSHARE));
        const uint16_t hv = km_ld16(ev + KM_SSLVER);
        if (hv > 0) {                                                                        // flows.c:111-118
            // the flow's version: the one it had, else the one of its first record carrying a version.  That
            // record stores exactly this value, so reading the field before or after its store gives the same.
            const uint32_t first_ver = ~km_ld32(L + KS_NFIRST_VER);
            uint16_t v = *reinterpret_cast<const volatile uint16_t*>(M + KM_SSLVER);
            if (v == 0) {
                v = km_ld16(km_rec(P, first_ver) + kKeyBytes + KM_SSLVER);
                if (first_ver == i) km_st16(M + KM_SSLVER, hv);
            }
            if (hv != v) km_or32(M + KM_KEYSHARE, 0x01u << 24);                              // MISC_FLAGS_SSL_MISMATCH
        }
        return;
    }
    // class B (flows.c:126-142)
    const uint32_t full_at = km_ld32(L + KS_FULLAT);
    if (full_at != 0 && i + 2u > full_at) {                 // the list was full when this record arrived
        if (R[36] != 0) km_add64(&P.c->intf_missed, 1ull);
        return;
    }
    const uint64_t key = km_bkey(slot, ifindex);
    uint32_t s = km_bhash(key, P.bset_mask);
    while (P.bset[s].key != key) s = (s + 1) & P.bset_mask;
    const KmBEntry* e = &P.bset[s];
    if (e->kind == 2 && (uint32_t)~e->nfirst == i) return;  // this record added the interface
    if (e->kind == 0) return;                               // unreachable: every interface seen before the list filled is listed
    volatile uint8_t* dirp = M + KM_OBSDIR + e->pos;
    const uint8_t cur = *dirp, d = ev[KM_DIR];
    if (cur != d && cur != 3) *dirp = 3;                    // OBSERVED_DIRECTION_BOTH (flows.c:83-86)
}

// ---- cleanup -------------------------------------------------------------------------------------------------
FA_HD void km_cleanup_record_body(const KmParams& P, uint32_t i) {
    const uint32_t so = P.slot_of[i];
    if (so == kKmNone) return;
    uint8_t* L = km_ident(P, so & ~kKmBorn);
    km_st64(L + 48, 0ull); km_st64(L + 56, 0ull); km_st64(L + 64, 0ull); km_st64(L + 72, 0ull);
}
FA_HD void km_cleanup_bset_body(const KmParams& P, uint32_t j) {
    KmBEntry* e = &P.bset[P.blist[j]];
    e->key = 0ull; e->nfirst = 0u; e->next = 0u; e->kind = 0u; e->pos = 0u;
}

// ================================================================================================================
// v2: the same decomposition with the per-record passes cut down to one.  Flows that existed before the batch know
// their first-seen interface already, so their records are classified and folded inside `resolve`; what is
// order-dependent is finished per FLOW (one thread per touched flow gathers the winning records by index) instead of
// per record.  Only the records of flows created in this batch (the creator is not known until all of them have been
// seen) and class B records (they need the result of bresolve) are revisited, through compact lists.
//   resolve+fold [records] -> init, fold [deferred records] -> bresolve [new (flow, ifindex)] -> order B [B records]
//   -> finish [touched flows] -> cleanup of the (flow, ifindex) set
// ================================================================================================================

// classify record i of an existing flow against its first-seen interface and fold the commutative parts
FA_HD void km2_fold_record(const KmParams& P, uint32_t slot, uint32_t i, bool list_touch) {
    const uint8_t* ev = km_rec(P, i) + kKeyBytes;
    uint8_t* M = km_met(P, slot);
    uint8_t* L = km_ident(P, slot);
    const uint32_t ifindex = km_ld32(ev + KM_IFINDEX);
    const int cls = km_class(M, ifindex);
    if (cls == 0) return;
    const uint32_t flags = km_ld16(ev + KM_FLAGS);
    if (flags) km_or32(M + KM_ETH, flags << 16);
    const uint32_t before = km_max32_ret(L + KS_LAST_AB, i + 1);
    if (list_touch && before == 0u) P.touched[km_add64(&P.c->touched_count, 1ull)] = slot;     // first A/B record of the flow
    if (cls == 1) {
        km_add32(M + KM_PACKETS, 1u);
        km_add64(M + KM_BYTES, km_ld64(ev + KM_BYTES));
        km_max32(L + KS_LAST_A, i + 1);
        const uint32_t ty = ev[KM_TLSTYPES];
        if (ty) km_or32(M + KM_KEYSHARE, ty << 16);
        if (ty == 0x02) {                                   // SERVER_HELLO (flows.c:119-124)
            if (km_ld16(ev + KM_CIPHER) > 0) km_max32(L + KS_LAST_CIPHER, i + 1);
            if (km_ld16(ev + KM_KEYSHARE) > 0) km_max32(L + KS_LAST_KEYSHARE, i + 1);
        }
        const uint32_t hv = km_ld16(ev + KM_SSLVER);
        if (hv > 0) {
            km_max32(L + KS_NFIRST_VER, ~i);
            km_max32(L + KS_HVMAX, hv);
            km_max32(L + KS_NHVMIN, 0x10000u | (~hv & 0xFFFFu));
        }
        return;
    }
    // class B: remember (flow, ifindex) with the first index it was seen at, and the record for the direction pass
    P.brec[km_add64(&P.c->brec_count, 1ull)] = i;
    const uint64_t key = km_bkey(slot, ifindex);
    uint32_t s = km_bhash(key, P.bset_mask);
    for (;;) {
        KmBEntry* e = &P.bset[s];
        unsigned long long cur = km_ld_coherent64(&e->key);
        if (cur == 0ull) {
            cur = km_cas64(&e->key, 0ull, key);
            if (cur == 0ull) {
                e->next = km_exch32(L + KS_BHEAD, s + 1);
                P.blist[km_add64(&P.c->bset_count, 1ull)] = s;
                cur = key;
            }
        }
        if (cur == key) { km_max32(&e->nfirst, ~i); return; }
        s = (s + 1) & P.bset_mask;
    }
}

FA_HD void km2_resolve_fold_body(const KmParams& P, uint32_t i) {
    km_resolve_body(P, i);
    const uint32_t so = P.slot_of[i];
    if (so == kKmNone) return;
    if (so & kKmBorn) { P.deferred[km_add64(&P.c->deferred_count, 1ull)] = i; return; }   // creator not known yet
    km2_fold_record(P, so, i, true);
}
FA_HD void km2_init_body(const KmParams& P, uint32_t k) {
    const uint32_t i = P.deferred[k];
    const uint32_t so = P.slot_of[i];
    if (!km_is_creator(P, so, i)) return;
    const uint32_t slot = so & ~kKmBorn;
    uint8_t* M = km_met(P, slot);
    km_new_flow(km_rec(P, i) + kKeyBytes, M, 0);
    km_st64(M + 104, 0ull); km_st64(M + 112, 0ull); km_st64(M + 120, 0ull);
    P.touched[km_add64(&P.c->touched_count, 1ull)] = slot;      // every flow created in this batch is finished below
}
FA_HD void km2_fold_deferred_body(const KmParams& P, uint32_t k) {
    const uint32_t i = P.deferred[k];
    const uint32_t so = P.slot_of[i];
    if (km_is_creator(P, so, i)) return;
    km2_fold_record(P, so & ~kKmBorn, i, false);
}
// class B record after bresolve (flows.c:126-142): missed counter or direction merge
FA_HD void km2_order_b_body(const KmParams& P, uint32_t k) {
    const uint32_t i = P.brec[k];
    const uint32_t slot = P.slot_of[i] & ~kKmBorn;
    const uint8_t* R = km_rec(P, i);
    const uint8_t* ev = R + kKeyBytes;
    uint8_t* M = km_met(P, slot);
    const uint8_t* L = km_ident(P, slot);
    const uint32_t full_at = km_ld32(L + KS_FULLAT);
    if (full_at != 0 && i + 2u > full_at) {
        if (R[36] != 0) km_add64(&P.c->intf_missed, 1ull);
        return;
    }
    const uint64_t key = km_bkey(slot, km_ld32(ev + KM_IFINDEX));
    uint32_t s = km_bhash(key, P.bset_mask);
    while (P.bset[s].key != key) s = (s + 1) & P.bset_mask;
    const KmBEntry* e = &P.bset[s];
    if (e->kind == 2 && (uint32_t)~e->nfirst == i) return;
    if (e->kind == 0) return;
    volatile uint8_t* dirp = M + KM_OBSDIR + e->pos;
    const uint8_t cur = *dirp, d = ev[KM_DIR];
    if (cur != d && cur != 3) *dirp = 3;
}
// one thread per touched flow: the order-dependent fields from the records that won, then the scratch back to zero
FA_HD void km2_finish_flow_body(const KmParams& P, uint32_t k) {
    const uint32_t slot = P.touched[k];
    uint8_t* M = km_met(P, slot);
    uint8_t* L = km_ident(P, slot);
    const uint32_t last_ab = km_ld32(L + KS_LAST_AB), last_a = km_ld32(L + KS_LAST_A);
    if (last_ab) km_st64(M + KM_END, km_ld64(km_rec(P, last_ab - 1) + kKeyBytes + KM_START));       // last writer
    if (last_a) {
        const uint8_t* ev = km_rec(P, last_a - 1) + kKeyBytes;
        M[KM_DSCP] = ev[KM_DSCP];
        km_st32(M + KM_SAMPLING, km_ld32(ev + KM_SAMPLING));
    }
    const uint32_t lc = km_ld32(L + KS_LAST_CIPHER), lk = km_ld32(L + KS_LAST_KEYSHARE);
    if (lc) km_st16(M + KM_CIPHER, km_ld16(km_rec(P, lc - 1) + kKeyBytes + KM_CIPHER));
    if (lk) km_st16(M + KM_KEYSHARE, km_ld16(km_rec(P, lk - 1) + kKeyBytes + KM_KEYSHARE));
    const uint32_t hvmax = km_ld32(L + KS_HVMAX);
    if (hvmax) {                                                       // flows.c:111-118 over all class A records
        const uint32_t hvmin = ~km_ld32(L + KS_NHVMIN) & 0xFFFFu;
        const uint32_t v0 = km_ld16(M + KM_SSLVER);
        if (v0 == 0) {                                                 // first record with a version sets it ...
            const uint32_t first_ver = ~km_ld32(L + KS_NFIRST_VER);
            km_st16(M + KM_SSLVER, km_ld16(km_rec(P, first_ver) + kKeyBytes + KM_SSLVER));
            if (hvmax != hvmin) M[KM_MISC] |= 0x01;                    // ... any other value afterwards is a mismatch
        } else if (hvmax != v0 || hvmin != v0) {
            M[KM_MISC] |= 0x01;
        }
    }
    km_st64(L + 48, 0ull); km_st64(L + 56, 0ull); km_st64(L + 64, 0ull); km_st64(L + 72, 0ull); km_st64(L + 80, 0ull);
}

// ---- evict: one call per occupancy word (32 slots) -------------------------------------------------------------
// the 144-byte record of `slot`: key (identity line) + flow_metrics (metric line).  Shared by the eviction and the
// fa_top_flows gather (evict.cu).
FA_HD void km_emit_record(const Table& t, const uint8_t* met, uint32_t slot, uint8_t* out_rec) {
    const uint64_t* L = reinterpret_cast<const uint64_t*>(reinterpret_cast<const uint8_t*>(t.ident) + (size_t)slot * kIdentBytes);
    const uint64_t* M = reinterpret_cast<const uint64_t*>(met + (size_t)slot * kMetLineBytes);
    uint64_t* O = reinterpret_cast<uint64_t*>(out_rec);
    for (int k = 0; k < 5; k++) O[k] = L[k];
    for (int k = 0; k < 13; k++) O[5 + k] = M[k];
}
FA_HD void km_evict_word_body(const Table& t, uint8_t* met, uint32_t w, uint8_t* out, unsigned long long cap,
                              unsigned long long* cursor, uint32_t* slot_of_out = nullptr) {
    uint32_t bits = t.occ[w];
    if (!bits) return;
    t.occ[w] = 0u;
    for (uint32_t b = 0; b < 32; b++) {
        if (!((bits >> b) & 1u)) continue;
        const uint32_t slot = w * 32 + b;
        uint64_t* L = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(t.ident) + (size_t)slot * kIdentBytes);
        uint64_t* M = reinterpret_cast<uint64_t*>(met + (size_t)slot * kMetLineBytes);
        const unsigned long long at = km_add64(cursor, 1ull);
        if (at < cap) {
            km_emit_record(t, met, slot, out + (size_t)at * kRecBytes);
            if (slot_of_out) slot_of_out[at] = slot;                    // for the feature pass (evict_features_kernel)
        }
        for (int k = 0; k < 16; k++) { L[k] = 0ull; M[k] = 0ull; }
    }
}

}  // namespace fa
