/*
 * flowagg.h — C ABI of the H100 flow-aggregation engine (libflowagg.so).
 *
 * This is the drop-in boundary for the netobserv agent's per-packet hot path.
 * A thin cgo wrapper (see INTEGRATION.md) implements the Go interface
 * `agent.ebpfFlowFetcher` (reference pkg/agent/agent.go:94-102) and the
 * gopipes stage `Accounter.Account` (reference pkg/flow/account.go:58) on top
 * of these entry points.  Only plain pointers and sizes cross the boundary;
 * no CUDA or torch types appear in any signature.
 *
 * Record layouts are an independent restatement of the agent's ring-buffer /
 * BPF-map ABI (offsets listed in SURVEY.md §8a, verified against the golden
 * byte vectors of reference pkg/model/record_test.go:19-102,193-224,323-347).
 * All integers are little-endian; every struct is "not packed" C layout.
 *
 * Error convention (mirrors the reference: never abort on data, count and
 * continue — pkg/tracer/tracer.go:1090-1092): every function returns an int,
 * 0 = OK, negative = -errno style failure (FA_E_*), positive = a condition the
 * caller is expected to handle (FA_FULL).
 *
 * Threading: at most one thread in fa_ingest*() and one other thread in
 * fa_evict()/fa_expire_flows()/fa_purge_stale_dns() at the same time (the reference's
 * model: one RingBufTracer/Accounter goroutine, one single-flight evictor —
 * pkg/flow/tracer_map.go:83-101).  The engine never retains a host pointer
 * after the call that received it returns.
 */
#ifndef FLOWAGG_H
#define FLOWAGG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FA_ABI_VERSION 1

/* ---------------------------------------------------------------- layouts */

#define FA_IP_LEN 16
#define FA_MAC_LEN 6
#define FA_MAX_OBSERVED_INTF 6
#define FA_DNS_NAME_LEN 32

/* Flow key, 40 bytes (reference bpf/types.h:191-204; Go mirror
 * pkg/ebpf/bpf_x86_bpfel.go:110-120).  IPv4 is carried as ::ffff:a.b.c.d.
 * Byte 39 is padding: ignored on input, always 0 on output (Go `==` on
 * BpfFlowId ignores the blank field). */
typedef struct fa_flow_id {
    uint8_t  src_ip[FA_IP_LEN];      /*  0 */
    uint8_t  dst_ip[FA_IP_LEN];      /* 16 */
    uint16_t src_port;               /* 32 host order */
    uint16_t dst_port;               /* 34 */
    uint8_t  transport_protocol;     /* 36 */
    uint8_t  icmp_type;              /* 37 */
    uint8_t  icmp_code;              /* 38 */
    uint8_t  pad_;                   /* 39 */
} fa_flow_id;

/* Per-flow accumulators, 104 bytes (reference bpf/types.h:94-126; Go mirror
 * pkg/ebpf/bpf_x86_bpfel.go:124-153). */
typedef struct fa_flow_metrics {
    uint64_t start_mono_time_ts;                        /*   0 */
    uint64_t end_mono_time_ts;                          /*   8 */
    uint64_t bytes;                                     /*  16 */
    uint32_t packets;                                   /*  24 wraps mod 2^32 */
    uint16_t eth_protocol;                              /*  28 */
    uint16_t flags;                                     /*  30 */
    uint8_t  src_mac[FA_MAC_LEN];                       /*  32 */
    uint8_t  dst_mac[FA_MAC_LEN];                       /*  38 */
    uint32_t if_index_first_seen;                       /*  44 */
    uint32_t lock;                                      /*  48 */
    uint32_t sampling;                                  /*  52 */
    uint8_t  direction_first_seen;                      /*  56 */
    uint8_t  errno_;                                    /*  57 */
    uint8_t  dscp;                                      /*  58 */
    uint8_t  nb_observed_intf;                          /*  59 */
    uint8_t  observed_direction[FA_MAX_OBSERVED_INTF];   /*  60 */
    uint8_t  pad0_[2];                                  /*  66 */
    uint32_t observed_intf[FA_MAX_OBSERVED_INTF];       /*  68 */
    uint16_t ssl_version;                               /*  92 */
    uint16_t tls_cipher_suite;                          /*  94 */
    uint16_t tls_key_share;                             /*  96 */
    uint8_t  tls_types;                                 /*  98 */
    uint8_t  misc_flags;                                /*  99 */
    uint8_t  pad1_[4];                                  /* 100 */
} fa_flow_metrics;

/* Ring-buffer wire record == Go model.RawRecord, 144 bytes
 * (reference bpf/types.h:212-215; pkg/model/record.go:63). */
typedef struct fa_flow_record {
    fa_flow_id      id;        /*  0 */
    fa_flow_metrics metrics;   /* 40 */
} fa_flow_record;

/* DNS feature metrics, 64 bytes (reference bpf/types.h:131-140). */
typedef struct fa_dns_metrics {
    uint64_t start_mono_time_ts;     /*  0 */
    uint64_t end_mono_time_ts;       /*  8 */
    uint64_t latency;                /* 16 */
    uint16_t id;                     /* 24 */
    uint16_t flags;                  /* 26 */
    uint16_t eth_protocol;           /* 28 */
    uint8_t  errno_;                 /* 30 */
    char     name[FA_DNS_NAME_LEN];  /* 31 */
    uint8_t  pad_;                   /* 63 */
} fa_dns_metrics;

/* RTT / IPsec feature metrics, 32 bytes (reference bpf/types.h:174-181). */
typedef struct fa_additional_metrics {
    uint64_t start_mono_time_ts;     /*  0 */
    uint64_t end_mono_time_ts;       /*  8 */
    uint64_t flow_rtt;               /* 16 */
    int32_t  ipsec_encrypted_ret;    /* 24 */
    uint16_t eth_protocol;           /* 28 */
    uint8_t  ipsec_encrypted;        /* 30 bool */
    uint8_t  pad_;                   /* 31 */
} fa_additional_metrics;

/* Packet-drop feature metrics, 32 bytes (reference bpf/types.h:142-151). */
typedef struct fa_pkt_drop_metrics {
    uint64_t start_mono_time_ts;     /*  0 */
    uint64_t end_mono_time_ts;       /*  8 */
    uint16_t bytes;                  /* 16 saturating */
    uint16_t packets;                /* 18 saturating */
    uint32_t latest_drop_cause;      /* 20 */
    uint16_t latest_flags;           /* 24 */
    uint16_t eth_protocol;           /* 26 */
    uint8_t  latest_state;           /* 28 */
    uint8_t  pad_[3];
} fa_pkt_drop_metrics;

/* Raw packet snapshot for fa_ingest_snaps ((f4), the front end of flow_monitor): 24 bytes of what the TC hook knows
 * about the skb, followed by the first (stride - 24) bytes of the frame, Ethernet header first.  `stride` is chosen by
 * the caller (a multiple of 8, 40..256): 88 carries a "64-byte header snap"; 104 reaches the TCP flags of an IPv6 frame
 * (14 + 40 + 20 = 74 header bytes).  cap_len = min(data_end - data, stride - 24) is the bound every header check of
 * bpf/utils.h:54-167 runs against (a header that does not fit is not parsed, exactly as there). */
typedef struct fa_packet_snap_hdr {
    uint64_t mono_ts;                /*  0 pkt.current_ts = bpf_ktime_get_ns() (flows.c:180) */
    uint32_t len;                    /*  8 skb->len */
    uint32_t if_index;               /* 12 skb->ifindex */
    uint32_t sampling;               /* 16 flow_sampling */
    uint16_t cap_len;                /* 20 valid bytes of data[] */
    uint8_t  direction;              /* 22 */
    uint8_t  pad_;                   /* 23 */
    /* uint8_t data[stride - 24] follows */
} fa_packet_snap_hdr;                /* 24 bytes */

/* Flow filter in front of fa_ingest_snaps: the rules of the reference's filter_map / peer_filter_map LPM tries
 * (bpf/maps_definition.h:108-127, at most 16 entries each) and the matching of bpf/flows_filter.h:14-255 +
 * check_and_do_flow_filtering (bpf/utils.h:179-222).  A rule = its LPM key (CIDR: prefix_len + address bytes, IPv4
 * rules carry their 4 address bytes first, exactly like the trie key) + filter_value_t (bpf/types.h:300-322). */
typedef struct fa_filter_rule {
    uint8_t  ip[FA_IP_LEN];          /*  0 LPM key data */
    uint32_t prefix_len;             /* 16 LPM key prefix length in bits */
    uint32_t sample;                 /* 20 != 0: becomes the packet's sampling */
    uint16_t dst_port_start, dst_port_end, dst_port1, dst_port2;   /* 24 */
    uint16_t src_port_start, src_port_end, src_port1, src_port2;   /* 32 */
    uint16_t port_start, port_end, port1, port2;                   /* 40 */
    uint16_t tcp_flags;              /* 48 compared with the packet's set_flags() value when != 0 */
    uint8_t  protocol;               /* 50 0 = any */
    uint8_t  icmp_type, icmp_code;   /* 51 */
    uint8_t  direction;              /* 53 0 ingress, 1 egress, 2 (MAX_DIRECTION) = any */
    uint8_t  action;                 /* 54 0 ACCEPT, 1 REJECT, 2 (MAX_FILTER_ACTIONS) = none */
    uint8_t  filter_drops;           /* 55 rule wants packets with a drop reason: never matches here (flows.c:194 passes 0) */
    uint8_t  do_peer_cidr_lookup;    /* 56 */
    uint8_t  pad_[7];                /* 57 */
} fa_filter_rule;                    /* 64 bytes */

typedef struct fa_filter_cidr {      /* one peer_filter_map key */
    uint8_t  ip[FA_IP_LEN];
    uint32_t prefix_len;
} fa_filter_cidr;                    /* 20 bytes */

/* Feature-stream input records: the key plus one feature sample — what the
 * reference keeps per CPU slot in aggregated_flows_dns / additional_flow_metrics
 * (bpf/maps_definition.h:24-31,64-71). */
typedef struct fa_dns_record {
    fa_flow_id     id;               /*  0 */
    fa_dns_metrics dns;              /* 40 */
} fa_dns_record;                     /* 104 bytes */

typedef struct fa_additional_record {
    fa_flow_id            id;          /*  0 */
    fa_additional_metrics additional;  /* 40 */
} fa_additional_record;              /* 72 bytes */

typedef struct fa_pkt_drop_record {
    fa_flow_id          id;            /*  0 */
    fa_pkt_drop_metrics drops;         /* 40 */
} fa_pkt_drop_record;                /* 72 bytes */

/* Compact packet event, 64 bytes (SURVEY.md §8d): what flow_monitor knows about one packet before it touches the map
 * (bpf/flows.c:176-245) minus the MAC addresses and TLS fields — id 40 + ts 8 + len 4 + flags 2 + dscp 1 + dir 1 +
 * ifindex 4 + sampling 4.  fa_ingest_events folds each event exactly like the single-packet flow record
 * new_flow = {start = end = ts, bytes = len, packets = 1, eth_protocol (0x0800 for ::ffff:a.b.c.d keys, else 0x86DD),
 * flags, dscp, sampling, if_index_first_seen, direction_first_seen, MACs = 0, everything else 0} (flows.c:228-245).
 * 2.25 x fewer bytes over PCIe than the 144-byte ring-buffer record. */
typedef struct fa_packet_event {
    fa_flow_id id;                   /*  0 */
    uint64_t mono_ts;                /* 40 pkt.current_ts */
    uint32_t len;                    /* 48 */
    uint16_t flags;                  /* 52 collapsed TCP flags (bpf/utils.h:24-51) */
    uint8_t  dscp;                   /* 54 */
    uint8_t  direction;              /* 55 */
    uint32_t if_index;               /* 56 */
    uint32_t sampling;               /* 60 */
} fa_packet_event;                   /* 64 bytes */

/* ------------------------------------------------------------- error codes */

#define FA_OK          0
#define FA_FULL        1    /* ACCOUNTER mode: the flow cache reached max_entries at
                               record `*consumed`; call fa_evict() (reason "full",
                               reference pkg/flow/account.go:85-94) and resume. */
#define FA_E_INVAL   (-22)
#define FA_E_NOMEM   (-12)
#define FA_E_CUDA    (-5)   /* CUDA runtime failure; see fa_last_error() */
#define FA_E_NODEV   (-19)  /* no usable CUDA device: the engine has NO CPU fallback */
#define FA_E_2BIG    (-7)   /* output capacity too small */
#define FA_E_CLOSED  (-9)

/* ------------------------------------------------------------------ config */

enum fa_mode {
    FA_MODE_ACCOUNTER  = 0, /* pkg/flow/account.go + pkg/model/flow_content.go:28-61 */
    FA_MODE_KERNEL_MAP = 1  /* bpf/flows.c:76-143,222-288: the map update of flow_monitor (first-seen-interface
                               de-duplication, last-writer fields, observed-interface list, full map -> ring buffer
                               or counter).  fa_ingest never returns FA_FULL in this mode; fa_evict is
                               LookupAndDeleteMap, merged with the feature folds when FA_F_ENABLE_RTT / FA_F_ENABLE_DNS are
                               set (a flow first seen through a feature sample gets its base from the first packet that
                               follows; such entries count towards max_entries, unlike in the reference where the
                               feature maps are separate).  FA_F_ENABLE_SKETCH / FA_F_NO_FULL_CUT are refused.  With
                               FA_F_NONBLOCKING_EVICT, fa_ingest* goes on while fa_evict scans the retired map, as
                               flow_monitor goes on while the evictor runs LookupAndDeleteMap. */
};

typedef struct fa_config {
    uint32_t abi_version;     /* FA_ABI_VERSION */
    int32_t  device;          /* CUDA device ordinal */
    uint32_t mode;            /* enum fa_mode */
    uint32_t flags;           /* FA_F_* */
    uint64_t max_entries;     /* CACHE_MAX_FLOWS (reference pkg/config/config.go:146): live-flow cap */
    uint64_t max_batch;       /* largest number of records staged per kernel launch (0 = default 1<<22) */
    uint32_t cms_log2_width;  /* count-min width = 2^this (0 = default 20) */
    uint32_t cms_depth;       /* count-min rows (0 = default 4, max 8) */
    uint32_t hll_precision;   /* HyperLogLog p (0 = default 14, 4..18) */
    uint32_t reserved0;
    uint64_t sketch_seed;     /* seed of the sketch hash family */
    void*    cuda_stream;     /* optional cudaStream_t to run ingest work on (NULL = engine-owned) */
} fa_config;

#define FA_F_ENABLE_RTT     0x1u  /* ENABLE_RTT            (config.go:230) */
#define FA_F_ENABLE_DNS     0x2u  /* ENABLE_DNS_TRACKING   (config.go:236) */
#define FA_F_ENABLE_SKETCH  0x4u  /* fused count-min + HyperLogLog update in fa_ingest */
#define FA_F_NO_FULL_CUT    0x8u  /* never return FA_FULL: max_entries only sizes the table (KERNEL_MAP-style caches,
                                     multi-GPU scratch / owner tables); a physically full table spills (fa_stats.spills) */
#define FA_F_ENABLE_PKT_DROP 0x20u /* ENABLE_PKT_DROPS     (config.go) : fa_ingest_pkt_drops + the drop blocks at eviction */
#define FA_F_NONBLOCKING_EVICT 0x40u /* keep a second, empty flow table: fa_evict swaps the two under the engine lock — the
                                     Accounter hands its map over and goes on with a fresh one, pkg/flow/account.go:67-68,
                                     86-87 — and scans the retired table on its own stream, so fa_ingest (another thread)
                                     never waits for the scan or the copy to the host.  ACCOUNTER mode without feature
                                     folds, or KERNEL_MAP mode with any of FA_F_ENABLE_RTT / FA_F_ENABLE_DNS /
                                     FA_F_ENABLE_PKT_DROP / FA_F_RINGBUF_FALLBACK (the map and its feature lines are
                                     swapped together; the DNS correlation table, the fallback ring and the counters are
                                     not, and max_entries counts against the new map only, as after LookupAndDeleteMap).
                                     The swapped memory doubles: KERNEL_MAP with all three feature folds keeps 560 B per
                                     slot, about 2 x 9.4 GB at 2^24 slots.  Flows keep arriving while fa_evict runs, so its
                                     `cap` must cover max_entries (plus, with feature folds, the flows first seen through
                                     a feature sample), not the live count read before the call */
#define FA_F_RINGBUF_FALLBACK 0x10u /* KERNEL_MAP mode: ENABLE_FLOWS_RINGBUF_FALLBACK (config.go:286-288): packets whose flow
                                     cannot be created because the map is full are kept as single-packet records
                                     (errno = E2BIG, bpf/flows.c:262-279) and read back with fa_read_spilled(); without
                                     it they only increment hashmap_fail_create (flows.c:285) */

typedef struct fa_stats {
    uint64_t records_ingested;    /* flow records consumed by fa_ingest          */
    uint64_t dns_ingested;
    uint64_t additional_ingested;
    uint64_t flows_evicted;       /* EvictedFlowsCounter                          */
    uint64_t evictions;           /* EvictionCounter                              */
    uint64_t live_flows;          /* FlowBufferSizeGauge("accounter-entries")     */
    uint64_t spills;              /* records that found the table physically full */
    uint64_t order_fixups;        /* flows whose order-dependent fields needed the ordered re-fold */
    uint64_t full_cuts;           /* times fa_ingest returned FA_FULL             */
    uint64_t kernel_launches;     /* CUDA kernels launched by the engine          */
    uint64_t h2d_bytes;           /* bytes copied host->device by fa_ingest*      */
    uint64_t d2h_bytes;           /* bytes copied device->host by fa_evict etc.   */
    uint64_t observed_intf_missed;/* KERNEL_MAP mode: OBSERVED_INTF_MISSED counter (flows.c:134-142) */
    uint64_t hashmap_fail_create; /* KERNEL_MAP mode: HASHMAP_FAIL_CREATE_FLOW (flows.c:285)               */
    uint64_t ringbuf_spilled;     /* KERNEL_MAP mode: single-packet records handed to the fallback ring     */
    uint64_t ringbuf_dropped;     /* ... that found the ring full ("couldn't reserve space", flows.c:270)   */
    uint64_t pkt_drops_ingested;  /* samples consumed by fa_ingest_pkt_drops */
    uint64_t snaps_ingested;      /* packet snapshots consumed by fa_ingest_snaps ...                       */
    uint64_t snaps_discarded;     /* ... of which fill_ethhdr said DISCARD (not IP, truncated IP header)    */
    uint64_t filter_accept;       /* global counter FILTER_ACCEPT  (utils.h:196-197)                        */
    uint64_t filter_reject;       /* global counter FILTER_REJECT  (utils.h:192-194), packet skipped        */
    uint64_t filter_nomatch;      /* global counter FILTER_NOMATCH (utils.h:211)                            */
    uint64_t dns_packets_ingested;/* DNS packets consumed by fa_ingest_dns_packets (K7)                     */
    uint64_t dns_queries_pending; /* len(dns_flows): queries waiting for their response                     */
    uint64_t dns_map_full;        /* queries that found dns_flows at max_entries (errno 249 = (u8)-E2BIG)   */
    uint64_t dns_queries_purged;  /* deleted by fa_purge_stale_dns                                          */
} fa_stats;

typedef struct fa_engine fa_engine;

/* ----------------------------------------------------------------- engine */

uint32_t fa_abi_version(void);
const char* fa_last_error(void);               /* thread-local description of the last failure */

/* Replaces: tracer.NewFlowFetcher's map sizing (pkg/tracer/tracer.go:157-176)
 * and flow.NewAccounter (pkg/flow/account.go:34-53). */
int  fa_create(const fa_config* cfg, fa_engine** out);
/* Replaces: FlowFetcher.Close (pkg/tracer/tracer.go:834-838). */
void fa_destroy(fa_engine* e);

/* Aggregate n 144-byte flow records (host or device pointer; detected).
 * Replaces: the per-record body of Accounter.Account (pkg/flow/account.go:82-96)
 * fed by RingBufTracer (pkg/flow/tracer_ringbuf.go:112-134), and in
 * KERNEL_MAP mode the map update of flow_monitor (bpf/flows.c:222-288).
 * Stream order == array order.  *consumed (may be NULL) receives the number of
 * records folded; it is < n only when the call returns FA_FULL. */
int fa_ingest(fa_engine* e, const void* flow_records, size_t n, size_t* consumed);

/* Same fold for n 64-byte packet events (host or device pointer): each event is expanded on the device into the
 * single-packet record described at fa_packet_event and goes through the same kernels.  A separate measurement row
 * (64 algorithmic bytes per packet); the headline stays on 144-byte records. */
int fa_ingest_events(fa_engine* e, const void* packet_events, size_t n, size_t* consumed);

/* (f4) Raw-header front end: parse n packet snapshots (host or device pointer) on the device the way flow_monitor does
 * before it touches the map — fill_ethhdr / fill_iphdr / fill_ip6hdr / fill_l4info / set_flags (bpf/utils.h:24-167) and
 * the single-packet flow of bpf/flows.c:176-245 (start = end = ts, bytes = len, packets = 1, MACs, dscp, flags,
 * sampling, if_index / direction first seen; no TLS / DNS / QUIC tracking: those read payload) — and fold the resulting
 * records like fa_ingest.  Packets the reference discards (neither IPv4 nor IPv6, IP header beyond cap_len) are
 * dropped and counted in fa_stats.snaps_discarded.  *consumed counts SNAPSHOTS (parsed or discarded); < n only with
 * FA_FULL.  The flow filter (bpf/flows_filter.h) is not part of this entry point. */
int fa_ingest_snaps(fa_engine* e, const void* snaps, size_t n, uint32_t stride, size_t* consumed);

/* Install (n_rules > 0) or remove (n_rules == 0) the flow filter applied by fa_ingest_snaps right after the header
 * parse, where flow_monitor calls check_and_do_flow_filtering (flows.c:193-195): longest-prefix match of the source
 * address in `rules`, then of the destination address, the rule's protocol / port / ICMP / TCP-flag / direction / peer-CIDR
 * conditions, ACCEPT / REJECT semantics and the three global counters exactly as in the reference; a matching rule's
 * `sample` becomes the packet's sampling.  The random 1-in-N sampling decision itself (bpf_get_prandom_u32) is NOT
 * taken here.  At most 16 rules and 16 peer CIDRs (MAX_FILTER_ENTRIES). */
int fa_set_flow_filter(fa_engine* e, const fa_filter_rule* rules, size_t n_rules, const fa_filter_cidr* peers, size_t n_peers);

/* Fold n (flow_id + additional_metrics) samples: RTT keep-max, IPsec rules.
 * Replaces: bpf/rtt_tracker.h:12-22,73-91 + AccumulateAdditional
 * (pkg/model/flow_content.go:154-177). */
int fa_ingest_additional(fa_engine* e, const void* additional_records, size_t n);

/* Fold n (flow_id + dns_metrics) samples.
 * Replaces: bpf/flows.c:145-158,291-330 + AccumulateDNS
 * (pkg/model/flow_content.go:76-96). */
int fa_ingest_dns(fa_engine* e, const void* dns_records, size_t n);

/* Fold n (flow_id + pkt_drop_metrics) samples: saturating u16 byte / packet sums, flags OR, latest non-zero cause and
 * state.  Replaces: bpf/pkt_drops.h:10-23,80-98 + AccumulateDrops (pkg/model/flow_content.go:98-117). */
int fa_ingest_pkt_drops(fa_engine* e, const void* pkt_drop_records, size_t n);

/* Lookup-and-delete every live flow (host or device output pointers).
 * Replaces: FlowFetcher.LookupAndDeleteMap (pkg/tracer/tracer.go:1063-1157)
 * and Accounter.evict's map hand-over (pkg/flow/account.go:67-68,86-87).
 * out_records: cap x 144 B.  out_dns (cap x 64 B), out_additional (cap x 32 B)
 * and out_present (cap bytes; bit0 = has DNS, bit1 = has additional) may be NULL.
 * Output order is unspecified, as in the reference (Go map iteration). */
int fa_evict(fa_engine* e, void* out_records, void* out_dns, void* out_additional,
             uint8_t* out_present, size_t cap, size_t* n_out);

/* fa_evict with every per-flow block the engine can produce (all pointers but `records` may be NULL; host or device):
 *   pkt_drops: cap x 32 B fa_pkt_drop_metrics (present bit 2);
 *   rtt_min:   cap x u64, the smallest non-zero flow_rtt of the flow's samples, 0 if none — an extension for BASELINE
 *              config 5 ("RTT min/max"); the reference keeps only the maximum (AccumulateAdditional), so this field has
 *              no reference analogue and is PARITY UNPINNED (checked against the oracle's own definition). */
typedef struct fa_evict_out {
    void*     records;               /* cap x 144 B */
    void*     dns;                   /* cap x 64 B  */
    void*     additional;            /* cap x 32 B  */
    void*     pkt_drops;             /* cap x 32 B  */
    uint64_t* rtt_min;               /* cap x 8 B   */
    uint8_t*  present;               /* cap bytes: bit0 DNS, bit1 additional, bit2 packet drops */
} fa_evict_out;
int fa_evict_ex(fa_engine* e, const fa_evict_out* out, size_t cap, size_t* n_out);

/* Top talkers of the current window: the min(k, live) live flows with the largest byte (FA_TOP_BYTES) or packet
 * (FA_TOP_PACKETS) count, ranked on the device, WITHOUT removing or changing anything (table, feature lines, counters
 * and live flow count are as before; a later eviction returns what it would have returned without the call).
 *   Metric: the field as fa_evict_ex returns it: bytes (record offset 56) or packets (offset 64; wraps mod 2^32 in
 *           ACCOUNTER mode; in KERNEL_MAP mode only packets of the first-seen interface).  Feature-only flows have 0.
 *   Order:  metric descending; ties by ascending slot hash (fmix64(key_premix(key)), DESIGN.md §4), then by ascending
 *           key bytes (memcmp over the 40 bytes).  Independent of slot position, table size, insertion order and mode.
 *   Output: the blocks of `out` as in fa_evict_ex (host or device memory; `records` required, others may be NULL),
 *           each with room for k rows; row i of every block is bit-identical to the row fa_evict_ex would return for
 *           that flow now (feature blocks and the base patch included).  A requested block the engine does not produce
 *           comes back zero.  *n_out = min(k, live); rows past it are not written.
 *   Runs on the engine stream after every queued fold, under the engine lock, and returns when the outputs are
 *   complete.  FA_F_NONBLOCKING_EVICT: ranks the live table only, not a retired table still being evicted.  The
 *   fallback ring (fa_read_spilled) is not part of the table.  Device scratch O(k), allocated on first use.
 *   FA_E_INVAL: null engine / out / out->records / n_out, unknown `by`, k == 0 or k > FA_TOP_MAX_K (nothing changes).
 *   FA_E_CUDA: also when more than 4096 live flows share the k-th flow's metric value and 64-bit key premix (keys
 *   built to collide on purpose; the table's probe chains would be as long). */
#define FA_TOP_BYTES    0u
#define FA_TOP_PACKETS  1u
#define FA_TOP_MAX_K    (1u << 20)
int fa_top_flows(fa_engine* e, uint32_t by, size_t k, const fa_evict_out* out, size_t* n_out);

/* Point lookups of the flows the caller names (bpf_map_lookup_elem for a batch of keys), on the device, WITHOUT
 * removing or changing anything (table, feature lines, counters, live flow count, sketch and DNS correlation table are
 * as before; a later eviction returns what it would have returned without the call; fa_stats changes only in
 * kernel_launches, h2d_bytes and d2h_bytes).
 *   keys:   n x 40-byte fa_flow_id, host (pageable or pinned) or device memory; device keys 8-byte aligned.  Byte 39
 *           (padding) is ignored, as on ingest.
 *   Output: the blocks of `out` as in fa_evict_ex (`records` required, others may be NULL), each in host or device memory
 *           on its own, each with room for n rows.  Row i is keys[i]: when its flow is live, row i of every block is
 *           bit-identical to the row fa_evict_ex would return for that flow now (feature blocks, rtt_min, present and the
 *           base patch of feature-only flows included); otherwise row i of every requested block is all zero.  A
 *           requested block the engine does not produce comes back zero.  Duplicate keys each get their own row.
 *   found:  n bytes (host or device; may be NULL): 1 if keys[i] is live, else 0.  *n_found = the number of found keys.
 *   Runs on the engine stream after every queued fold, under the engine lock, and returns when the outputs are
 *   complete.  Any n: the keys go through in chunks, device scratch and staging are O(chunk), allocated on first use.
 *   Not looked up: with FA_F_NONBLOCKING_EVICT a retired table still being evicted (once fa_evict returns, every key it
 *   evicted misses); the fallback ring (fa_read_spilled); DNS queries waiting for their response.
 *   n == 0: FA_OK with *n_found = 0.  FA_E_INVAL: null engine / out / out->records / n_found, null keys with n > 0,
 *   device keys not 8-byte aligned (nothing is written). */
int fa_lookup_flows(fa_engine* e, const void* keys, size_t n, const fa_evict_out* out, uint8_t* found, size_t* n_found);

/* Flow expiry on the two timers of NetFlow / IPFIX exporters, OVS and conntrack: lookup-and-delete only the live flows
 * past an idle or an active timeout, on the device; every other flow stays live (no reference analogue: the reference
 * evicts the whole window every CACHE_ACTIVE_TIMEOUT).
 *   Expires: a live flow with (idle_timeout_ns != 0 and (int64_t)(mono_now_ns - end) >= (int64_t)idle_timeout_ns) or
 *            (active_timeout_ns != 0 and (int64_t)(mono_now_ns - start) >= (int64_t)active_timeout_ns), where start and
 *            end are start_mono_time_ts / end_mono_time_ts (record offsets 40 / 48) of the row fa_evict_ex would return
 *            for it now (base patch of feature-only flows and feature effects included).  The compare is signed, as in
 *            fa_purge_stale_dns: a zero timestamp is infinitely old, a timestamp after mono_now_ns (skewed per-CPU
 *            clocks) never expires.
 *   Output: the blocks of `out` as in fa_evict_ex (`records` required, others may be NULL; host or device memory), each
 *           with room for cap rows: the expired flows' rows, bit-identical to fa_evict_ex's (feature blocks, rtt_min,
 *           present and base patch included), in unspecified order.  A requested block the engine does not produce comes
 *           back zero.  *n_out = the number of expired flows.  They are removed with their metric and feature lines; every
 *           other flow keeps every field bit for bit (its slot may move), and later folds into it go on as before.
 *   Stats:  flows_evicted += *n_out, evictions += 1, live_flows -= *n_out, kernel_launches and d2h_bytes as usual; the
 *           sketch, the DNS correlation table and the fallback ring are untouched.
 *   Runs on the engine stream after every queued fold, under the engine lock (the evictor side of the threading
 *   contract; fa_ingest* waits for it as for a blocking eviction), and returns when the outputs are complete.  Both
 *   modes; FA_F_NONBLOCKING_EVICT: expires the live table only.  ACCOUNTER mode after FA_FULL: expire instead of
 *   evicting, then resume fa_ingest at *consumed; the next cut is computed against the new live count.  Device scratch:
 *   slots / 8 bytes + 4 bytes per live flow, allocated on first use.
 *   FA_E_2BIG: more than cap flows would expire; *n_out = that count and nothing changes.
 *   FA_E_INVAL: null engine / out / out->records / n_out, both timeouts zero, a timeout above INT64_MAX (nothing changes). */
int fa_expire_flows(fa_engine* e, uint64_t mono_now_ns, uint64_t idle_timeout_ns, uint64_t active_timeout_ns,
                    const fa_evict_out* out, size_t cap, size_t* n_out);

/* One group of fa_group_flows, 88 bytes. */
typedef struct fa_flow_group {
    fa_flow_id key;                  /*  0 the group: a flow key AND key_mask (byte 39 = 0) */
    uint64_t   flows;                /* 40 live flows in the group (feature-only flows included) */
    uint64_t   bytes;                /* 48 sum of the rows' bytes (record offset 56), mod 2^64 */
    uint64_t   packets;              /* 56 sum of the rows' u32 packets (record offset 64), in 64 bits: no wrap */
    uint64_t   start_mono_time_ts;   /* 64 smallest non-zero row start; 0 if every row's start is 0 */
    uint64_t   end_mono_time_ts;     /* 72 largest row end */
    uint16_t   flags;                /* 80 OR of the rows' TCP flags (record offset 70) */
    uint8_t    pad_[6];              /* 82 always 0 */
} fa_flow_group;

/* Roll-ups of the live flows by a key mask (per subnet, per service port, per protocol, fan-out of one host, totals of
 * the window), on the device, WITHOUT removing or changing anything (no reference analogue: downstream of the agent
 * the same group-by runs on the host over evicted flows).
 *   Group:  a flow belongs to the group of its 40-byte key ANDed with key_mask (host memory, 40 bytes; byte 39 is
 *           ignored and the group key's byte 39 is 0).  IPv4 keys are ::ffff:a.b.c.d, so an IPv4 /p is a mask of 96 + p
 *           bits over the 16 address bytes.  An all-zero mask gives one group (the window's totals), an all-ones mask
 *           one group per flow.
 *   Values: "the row" of a flow is the row fa_evict_ex would return for it now, in both modes, base patch of feature-only
 *           flows included (their start and end come from the feature lines; their bytes, packets and flags are 0, and
 *           they count in `flows`).  In KERNEL_MAP mode packets and bytes are those of the first-seen interface, as that
 *           row carries them.  Sums and extremes as documented in fa_flow_group.
 *   Output: every group exactly once, in unspecified order, into `out` (host pageable / pinned or device memory; device
 *           memory 8-byte aligned), room for cap rows.  *n_groups = the number of groups.
 *   Nothing changes: the table, the feature lines, the live count, the sketch, the DNS correlation table and the
 *           fallback ring are as before, and a later eviction returns what it would have returned without the call; in
 *           fa_stats only kernel_launches and d2h_bytes move.
 *   Runs on the engine stream after every queued fold, under the engine lock, and returns when `out` is complete.
 *   FA_F_NONBLOCKING_EVICT: groups the live table only, not a retired table still being evicted.  The fallback ring
 *   (fa_read_spilled) is not part of the table.  Device scratch, allocated on first use and grown with the live count:
 *   a group table of the smallest power of two >= max(1024, 4/3 x live) slots of 96 B + 4 B (about 1.6 GB at 10^7
 *   live flows), and 88 B per group of staging for a host `out`.
 *   FA_E_2BIG: more than cap groups; *n_groups = the exact count and nothing is written to `out`.  `out` may be NULL
 *   when cap == 0: a count query.
 *   FA_E_INVAL: null engine / key_mask / n_groups, out == NULL with cap > 0, device `out` not 8-byte aligned. */
int fa_group_flows(fa_engine* e, const uint8_t key_mask[40], fa_flow_group* out, size_t cap, size_t* n_groups);

/* The per-flow value fa_histogram_flows bins, and which flows have one. */
#define FA_HIST_BYTES        0u  /* record bytes (offset 56): every flow */
#define FA_HIST_PACKETS      1u  /* record packets (offset 64, u32): every flow */
#define FA_HIST_DURATION     2u  /* end - start of the row (offsets 48 - 40), 0 if end < start: flows with start != 0 */
#define FA_HIST_RTT          3u  /* additional.flow_rtt (ns): flows whose value is != 0       (needs FA_F_ENABLE_RTT) */
#define FA_HIST_DNS_LATENCY  4u  /* dns.latency (ns): flows with a DNS block and dns.id != 0  (needs FA_F_ENABLE_DNS) */
#define FA_HIST_MAX_BOUNDS   63u
#define FA_HIST_ROW_BYTES(n_bounds) (80u + 8u * ((n_bounds) + 1u))

typedef struct fa_hist_row {     /* header of one row; n_bounds + 1 u64 bucket counts follow at offset 80 */
    fa_flow_id key;              /*  0 the group: flow key AND key_mask, byte 39 = 0 (as fa_flow_group.key) */
    uint64_t   flows;            /* 40 live flows in the group (as fa_flow_group.flows) */
    uint64_t   count;            /* 48 flows of the group that have a value (= the sum of the bucket counts) */
    uint64_t   sum;              /* 56 sum of those values, mod 2^64 */
    uint64_t   min, max;         /* 64, 72 smallest / largest value; 0 when count == 0 */
} fa_hist_row;

/* Per-group histograms of one per-flow value over the live flows (flow size, duration, RTT or DNS latency per subnet,
 * per service, per server), on the device, WITHOUT removing or changing anything (no reference analogue: downstream of
 * the agent RTT and DNS latency are published as Prometheus histograms with fixed `le` buckets).
 *   Group:  as fa_group_flows with the same key_mask: the same groups, keys and flow counts.
 *   Value:  `value` (FA_HIST_*) of the row fa_evict_ex would return for the flow now, in both modes, base patch of
 *           feature-only flows included.  A flow without the value (the decoder's presence rules: no start, a zero RTT,
 *           no DNS block or a zero DNS id, as for an IPsec-only or an errno-only sample) counts in `flows` only.
 *   Buckets: bounds (host memory) holds n_bounds Prometheus `le` upper bounds, strictly increasing, 1 <= n_bounds <=
 *           FA_HIST_MAX_BOUNDS.  Bucket 0 counts the values v <= bounds[0], bucket i < n_bounds those with
 *           bounds[i-1] < v <= bounds[i], bucket n_bounds (+Inf) those above bounds[n_bounds-1].  Per bucket, not
 *           cumulative.
 *   Output: every group exactly once, in unspecified order, into `out` (host pageable / pinned or device memory; device
 *           memory 8-byte aligned), room for cap rows of FA_HIST_ROW_BYTES(n_bounds) bytes.  *n_groups = the number of
 *           groups.
 *   Nothing changes: the table, the feature lines, the live count, the sketch, the DNS correlation table, the fallback
 *           ring and fa_group_flows' group table are as before, and a later eviction returns what it would have returned
 *           without the call; in fa_stats only kernel_launches and d2h_bytes move.
 *   Runs on the engine stream after every queued fold, under the engine lock, and returns when `out` is complete.
 *   FA_F_NONBLOCKING_EVICT: bins the live table only, not a retired table still being evicted.  The fallback ring
 *   (fa_read_spilled) is not part of the table.  Device scratch, allocated on first use and grown with the live count:
 *   fa_group_flows' group table plus 4 B per slot of it, and FA_HIST_ROW_BYTES(n_bounds) per group of staging for a
 *   host `out` (592 B at 63 bounds: an all-ones mask over 10^7 live flows stages about 5.9 GB; cap bounds it).
 *   FA_E_2BIG: more than cap groups; *n_groups = the exact count and nothing is written to `out`.  `out` may be NULL
 *   when cap == 0: a count query.
 *   FA_E_INVAL: null engine / key_mask / bounds / n_groups, out == NULL with cap > 0, device `out` not 8-byte aligned,
 *   an unknown value, n_bounds == 0 or > FA_HIST_MAX_BOUNDS, bounds not strictly increasing, FA_HIST_RTT without
 *   FA_F_ENABLE_RTT, FA_HIST_DNS_LATENCY without FA_F_ENABLE_DNS (nothing changes). */
int fa_histogram_flows(fa_engine* e, const uint8_t key_mask[40], uint32_t value, const uint64_t* bounds, uint32_t n_bounds,
                       void* out, size_t cap, size_t* n_groups);

/* One group of fa_distinct_flows, 56 bytes. */
typedef struct fa_distinct_group {
    fa_flow_id key;                  /*  0 the group: a flow key AND group_mask (byte 39 = 0), as fa_flow_group.key */
    uint64_t   flows;                /* 40 live flows in the group (feature-only flows included), as fa_flow_group.flows */
    uint64_t   distinct;             /* 48 distinct values of (flow key AND distinct_mask) among those flows, >= 1 */
} fa_distinct_group;

/* Per-group distinct counts of a second key mask over the live flows (distinct destination ports per source: a port
 * scan; distinct peers per host: fan-out; distinct clients per service: fan-in; distinct destinations of the window),
 * on the device, WITHOUT removing or changing anything (no reference analogue: downstream of the agent the same COUNT
 * DISTINCT runs on the host over evicted flows).
 *   Group:  as fa_group_flows with key_mask = group_mask: the same groups, keys and flow counts.  `distinct` counts the
 *           distinct 40-byte values key AND distinct_mask among the group's live flows.  Both masks are host memory, 40
 *           bytes; byte 39 of each is ignored.  The masks may overlap: distinct_mask within group_mask gives 1 for every
 *           group, an all-zero group_mask one row with the window's distinct count, an all-ones distinct_mask
 *           distinct == flows.  Only the keys of the rows fa_evict_ex would return matter, in both modes (feature-only
 *           flows included).
 *   Threshold: only the groups with distinct >= min_distinct are returned (0 and 1: every group), so that a scan
 *           detector is one call that returns a handful of rows.
 *   Output: every passing group exactly once, in unspecified order, into `out` (host pageable / pinned or device
 *           memory; device memory 8-byte aligned), room for cap rows.  *n_groups = the number of passing groups.
 *   Nothing changes: the table, the feature lines, the live count, the sketch, the DNS correlation table, the fallback
 *           ring and fa_group_flows' group table are as before, and a later eviction returns what it would have returned
 *           without the call; in fa_stats only kernel_launches and d2h_bytes move.
 *   Runs on the engine stream after every queued fold, under the engine lock, and returns when `out` is complete.
 *   FA_F_NONBLOCKING_EVICT: counts the live table only, not a retired table still being evicted.  The fallback ring
 *   (fa_read_spilled) is not part of the table.  Device scratch, allocated on first use and grown with the live count:
 *   fa_group_flows' group table (it holds the distinct (group, value) pairs), a second group table of the same slot
 *   layout sized from the number of those pairs, and 56 B per passing group of staging for a host `out`.
 *   FA_E_2BIG: more than cap passing groups; *n_groups = the exact count and nothing is written to `out`.  `out` may be
 *   NULL when cap == 0: a count query.
 *   FA_E_INVAL: null engine / group_mask / distinct_mask / n_groups, out == NULL with cap > 0, device `out` not 8-byte
 *   aligned (nothing changes).
 *   FA_E_CUDA: a fold found no slot in a group table (never expected; the group tables are cleared all the same). */
int fa_distinct_flows(fa_engine* e, const uint8_t group_mask[40], const uint8_t distinct_mask[40], uint64_t min_distinct,
                      fa_distinct_group* out, size_t cap, size_t* n_groups);

/* Lookup-and-RESET (no reference analogue; building block of the multi-GPU local combiner, the counterpart of
 * the reference folding its per-CPU maps in user space, pkg/tracer/tracer.go:1159-1187): every flow that received
 * records since the previous drain is written to out_records (device memory, cap x 144 B) as a partial flow record
 * and its counters are reset to the fold identity; the flows themselves stay cached.  A partial whose start is
 * already covered by an earlier partial carries start = 0 ("unset"), which AccumulateBase ignores. */
int fa_drain_active(fa_engine* e, void* out_records_dev, size_t cap, size_t* n_out);

/* Number of live flows right now (len(c.entries), account.go:98). */
int fa_live_flows(fa_engine* e, size_t* n);

/* KERNEL_MAP mode with FA_F_RINGBUF_FALLBACK.  Replaces: FlowFetcher.ReadRingBuf on `direct_flows`
 * (pkg/tracer/tracer.go:1052-1054; bpf/flows.c:262-279), batched: copies out and removes the single-packet
 * records spilled since the last call (at most 131072 are kept = the reference's 16 MiB ring,
 * bpf/maps_definition.h:7-11; later ones are dropped and counted).  out: host or device, cap records. */
int fa_read_spilled(fa_engine* e, void* out_records, size_t cap, size_t* n_out);

/* K7 — DNS query -> response correlation on the device.  Replaces: track_dns_packet and its dns_flows map
 * (bpf/dns_tracker.h:23-37,68-127; bpf/maps_definition.h:81-89, max_entries 1 << 20) together with the dns_metrics
 * sample flow_monitor derives from it (bpf/flows.c:210-213,291-330), followed by the fold of fa_ingest_dns.
 * pkts: n x 104 bytes (host or device) in stream order, laid out like fa_dns_record: id = the packet's flow id;
 * dns.end_mono_time_ts = the packet's timestamp; dns.id / dns.flags = the DNS header's id / flags in host order
 * (QR = 0x8000); dns.eth_protocol; dns.name = the raw QNAME bytes; start / latency / errno are ignored.
 *   query:    inserted if absent.  Already there -> the packet's flow gets a sample with errno 239 ((u8)-EEXIST: the
 *             reference hands bpf_map_update_elem's return value on as dns_errno) and id = flags = latency = 0;
 *             map at max_entries -> the same with errno 249 ((u8)-E2BIG; WHICH queries of a batch meet the full map is
 *             not order-exact on the device).
 *   response: the reversed tuple is looked up: found -> latency = ts - query ts and the entry is deleted, else errno 2
 *             (ENOENT); one sample {start = end = ts, id, flags, latency, eth_protocol, name, errno} unless id == 0 and
 *             errno == 0.
 * Needs FA_F_ENABLE_DNS.  Bit-exact against the sequential restatement for any interleaving of the packets of a key. */
int fa_ingest_dns_packets(fa_engine* e, const void* dns_packets, size_t n);

/* Replaces: FlowFetcher.DeleteMapsStaleEntries (pkg/tracer/tracer.go:1229-1257): deletes the queries of
 * fa_ingest_dns_packets with time.Duration(mono_now_ns - ts) >= timeout_ns (a signed compare, as in Go).  Without a
 * correlated packet stream (latency pre-computed by the caller, fa_ingest_dns) there is nothing to purge. */
int fa_purge_stale_dns(fa_engine* e, uint64_t mono_now_ns, uint64_t timeout_ns);

/* Count-min point queries for n 40-byte keys (new capability; no reference). */
int fa_cms_query(fa_engine* e, const void* keys, size_t n, uint64_t* estimates);
/* HyperLogLog distinct-flow estimate (new capability; no reference). */
int fa_hll_estimate(fa_engine* e, double* estimate);
/* Raw sketch state for exact cross-checks / multi-GPU merges:
 * cms: depth x width u64 (row-major); hll: 2^p u8 registers. Host pointers. */
int fa_sketch_export(fa_engine* e, uint64_t* cms_out, size_t cms_words, uint8_t* hll_out, size_t hll_regs);
int fa_sketch_reset(fa_engine* e);

/* ----------------------------------------------- evicted flows -> protobuf (K8) */

/* One row of the agent's interface table (ifaces.Registerer: ifindex -> {MAC -> name}, pkg/ifaces/registerer.go:153-190)
 * with the UDN label NewIntfDirUdn would attach to that interface (pkg/model/record.go:168-185; "" = none). */
typedef struct fa_iface_name {
    uint32_t if_index;
    uint8_t  mac[FA_MAC_LEN];
    uint8_t  name_len;               /* <= 16 */
    uint8_t  udn_len;                /* <= 64 */
    char     name[16];
    char     udn[64];
} fa_iface_name;                     /* 92 bytes */

#define FA_PB_WRAP_ENTRIES 0x1u      /* prefix every record with the pbflow.Records `entries` tag + length: the output (or any
                                        run of whole records of it) is then a serialized pbflow.Records (gRPC exporter,
                                        pkg/pbflow/proto.go:19-35); without it every record is one Kafka message value
                                        (pkg/exporter/kafka_proto.go:49-60) */
typedef struct fa_pb_params {
    uint64_t now_unix_ns;            /* clock() at eviction  (pkg/flow/account.go:103); wall clocks are exact in seconds +
                                        nanoseconds like time.Time.Add, also past the int64 nanosecond range */
    uint64_t mono_now_ns;            /* monoClock()          (account.go:104) */
    uint8_t  agent_ip[FA_IP_LEN];    /* agent IP in 16-byte form (IPv4: ::ffff:a.b.c.d) */
    uint32_t agent_ip_is_v4;         /* net.IP.To4() != nil */
    uint32_t flags;                  /* FA_PB_* */
    const fa_iface_name* ifaces;     /* host pointer, n_ifaces rows, copied by the call; NULL = every interface is "unknown" */
    uint32_t n_ifaces;
    uint32_t reserved;
} fa_pb_params;

/* Serialize n evicted flows (the outputs of fa_evict: records n x 144 B, and optionally dns n x 64 B, additional
 * n x 32 B, pkt_drops n x 32 B, present n bytes; host or device pointers) as pbflow.Record messages, fields in field-number order as
 * protobuf-go writes them.  Replaces, batched: model.NewRecord (pkg/model/record.go:82-159: wall-clock times, interface
 * list, DNS latency, RTT), pbflow.FlowToPB + proto.Marshal (pkg/pbflow/proto.go:39-149, proto/flow.proto:31-126) and
 * getFlowKey (pkg/exporter/kafka_proto.go:37-47).
 * out_bytes (host or device, out_cap bytes) receives the messages back to back; offsets (n + 1 u64, may be NULL) the
 * start of each; keys_out (n x 32 B, may be NULL) the Kafka keys.  *out_len = bytes needed; FA_E_2BIG if > out_cap
 * (nothing written).  Not produced (no such state in the engine): xlat, quic, network_events_metadata.
 * A feature block is used for flow i only where its pointer is given and present[i] has its bit (1 dns, 2 additional,
 * 4 pkt_drops); present NULL = no block for any flow.
 * A flow whose dns_name, interface name or UDN is not valid UTF-8 is written as zero bytes (offsets[i] ==
 * offsets[i + 1]; no Records entry with FA_PB_WRAP_ENTRIES; its key is still written): protobuf-go refuses to marshal
 * such a `string` field and the Kafka exporter drops the record (pkg/exporter/kafka_proto.go:53-57).  Any other record
 * is at least a few dozen bytes, so callers skip empty entries.  When every flow is dropped, *out_len is 0 and
 * out_bytes may be NULL. */
int fa_pb_encode(fa_engine* e, const void* records, const void* dns, const void* additional, const void* pkt_drops,
                 const uint8_t* present, size_t n, const fa_pb_params* p, void* out_bytes, size_t out_cap, uint64_t* offsets,
                 void* keys_out, size_t* out_len);

/* Replaces: ReadGlobalCounter (pkg/tracer/tracer.go:1190-1226) + the metrics the
 * hot path increments (pkg/metrics/metrics.go:66-161). */
int fa_get_stats(fa_engine* e, fa_stats* out);

/* Block until all queued engine work has finished. */
int fa_sync(fa_engine* e);

/* -------------------------------------------------- multi-GPU routing (K3) */

/* owner = fa_owner_hash(key) % n_shards; independent of the in-table probe hash. */
uint64_t fa_owner_hash(const fa_flow_id* key);

/* Partition n device-resident flow records by owner into `out` (n x 144 B,
 * grouped by shard, order within a shard preserved by source index) and write
 * the n_shards per-shard counts to counts_host.  All pointers except counts_host
 * are device pointers. */
int fa_route(fa_engine* e, const void* flow_records, size_t n, uint32_t n_shards,
             void* out, uint64_t* counts_host);

/* ---- fused routing + exchange over peer memory (one process per GPU, same box) ----
 * The owners' receive buffers and record counters are plain device allocations (fa_device_alloc) exported with
 * CUDA IPC and mapped by every peer.  fa_route_peer is K3 fused with the all-to-all: it partitions the records by
 * owner and stores them straight into the owners' buffers over NVLink, reserving room with one remote atomic per
 * CTA and shard.  Sizes never travel through the host: *_counted entry points read their record count from device
 * memory, so a whole round (combine, drain, route+exchange, owner fold) is enqueued without a host synchronisation. */
#define FA_IPC_HANDLE_BYTES 64
int fa_ipc_export(fa_engine* e, void* dev_ptr, uint8_t handle_out[FA_IPC_HANDLE_BYTES]);
int fa_ipc_open(fa_engine* e, const uint8_t handle[FA_IPC_HANDLE_BYTES], void** out);
int fa_ipc_close(fa_engine* e, void* mapped);
/* Like fa_drain_active, but asynchronous: the number of partial records lands in *n_dev_out (device memory). */
int fa_drain_active_counted(fa_engine* e, void* out_records_dev, size_t cap, uint64_t* n_dev_out);
/* Partition min(*n_dev, max_n) device-resident records (n_dev may be NULL: exactly max_n) by owner and store them
 * into peer_bufs[owner] (capacity cap records each), advancing *peer_counts[owner].  overflow_dev points at two
 * device u64: [0] += records that did not fit their receive buffer, [1] += records stored into a shard other than
 * self_shard (x 144 B = the NVLink payload). */
int fa_route_peer(fa_engine* e, const void* records_dev, const uint64_t* n_dev, size_t max_n, uint32_t n_shards,
                  uint32_t self_shard, void* const* peer_bufs, uint64_t* const* peer_counts, size_t cap, uint64_t* overflow_dev);

/* ---- the same exchange with ONE process driving all GPUs of a box (csrc/sharded.cu) ----
 * What a Go host links: fa_sharded_* own one owner engine (+ one scratch combiner) per device, their streams, peer
 * access and the double-buffered receive buffers; fa_sharded_ingest deals every host batch to the GPUs by position
 * (each slice crosses its own PCIe link), every GPU combines its slice locally, routes the partial flow records to
 * their owners over NVLink (fa_route_peer) and folds what it receives; the only synchronisation is device-side
 * (events between the N streams).  cfg: mode ACCOUNTER; max_entries = flows of the whole box; max_batch = records per
 * GPU and round (0 = 2^22); reserved0 bit 0 = route raw records (no local combiner); device / cuda_stream ignored.
 * flags: FA_F_ENABLE_RTT / _DNS / _PKT_DROP are passed to the owners (the combiners do not get them: samples bypass
 * the combiner); FA_F_ENABLE_SKETCH is refused (FA_E_INVAL).  A device id may appear more than once: several shards
 * then share one GPU (peer access is only enabled between distinct devices).
 * fa_sharded_evict == LookupAndDeleteMap over all owners (disjoint key sets, concatenated).
 * All calls take the object's lock: one thread at a time, calls of several threads are serialised. */
typedef struct fa_sharded fa_sharded;
int  fa_sharded_create(const fa_config* cfg, const int32_t* devices, uint32_t n_devices, fa_sharded** out);
void fa_sharded_destroy(fa_sharded* s);
int  fa_sharded_ingest(fa_sharded* s, const void* flow_records_host, size_t n);
/* device-resident batches: records_dev[i] (n_per_gpu[i] records) lives on devices[i] */
int  fa_sharded_ingest_device(fa_sharded* s, const void* const* records_dev, const size_t* n_per_gpu);
/* Feature samples, host memory (pageable or pinned, released before return, as fa_sharded_ingest): n (flow_id +
 * additional_metrics), (flow_id + dns_metrics) or (flow_id + pkt_drop_metrics) samples, folded on the GPU that owns their
 * flow.  A call is cut into rounds of at most N x max_batch samples; slice i of a round goes to GPU i, which routes it
 * stably (fa_route_peer_samples) into its segment of every owner's receive buffer; each owner folds the segments in
 * source order (fa_ingest_samples_counted), so every owner folds a flow's samples in stream order.
 * Exactness: for any sequence of fa_sharded_ingest / _additional / _dns / _pkt_drops calls, fa_sharded_evict_ex returns,
 * sorted by key, the rows one engine with the same flags returns for the same calls in the same order, bit for bit in the
 * dns, additional, pkt_drops, rtt_min and present blocks and in the base patch of feature-only flows, for arbitrary
 * sample values.  The 144-byte base rows themselves are exact under fa_sharded_ingest's condition (per-flow-constant
 * descriptors).  Sample and record calls share the rounds and stay ordered on every GPU.  Counted in fa_sharded_get_stats'
 * additional / dns / pkt_drops_ingested.  FA_E_INVAL: the object was created without the kind's FA_F_ENABLE_* flag,
 * null samples with n > 0, device memory (device-resident samples are not supported).  Not available: K7's
 * fa_ingest_dns_packets (a query and its response have reversed tuples, hence different owners), sketches, KERNEL_MAP. */
int  fa_sharded_ingest_additional(fa_sharded* s, const void* additional_records_host, size_t n);
int  fa_sharded_ingest_dns(fa_sharded* s, const void* dns_records_host, size_t n);
int  fa_sharded_ingest_pkt_drops(fa_sharded* s, const void* pkt_drop_records_host, size_t n);
int  fa_sharded_evict(fa_sharded* s, void* out_records_host, size_t cap, size_t* n_out);
/* fa_evict_ex over all owners: the blocks of `out` as in fa_evict_ex (host memory; `records` required when flows are
 * live, the others may be NULL), each with room for cap rows; the owners' rows are concatenated (disjoint key sets),
 * order unspecified.  The combiners' scratch tables are emptied as by fa_sharded_evict (which is this call with records
 * only).  FA_E_2BIG (nothing evicted): cap < live flows; FA_E_INVAL: null argument or records. */
int  fa_sharded_evict_ex(fa_sharded* s, const fa_evict_out* out, size_t cap, size_t* n_out);
int  fa_sharded_live_flows(fa_sharded* s, size_t* n);
int  fa_sharded_sync(fa_sharded* s);
/* sum of the owners' counters (records_ingested and the three sample counts: what was passed in); nvlink_records =
 * 144-byte records that crossed to another GPU (samples are not counted there); receive_overflow must stay 0 */
int  fa_sharded_get_stats(fa_sharded* s, fa_stats* sum, uint64_t* nvlink_records, uint64_t* receive_overflow);
const char* fa_sharded_last_error(void);
/* fa_ingest for a device-resident batch whose size (<= max_n) is only known on the device; reset_count != 0
 * zeroes *n_dev after the fold has been enqueued.  Requires FA_F_NO_FULL_CUT. */
int fa_ingest_counted(fa_engine* e, const void* records_dev, uint64_t* n_dev, size_t max_n, int reset_count);

/* ---- the exchange for feature samples (what fa_sharded_ingest_additional / _dns / _pkt_drops run on) ----
 * kind: which sample stream, as fa_ingest_additional (72 B), fa_ingest_dns (104 B) and fa_ingest_pkt_drops (72 B). */
enum fa_sample_kind { FA_SAMPLES_ADDITIONAL = 0, FA_SAMPLES_DNS = 1, FA_SAMPLES_PKT_DROPS = 2 };

/* Route min(*n_dev, max_n) device-resident samples of `kind` (n_dev may be NULL: exactly max_n) to their owners, STABLY:
 * the samples bound for owner o = fa_owner_hash(key) % n_shards (the owner of the flow's base records) are stored into
 * peer_segs[o], this source's segment of o's receive buffer, in the order they have in `samples_dev`, and their number
 * is stored (not added) into *peer_seg_counts[o].  Each segment holds seg_cap samples; seg_cap >= max_n cannot
 * overflow.  A sample past the end is not stored and adds 1 to overflow_dev[0] (as does *n_dev - max_n when *n_dev >
 * max_n); overflow_dev[1] is not touched (fa_route_peer counts 144-byte rows there).  Three kernels on the engine's
 * stream, no host synchronisation; the engine's flags do not matter.  Samples and segments 8-byte aligned, device (or
 * peer-mapped) memory.  FA_E_INVAL: null argument, kind, n_shards not 1..16 or self_shard >= n_shards, alignment. */
int fa_route_peer_samples(fa_engine* e, uint32_t kind, const void* samples_dev, const uint64_t* n_dev, size_t max_n, uint32_t n_shards,
                          uint32_t self_shard, void* const* peer_segs, uint64_t* const* peer_seg_counts, size_t seg_cap, uint64_t* overflow_dev);

/* Fold min(*n_dev, max_n) device-resident samples of `kind` whose count lives in device memory (one segment of a receive
 * buffer), as fa_ingest_additional / _dns / _pkt_drops would fold them: the samples get the engine's next max_n sample
 * numbers, so segments folded one after the other are folded in that order, bit-exactly (the unused numbers of a short
 * segment are a gap; only the relative order of a flow's samples matters).  reset_count != 0 zeroes *n_dev after the fold
 * has been enqueued.  Asynchronous on the engine's stream; the samples must stay valid until it has run.  Not counted in
 * fa_stats' additional / dns / pkt_drops_ingested (the count is not known on the host).  A sample whose flow cannot be
 * created counts in `spills`; there is no room check.  FA_E_INVAL: null argument, kind, engine without the kind's
 * FA_F_ENABLE_* flag or without FA_F_NO_FULL_CUT, KERNEL_MAP mode, max_n not 1..max_batch, samples not 8-byte aligned. */
int fa_ingest_samples_counted(fa_engine* e, uint32_t kind, const void* samples_dev, uint64_t* n_dev, size_t max_n, int reset_count);

/* ------------------------------------------- memory + synthetic generator */

int fa_device_alloc(fa_engine* e, size_t bytes, void** out);
int fa_device_free(fa_engine* e, void* p);
int fa_host_alloc(size_t bytes, void** out);   /* pinned host memory */
int fa_host_free(void* p);

enum fa_gen_dist { FA_GEN_UNIFORM = 0, FA_GEN_ZIPF = 1 };

/* Counter-based synthetic stream (SURVEY.md §8d): record i depends only on
 * (seed, first_index + i), so any slice can be generated anywhere. */
typedef struct fa_gen_params {
    uint64_t seed;
    uint64_t n_keys;          /* distinct 5-tuples (<= 2^32) */
    uint32_t dist;            /* enum fa_gen_dist */
    uint32_t zipf_s_milli;    /* Zipf exponent x 1000 (e.g. 1100) */
    uint64_t t0_ns;           /* ts(i) = t0_ns + i: strictly monotone */
    uint32_t varying_desc;    /* 0: per-key-constant MAC/ifindex/dscp/... ; 1: per-record random (order-dependent fields exercised) */
    uint32_t reserved;
} fa_gen_params;

/* dst may be a host or a device pointer (host generation runs on the CPU and is
 * bit-identical to the device generator). */
int fa_gen_records(fa_engine* e, const fa_gen_params* p, uint64_t first_index, size_t n, void* dst);
/* The 40-byte key of rank r (0-based) of the generator's key universe. Host pointer. */
int fa_gen_key(const fa_gen_params* p, uint64_t rank, fa_flow_id* out);

#ifdef __cplusplus
}
#endif
#endif /* FLOWAGG_H */
