"""ctypes binding of libflowagg.so — every symbol include/flowagg.h declares."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REC_BYTES, ID_BYTES, DNS_BYTES, ADD_BYTES, DNSREC_BYTES, ADDREC_BYTES = 144, 40, 64, 32, 104, 72

FA_OK, FA_FULL = 0, 1
FA_E_INVAL, FA_E_NOMEM, FA_E_CUDA, FA_E_NODEV, FA_E_2BIG, FA_E_CLOSED = -22, -12, -5, -19, -7, -9
FA_MODE_ACCOUNTER, FA_MODE_KERNEL_MAP = 0, 1
FA_F_ENABLE_RTT, FA_F_ENABLE_DNS, FA_F_ENABLE_SKETCH, FA_F_NO_FULL_CUT, FA_F_RINGBUF_FALLBACK, FA_F_ENABLE_PKT_DROP = 1, 2, 4, 8, 16, 32
FA_F_NONBLOCKING_EVICT = 64
FA_TOP_BYTES, FA_TOP_PACKETS, FA_TOP_MAX_K = 0, 1, 1 << 20
FA_HIST_BYTES, FA_HIST_PACKETS, FA_HIST_DURATION, FA_HIST_RTT, FA_HIST_DNS_LATENCY = 0, 1, 2, 3, 4
FA_HIST_MAX_BOUNDS = 63
FA_GEN_UNIFORM, FA_GEN_ZIPF = 0, 1
FA_SAMPLES_ADDITIONAL, FA_SAMPLES_DNS, FA_SAMPLES_PKT_DROPS = 0, 1, 2
FA_ABI_VERSION = 1


class FlowAggError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"flowagg error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("device", C.c_int32), ("mode", C.c_uint32), ("flags", C.c_uint32),
                ("max_entries", C.c_uint64), ("max_batch", C.c_uint64),
                ("cms_log2_width", C.c_uint32), ("cms_depth", C.c_uint32), ("hll_precision", C.c_uint32),
                ("reserved0", C.c_uint32), ("sketch_seed", C.c_uint64), ("cuda_stream", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "records_ingested", "dns_ingested", "additional_ingested", "flows_evicted", "evictions", "live_flows",
        "spills", "order_fixups", "full_cuts", "kernel_launches", "h2d_bytes", "d2h_bytes",
        "observed_intf_missed", "hashmap_fail_create", "ringbuf_spilled", "ringbuf_dropped", "pkt_drops_ingested",
        "snaps_ingested", "snaps_discarded", "filter_accept", "filter_reject", "filter_nomatch",
        "dns_packets_ingested", "dns_queries_pending", "dns_map_full", "dns_queries_purged")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_ if n != "reserved"}


class EvictOut(C.Structure):
    _fields_ = [("records", C.c_void_p), ("dns", C.c_void_p), ("additional", C.c_void_p), ("pkt_drops", C.c_void_p),
                ("rtt_min", C.c_void_p), ("present", C.c_void_p)]


class IfaceName(C.Structure):
    _fields_ = [("if_index", C.c_uint32), ("mac", C.c_uint8 * 6), ("name_len", C.c_uint8), ("udn_len", C.c_uint8),
                ("name", C.c_char * 16), ("udn", C.c_char * 64)]


class PbParams(C.Structure):
    _fields_ = [("now_unix_ns", C.c_uint64), ("mono_now_ns", C.c_uint64), ("agent_ip", C.c_uint8 * 16),
                ("agent_ip_is_v4", C.c_uint32), ("flags", C.c_uint32), ("ifaces", C.POINTER(IfaceName)),
                ("n_ifaces", C.c_uint32), ("reserved", C.c_uint32)]


FA_PB_WRAP_ENTRIES = 1

# fa_flow_group (88 bytes), include/flowagg.h
GROUP_DTYPE = np.dtype([("key", "u1", 40), ("flows", "<u8"), ("bytes", "<u8"), ("packets", "<u8"),
                        ("start_mono_time_ts", "<u8"), ("end_mono_time_ts", "<u8"), ("flags", "<u2"), ("pad_", "u1", 6)])
assert GROUP_DTYPE.itemsize == 88

# fa_distinct_group (56 bytes), include/flowagg.h
DISTINCT_DTYPE = np.dtype([("key", "u1", 40), ("flows", "<u8"), ("distinct", "<u8")])
assert DISTINCT_DTYPE.itemsize == 56


def hist_dtype(n_bounds):
    """One row of fa_histogram_flows with n_bounds bounds: fa_hist_row, then n_bounds + 1 bucket counts
    (FA_HIST_ROW_BYTES(n_bounds) bytes), include/flowagg.h."""
    assert 1 <= n_bounds <= FA_HIST_MAX_BOUNDS, n_bounds
    return np.dtype([("key", "u1", 40), ("flows", "<u8"), ("count", "<u8"), ("sum", "<u8"), ("min", "<u8"),
                     ("max", "<u8"), ("counts", "<u8", (n_bounds + 1,))])


class GenParams(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_keys", C.c_uint64), ("dist", C.c_uint32), ("zipf_s_milli", C.c_uint32),
                ("t0_ns", C.c_uint64), ("varying_desc", C.c_uint32), ("reserved", C.c_uint32)]


# name -> (restype, argtypes): exactly the entry points of include/flowagg.h
SIGNATURES = {
    "fa_abi_version": (C.c_uint32, []),
    "fa_last_error": (C.c_char_p, []),
    "fa_create": (C.c_int, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    "fa_destroy": (None, [C.c_void_p]),
    "fa_ingest": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_ingest_events": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_ingest_snaps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.POINTER(C.c_size_t)]),
    "fa_set_flow_filter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "fa_ingest_additional": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_ingest_dns": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_ingest_dns_packets": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_ingest_pkt_drops": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_evict_ex": (C.c_int, [C.c_void_p, C.POINTER(EvictOut), C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_top_flows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_size_t, C.POINTER(EvictOut), C.POINTER(C.c_size_t)]),
    "fa_lookup_flows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(EvictOut), C.c_void_p,
                                  C.POINTER(C.c_size_t)]),
    "fa_expire_flows": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(EvictOut), C.c_size_t,
                                  C.POINTER(C.c_size_t)]),
    "fa_group_flows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_histogram_flows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t,
                                     C.POINTER(C.c_size_t)]),
    "fa_distinct_flows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t,
                                    C.POINTER(C.c_size_t)]),
    "fa_evict": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                           C.POINTER(C.c_size_t)]),
    "fa_drain_active": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_drain_active_counted": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "fa_route_peer": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p),
                                C.POINTER(C.c_void_p), C.c_size_t, C.c_void_p]),
    "fa_sharded_create": (C.c_int, [C.POINTER(Config), C.POINTER(C.c_int32), C.c_uint32, C.POINTER(C.c_void_p)]),
    "fa_sharded_destroy": (None, [C.c_void_p]),
    "fa_sharded_ingest": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_sharded_ingest_device": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]),
    "fa_sharded_ingest_additional": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_sharded_ingest_dns": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_sharded_ingest_pkt_drops": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fa_sharded_evict": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_sharded_evict_ex": (C.c_int, [C.c_void_p, C.POINTER(EvictOut), C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_sharded_live_flows": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "fa_sharded_sync": (C.c_int, [C.c_void_p]),
    "fa_sharded_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "fa_sharded_last_error": (C.c_char_p, []),
    "fa_ingest_counted": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "fa_route_peer_samples": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                        C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_size_t, C.c_void_p]),
    "fa_ingest_samples_counted": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "fa_ipc_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fa_ipc_open": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "fa_ipc_close": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fa_live_flows": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "fa_read_spilled": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fa_purge_stale_dns": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64]),
    "fa_cms_query": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "fa_hll_estimate": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "fa_sketch_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "fa_sketch_reset": (C.c_int, [C.c_void_p]),
    "fa_pb_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(PbParams),
                               C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)]),
    "fa_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "fa_sync": (C.c_int, [C.c_void_p]),
    "fa_owner_hash": (C.c_uint64, [C.c_void_p]),
    "fa_route": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p]),
    "fa_device_alloc": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    "fa_device_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fa_host_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "fa_host_free": (C.c_int, [C.c_void_p]),
    "fa_gen_records": (C.c_int, [C.c_void_p, C.POINTER(GenParams), C.c_uint64, C.c_size_t, C.c_void_p]),
    "fa_gen_key": (C.c_int, [C.POINTER(GenParams), C.c_uint64, C.c_void_p]),
}

_lib = None


def lib_path():
    # FA_LIB_NAME: load an alternative build of the same ABI (A/B experiments only)
    return os.path.join(HERE, os.environ.get("FA_LIB_NAME", "libflowagg.so"))


def lib():
    """Load libflowagg.so (built in-tree by __graft_entry__.build()). Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise FlowAggError(FA_E_NODEV, f"{p} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                        "(there is no CPU fallback)")
    L = C.CDLL(p)
    alt = "FA_LIB_NAME" in os.environ  # an older build kept for a same-box A/B may lack the newest entry points
    for name, (res, args) in SIGNATURES.items():
        if alt and not hasattr(L, name):
            continue
        f = getattr(L, name)          # AttributeError if the .so does not export a declared symbol
        f.restype, f.argtypes = res, args
    _lib = L
    return L


def check(code):
    if code < 0:
        raise FlowAggError(code, lib().fa_last_error().decode(errors="replace"))
    return code
