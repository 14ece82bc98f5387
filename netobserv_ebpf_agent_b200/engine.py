"""FlowAggEngine — thin object wrapper over the C ABI (include/flowagg.h)."""
import ctypes as C

import numpy as np

from ._lib import (FA_ABI_VERSION, FA_FULL, FA_GEN_UNIFORM, FA_MODE_ACCOUNTER, REC_BYTES, Config, FlowAggError,  # noqa: F401
                   GenParams, Stats, check, lib)


def _ptr(x):
    """Pointer of a numpy array / torch tensor / int address."""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        assert x.flags["C_CONTIGUOUS"]
        return C.c_void_p(x.ctypes.data)
    if hasattr(x, "data_ptr"):          # torch tensor (host or device)
        assert x.is_contiguous()
        return C.c_void_p(x.data_ptr())
    raise TypeError(type(x))


def _nbytes(x):
    if isinstance(x, np.ndarray):
        return x.nbytes
    return x.numel() * x.element_size()


# fa_filter_rule (64 bytes) / fa_filter_cidr (20 bytes), include/flowagg.h
FILTER_RULE_DTYPE = np.dtype([("ip", "u1", 16), ("prefix_len", "<u4"), ("sample", "<u4"),
                              ("dst_port_start", "<u2"), ("dst_port_end", "<u2"), ("dst_port1", "<u2"), ("dst_port2", "<u2"),
                              ("src_port_start", "<u2"), ("src_port_end", "<u2"), ("src_port1", "<u2"), ("src_port2", "<u2"),
                              ("port_start", "<u2"), ("port_end", "<u2"), ("port1", "<u2"), ("port2", "<u2"), ("tcp_flags", "<u2"),
                              ("protocol", "u1"), ("icmp_type", "u1"), ("icmp_code", "u1"), ("direction", "u1"), ("action", "u1"),
                              ("filter_drops", "u1"), ("do_peer_cidr_lookup", "u1"), ("pad", "u1", 7)])
FILTER_CIDR_DTYPE = np.dtype([("ip", "u1", 16), ("prefix_len", "<u4")])
assert FILTER_RULE_DTYPE.itemsize == 64 and FILTER_CIDR_DTYPE.itemsize == 20


def _prefix_bytes(bits):
    """The 16 mask bytes of a prefix of `bits` bits (0..128) over a 16-byte address field."""
    assert 0 <= bits <= 128, bits
    m = np.zeros(16, np.uint8)
    m[: bits // 8] = 0xFF
    if bits % 8:
        m[bits // 8] = (0xFF00 >> (bits % 8)) & 0xFF
    return m


def group_mask(src_prefix=0, dst_prefix=0, src_port=False, dst_port=False, proto=False, icmp=False):
    """The 40-byte key mask of FlowAggEngine.group_flows / fa_group_flows: the first src_prefix / dst_prefix bits of the
    16-byte addresses (IPv4 keys are ::ffff:a.b.c.d, so an IPv4 /24 is 96 + 24 = 120), the ports, the transport
    protocol, the ICMP type and code."""
    m = np.zeros(40, np.uint8)
    m[0:16], m[16:32] = _prefix_bytes(src_prefix), _prefix_bytes(dst_prefix)
    if src_port:
        m[32:34] = 0xFF
    if dst_port:
        m[34:36] = 0xFF
    if proto:
        m[36] = 0xFF
    if icmp:
        m[37:39] = 0xFF
    return m


class FlowAggEngine:
    """One engine == one GPU flow cache (the reference's aggregated_flows map + Accounter)."""

    def __init__(self, max_entries, device=0, mode=FA_MODE_ACCOUNTER, flags=0, max_batch=0, cms_log2_width=0,
                 cms_depth=0, hll_precision=0, sketch_seed=0, cuda_stream=None):
        cfg = Config(abi_version=FA_ABI_VERSION, device=device, mode=mode, flags=flags, max_entries=max_entries,
                     max_batch=max_batch, cms_log2_width=cms_log2_width, cms_depth=cms_depth,
                     hll_precision=hll_precision, sketch_seed=sketch_seed, cuda_stream=cuda_stream)
        self._h = C.c_void_p()
        check(lib().fa_create(C.byref(cfg), C.byref(self._h)))
        self.max_entries = max_entries

    # -- ingest -----------------------------------------------------------------
    def ingest(self, recs, n=None):
        """Fold records (numpy host array, torch host/device tensor, or raw address with n).
        Returns (status, consumed): status is FA_OK or FA_FULL."""
        if n is None:
            nb = _nbytes(recs)
            assert nb % REC_BYTES == 0
            n = nb // REC_BYTES
        consumed = C.c_size_t(0)
        rc = check(lib().fa_ingest(self._h, _ptr(recs), n, C.byref(consumed)))
        return rc, consumed.value

    def ingest_events(self, events, n=None):
        """Fold 64-byte packet events (fa_packet_event; numpy / torch / raw address with n). Returns (status, consumed)."""
        if n is None:
            nb = _nbytes(events)
            assert nb % 64 == 0
            n = nb // 64
        consumed = C.c_size_t(0)
        rc = check(lib().fa_ingest_events(self._h, _ptr(events), n, C.byref(consumed)))
        return rc, consumed.value

    def ingest_snaps(self, snaps, stride, n=None):
        """(f4) Fold raw packet snapshots (24-byte fa_packet_snap_hdr + frame bytes, `stride` bytes apart): parsed on the
        device like flow_monitor's fill_ethhdr & co.  Returns (status, snapshots consumed)."""
        if n is None:
            nb = _nbytes(snaps)
            assert nb % stride == 0
            n = nb // stride
        consumed = C.c_size_t(0)
        rc = check(lib().fa_ingest_snaps(self._h, _ptr(snaps), n, stride, C.byref(consumed)))
        return rc, consumed.value

    def set_flow_filter(self, rules=None, peers=None):
        """Install the flow filter fa_ingest_snaps applies after the header parse (numpy arrays of FILTER_RULE_DTYPE /
        FILTER_CIDR_DTYPE = fa_filter_rule / fa_filter_cidr); no rules = no filter."""
        r = np.ascontiguousarray(rules if rules is not None else np.zeros(0, dtype=FILTER_RULE_DTYPE))
        p = np.ascontiguousarray(peers if peers is not None else np.zeros(0, dtype=FILTER_CIDR_DTYPE))
        assert r.dtype == FILTER_RULE_DTYPE and p.dtype == FILTER_CIDR_DTYPE
        check(lib().fa_set_flow_filter(self._h, r.ctypes.data if len(r) else None, len(r), p.ctypes.data if len(p) else None, len(p)))

    def ingest_all(self, recs, on_full):
        """Accounter loop: fold everything, calling on_full(evicted_records) at each "full" cut
        (reference pkg/flow/account.go:85-94)."""
        buf = np.ascontiguousarray(recs).view(np.uint8).reshape(-1)
        n = buf.size // REC_BYTES
        done = 0
        while done < n:
            rc, took = self.ingest(buf[done * REC_BYTES:])
            done += took
            if rc == FA_FULL:
                on_full(self.evict())

    def ingest_dns(self, recs):
        nb = _nbytes(recs)
        check(lib().fa_ingest_dns(self._h, _ptr(recs), nb // 104))

    def ingest_dns_packets(self, pkts):
        """K7: raw DNS packets (104 bytes each: flow id + timestamp, DNS id / flags, QNAME) in stream order; queries and
        responses are correlated on the device (bpf/dns_tracker.h:68-127) and the resulting samples folded like ingest_dns."""
        nb = _nbytes(pkts)
        check(lib().fa_ingest_dns_packets(self._h, _ptr(pkts), nb // 104))

    def purge_stale_dns(self, mono_now_ns, timeout_ns):
        """DeleteMapsStaleEntries (pkg/tracer/tracer.go:1229-1257) for the queries of ingest_dns_packets."""
        check(lib().fa_purge_stale_dns(self._h, mono_now_ns, timeout_ns))

    def ingest_additional(self, recs):
        nb = _nbytes(recs)
        check(lib().fa_ingest_additional(self._h, _ptr(recs), nb // 72))

    def ingest_pkt_drops(self, recs):
        nb = _nbytes(recs)
        check(lib().fa_ingest_pkt_drops(self._h, _ptr(recs), nb // 72))

    # -- evict ------------------------------------------------------------------
    def live_flows(self):
        n = C.c_size_t(0)
        check(lib().fa_live_flows(self._h, C.byref(n)))
        return n.value

    def evict(self, features=False, cap=None):
        """Lookup-and-delete all flows -> (n,144) uint8 array [, dns (n,64), additional (n,32), present (n,)].
        cap: output capacity in flows (default: the live count right now; pass max_entries when another thread keeps
        ingesting, FA_F_NONBLOCKING_EVICT)."""
        if cap is None:
            cap = max(self.live_flows(), 1)
        out = np.zeros((cap, REC_BYTES), dtype=np.uint8)
        got = C.c_size_t(0)
        if features:
            dns = np.zeros((cap, 64), dtype=np.uint8)
            add = np.zeros((cap, 32), dtype=np.uint8)
            pres = np.zeros(cap, dtype=np.uint8)
            check(lib().fa_evict(self._h, _ptr(out), _ptr(dns), _ptr(add), _ptr(pres), cap, C.byref(got)))
            g = got.value
            return out[:g], dns[:g], add[:g], pres[:g]
        check(lib().fa_evict(self._h, _ptr(out), None, None, None, cap, C.byref(got)))
        return out[: got.value]

    def evict_ex(self, cap=None):
        """Lookup-and-delete all flows with every block -> records (n,144), dns (n,64), additional (n,32),
        pkt_drops (n,32), rtt_min (n,) u64, present (n,).
        cap: output capacity in flows (default: the live count right now; pass max_entries when another thread keeps
        ingesting, FA_F_NONBLOCKING_EVICT)."""
        from ._lib import EvictOut
        if cap is None:
            cap = max(self.live_flows(), 1)
        out, dns, add = np.zeros((cap, REC_BYTES), np.uint8), np.zeros((cap, 64), np.uint8), np.zeros((cap, 32), np.uint8)
        drops, rmin, pres = np.zeros((cap, 32), np.uint8), np.zeros(cap, np.uint64), np.zeros(cap, np.uint8)
        o = EvictOut(records=out.ctypes.data, dns=dns.ctypes.data, additional=add.ctypes.data, pkt_drops=drops.ctypes.data,
                     rtt_min=rmin.ctypes.data, present=pres.ctypes.data)
        got = C.c_size_t(0)
        check(lib().fa_evict_ex(self._h, C.byref(o), cap, C.byref(got)))
        g = got.value
        return out[:g], dns[:g], add[:g], drops[:g], rmin[:g], pres[:g]

    def top_flows(self, k, by="bytes"):
        """The min(k, live) live flows with the most bytes (by="bytes") or packets (by="packets"), ranked, without
        removing or changing anything -> the six arrays of evict_ex (records, dns, additional, pkt_drops, rtt_min,
        present), each with min(k, live) rows.  Ties: ascending slot hash, then ascending key bytes."""
        from ._lib import FA_TOP_BYTES, FA_TOP_PACKETS, EvictOut
        metric = {"bytes": FA_TOP_BYTES, "packets": FA_TOP_PACKETS}[by]
        rows = max(int(k), 1)
        out, dns, add = np.zeros((rows, REC_BYTES), np.uint8), np.zeros((rows, 64), np.uint8), np.zeros((rows, 32), np.uint8)
        drops, rmin, pres = np.zeros((rows, 32), np.uint8), np.zeros(rows, np.uint64), np.zeros(rows, np.uint8)
        o = EvictOut(records=out.ctypes.data, dns=dns.ctypes.data, additional=add.ctypes.data, pkt_drops=drops.ctypes.data,
                     rtt_min=rmin.ctypes.data, present=pres.ctypes.data)
        got = C.c_size_t(0)
        check(lib().fa_top_flows(self._h, metric, int(k), C.byref(o), C.byref(got)))
        g = got.value
        return out[:g], dns[:g], add[:g], drops[:g], rmin[:g], pres[:g]

    def lookup_flows(self, keys):
        """Exact point lookups of live flows, without removing or changing anything: keys, (m, 40) uint8 flow ids in
        host memory -> the six arrays of evict_ex (records, dns, additional, pkt_drops, rtt_min, present) and found
        (m,) uint8, each with m rows.  Row i is keys[i]; its rows are all zero where found[i] == 0."""
        from ._lib import ID_BYTES, EvictOut
        k = np.ascontiguousarray(keys, dtype=np.uint8).reshape(-1, ID_BYTES)
        m = len(k)
        rows = max(m, 1)
        out, dns, add = np.zeros((rows, REC_BYTES), np.uint8), np.zeros((rows, 64), np.uint8), np.zeros((rows, 32), np.uint8)
        drops, rmin, pres = np.zeros((rows, 32), np.uint8), np.zeros(rows, np.uint64), np.zeros(rows, np.uint8)
        found = np.zeros(rows, np.uint8)
        o = EvictOut(records=out.ctypes.data, dns=dns.ctypes.data, additional=add.ctypes.data, pkt_drops=drops.ctypes.data,
                     rtt_min=rmin.ctypes.data, present=pres.ctypes.data)
        got = C.c_size_t(0)
        check(lib().fa_lookup_flows(self._h, k.ctypes.data, m, C.byref(o), found.ctypes.data, C.byref(got)))
        return out[:m], dns[:m], add[:m], drops[:m], rmin[:m], pres[:m], found[:m]

    def expire_flows(self, mono_now_ns, idle_timeout_ns=0, active_timeout_ns=0, cap=None):
        """Lookup-and-delete only the flows past the idle timeout (no record for idle_timeout_ns) or the active timeout
        (open for active_timeout_ns), 0 = that timer is off; every other flow stays live -> the six arrays of evict_ex
        (records, dns, additional, pkt_drops, rtt_min, present) for the expired flows.
        cap: output capacity in flows (default: the live count right now)."""
        from ._lib import EvictOut
        if cap is None:
            cap = max(self.live_flows(), 1)
        out, dns, add = np.zeros((cap, REC_BYTES), np.uint8), np.zeros((cap, 64), np.uint8), np.zeros((cap, 32), np.uint8)
        drops, rmin, pres = np.zeros((cap, 32), np.uint8), np.zeros(cap, np.uint64), np.zeros(cap, np.uint8)
        o = EvictOut(records=out.ctypes.data, dns=dns.ctypes.data, additional=add.ctypes.data, pkt_drops=drops.ctypes.data,
                     rtt_min=rmin.ctypes.data, present=pres.ctypes.data)
        got = C.c_size_t(0)
        check(lib().fa_expire_flows(self._h, int(mono_now_ns), int(idle_timeout_ns), int(active_timeout_ns), C.byref(o), cap,
                                    C.byref(got)))
        g = got.value
        return out[:g], dns[:g], add[:g], drops[:g], rmin[:g], pres[:g]

    def group_flows(self, mask, cap=None):
        """Roll the live flows up by a 40-byte key mask (group_mask) without changing anything -> a GROUP_DTYPE array,
        one row per group, in unspecified order.  cap: room in groups (default: the live count right now)."""
        from ._lib import GROUP_DTYPE
        m = np.ascontiguousarray(mask, dtype=np.uint8).reshape(-1)
        assert m.size == 40, m.size
        if cap is None:
            cap = max(self.live_flows(), 1)
        out = np.zeros(cap, GROUP_DTYPE)
        got = C.c_size_t(0)
        check(lib().fa_group_flows(self._h, m.ctypes.data, out.ctypes.data, cap, C.byref(got)))
        return out[: got.value]

    def histogram_flows(self, mask, value, bounds, cap=None):
        """Per-group histograms of one per-flow value (FA_HIST_*) over the live flows, grouped by a 40-byte key mask
        (group_mask), without changing anything -> a hist_dtype(len(bounds)) array, one row per group, in unspecified
        order.  bounds: the Prometheus `le` upper bounds, strictly increasing (counts are per bucket, the last bucket is
        +Inf).  cap: room in groups (default: the live count right now)."""
        from ._lib import FA_HIST_MAX_BOUNDS, hist_dtype
        m = np.ascontiguousarray(mask, dtype=np.uint8).reshape(-1)
        assert m.size == 40, m.size
        b = np.ascontiguousarray(bounds, dtype=np.uint64).reshape(-1)
        if cap is None:
            cap = max(self.live_flows(), 1)
        out = np.zeros(cap, hist_dtype(min(max(b.size, 1), FA_HIST_MAX_BOUNDS)))     # other sizes: FA_E_INVAL below
        got = C.c_size_t(0)
        check(lib().fa_histogram_flows(self._h, m.ctypes.data, value, b.ctypes.data, b.size, out.ctypes.data, cap,
                                       C.byref(got)))
        return out[: got.value]

    def distinct_flows(self, group_mask, distinct_mask, min_distinct=0, cap=None):
        """Per-group distinct counts over the live flows, without changing anything -> a DISTINCT_DTYPE array, one row
        per group of the 40-byte key mask group_mask (as group_flows) with at least min_distinct distinct values of
        key & distinct_mask (both masks from group_mask()), in unspecified order.  cap: room in groups (default: the live
        count right now)."""
        from ._lib import DISTINCT_DTYPE
        g = np.ascontiguousarray(group_mask, dtype=np.uint8).reshape(-1)
        d = np.ascontiguousarray(distinct_mask, dtype=np.uint8).reshape(-1)
        assert g.size == 40 and d.size == 40, (g.size, d.size)
        if cap is None:
            cap = max(self.live_flows(), 1)
        out = np.zeros(cap, DISTINCT_DTYPE)
        got = C.c_size_t(0)
        check(lib().fa_distinct_flows(self._h, g.ctypes.data, d.ctypes.data, int(min_distinct), out.ctypes.data, cap,
                                      C.byref(got)))
        return out[: got.value]

    def read_spilled(self, cap=131072):
        """KERNEL_MAP mode with FA_F_RINGBUF_FALLBACK: the single-packet records that could not enter the full map
        (the batched equivalent of reading the direct_flows ring buffer) -> (n,144) uint8 array."""
        out = np.zeros((max(cap, 1), REC_BYTES), dtype=np.uint8)
        got = C.c_size_t(0)
        check(lib().fa_read_spilled(self._h, _ptr(out), cap, C.byref(got)))
        return out[: got.value]

    def evict_into(self, out, cap):
        """Evict into a caller buffer (host or device address / tensor). Returns flow count."""
        got = C.c_size_t(0)
        check(lib().fa_evict(self._h, _ptr(out), None, None, None, cap, C.byref(got)))
        return got.value

    def drain_active(self, out_dev, cap):
        """Emit + reset the flows touched since the last drain into a device buffer (flows stay cached)."""
        got = C.c_size_t(0)
        check(lib().fa_drain_active(self._h, _ptr(out_dev), cap, C.byref(got)))
        return got.value

    # -- sketches ---------------------------------------------------------------
    def cms_query(self, keys):
        k = np.ascontiguousarray(keys).view(np.uint8).reshape(-1, 40)
        est = np.zeros(len(k), dtype=np.uint64)
        check(lib().fa_cms_query(self._h, _ptr(k), len(k), _ptr(est)))
        return est

    def hll_estimate(self):
        d = C.c_double(0)
        check(lib().fa_hll_estimate(self._h, C.byref(d)))
        return d.value

    def sketch_export(self, log2w, depth, p):
        cms = np.zeros(depth << log2w, dtype=np.uint64)
        hll = np.zeros(1 << p, dtype=np.uint8)
        check(lib().fa_sketch_export(self._h, _ptr(cms), cms.size, _ptr(hll), hll.size))
        return cms.reshape(depth, 1 << log2w), hll

    def sketch_reset(self):
        check(lib().fa_sketch_reset(self._h))

    # -- misc -------------------------------------------------------------------
    def stats(self):
        s = Stats()
        check(lib().fa_get_stats(self._h, C.byref(s)))
        return s.as_dict()

    def sync(self):
        check(lib().fa_sync(self._h))

    def route(self, recs_dev, n, n_shards, out_dev):
        counts = np.zeros(n_shards, dtype=np.uint64)
        check(lib().fa_route(self._h, _ptr(recs_dev), n, n_shards, _ptr(out_dev), _ptr(counts)))
        return counts

    def gen_records(self, params, first_index, n, dst):
        check(lib().fa_gen_records(self._h, C.byref(params), first_index, n, _ptr(dst)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().fa_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def gen_records_host(params, first_index, n):
    """CPU instance of the synthetic stream generator (bit-identical to the device one)."""
    out = np.zeros((n, REC_BYTES), dtype=np.uint8)
    check(lib().fa_gen_records(None, C.byref(params), first_index, n, _ptr(out)))
    return out


def gen_key(params, rank):
    out = np.zeros(40, dtype=np.uint8)
    check(lib().fa_gen_key(C.byref(params), rank, _ptr(out)))
    return out
