"""FA_F_NONBLOCKING_EVICT in KERNEL_MAP mode: fa_evict swaps in an empty map (identity, metric and feature lines) and
scans the retired one on its own stream, the way flow_monitor keeps updating aggregated_flows and the per-CPU feature
maps while the evictor runs LookupAndDeleteMap (pkg/tracer/tracer.go:1063-1157).  A packet or sample folded before the
swap is in the evicted generation, everything after it in the next one.  The DNS correlation table, the fallback ring
and the KERNEL_MAP counters are engine-wide and are not swapped.

Every check runs small on the engine emulation (CPU) and larger on the GPU, under both FA_KMAP_IMPL values."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_dns_correlate import dns_stream, query, response
from test_gpu_features import keys_of, make_add, make_dns
from test_kmap_emulation import messy_stream
from test_pktdrop import make_drops

pytestmark = pytest.mark.timeout(900)

BLOCKS = ("records", "dns", "additional", "pkt_drops", "rtt_min", "present")
WIDTHS = (144, 64, 32, 32, 8, 1)


@pytest.fixture(params=["2", "1"])
def kmap_impl(request, monkeypatch):
    """FA_KMAP_IMPL: 2 = one streaming pass + per-flow finalisation (default), 1 = seven per-record passes."""
    monkeypatch.setenv("FA_KMAP_IMPL", request.param)
    return request.param


def kmap_engine(max_entries, flags=0, **kw):
    import netobserv_ebpf_agent_b200 as fa
    return fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=fa.FA_F_NONBLOCKING_EVICT | flags, **kw)


def evict_ex_to(eng, cap, device, on_gpu):
    """fa_evict_ex with each block in host memory or, where device[i] is set, in device memory (torch on the GPU; on the
    emulation the engine's own device allocations, which are host memory there) -> the six blocks as numpy arrays."""
    from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib
    bufs, ptrs = [], []
    for w, dev in zip(WIDTHS, device):
        if not dev:
            b = np.zeros(cap * w, np.uint8); p = b.ctypes.data
        elif on_gpu:
            import torch
            b = torch.zeros(cap * w, dtype=torch.uint8, device="cuda"); p = b.data_ptr()
        else:
            b = C.c_void_p(); check(lib().fa_device_alloc(eng._h, cap * w, C.byref(b))); p = b.value
        bufs.append(b); ptrs.append(p)
    o = EvictOut(*ptrs)
    got = C.c_size_t(0)
    check(lib().fa_evict_ex(eng._h, C.byref(o), cap, C.byref(got)))
    g, out = got.value, []
    for b, w in zip(bufs, WIDTHS):
        if isinstance(b, C.c_void_p):
            a = np.frombuffer(C.string_at(b.value, cap * w), np.uint8).copy()
            check(lib().fa_device_free(eng._h, b))
        elif not isinstance(b, np.ndarray):
            a = b.cpu().numpy()
        else:
            a = b
        out.append(a[: g * w].reshape(g, w))
    out[4], out[5] = out[4].view(np.uint64).reshape(-1), out[5].reshape(-1)
    return tuple(out)


def assert_same_blocks(got, want, what=""):
    gp, op = O.sort_perm(got[0]), O.sort_perm(want[0])
    assert len(gp) == len(op), (what, len(gp), len(op))
    for name, g, o in zip(BLOCKS, got, want):
        gs, os_ = g.reshape(len(g), -1)[gp], o.reshape(len(o), -1)[op]
        if not np.array_equal(gs, os_):
            bad = np.nonzero((gs != os_).any(axis=1))[0]
            raise AssertionError(f"{what} {name}: {len(bad)} of {len(gs)} differ; first {bad[0]}:\n engine {gs[bad[0]].tolist()}\n oracle {os_[bad[0]].tolist()}")


# ------------------------------------------------------------------------------------------------- 1. flags
def check_flags():
    import netobserv_ebpf_agent_b200 as fa
    feats = (fa.FA_F_ENABLE_RTT, fa.FA_F_ENABLE_DNS, fa.FA_F_ENABLE_PKT_DROP)
    for extra in (0, fa.FA_F_RINGBUF_FALLBACK, *feats, fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS,
                  fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP | fa.FA_F_RINGBUF_FALLBACK):
        with kmap_engine(64, extra, max_batch=256) as eng:
            assert eng.live_flows() == 0 and len(eng.evict()) == 0
    for f in feats:
        with pytest.raises(fa.FlowAggError) as ei:
            fa.FlowAggEngine(64, flags=fa.FA_F_NONBLOCKING_EVICT | f)
        assert ei.value.code == -22


def test_flag_accepted_in_kernel_map_mode_refused_in_accounter_with_features(engine_emul):
    check_flags()


@pytest.mark.gpu
def test_flag_accepted_in_kernel_map_mode_refused_in_accounter_with_features_gpu():
    check_flags()


# ------------------------------------------------------------------------------------------------- 2. messy streams
def check_generations(recs, max_entries, max_batch, cuts, ringbuf=True):
    """Evict at fixed record indices: every generation equals O.KernelMap evicted at the same points."""
    import netobserv_ebpf_agent_b200 as fa
    b = O.as_bytes(recs)
    km = O.KernelMap(max_entries, ringbuf_fallback=ringbuf)
    with kmap_engine(max_entries, fa.FA_F_RINGBUF_FALLBACK if ringbuf else 0, max_batch=max_batch) as eng:
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            part = b[lo * O.REC: hi * O.REC]
            km.packets(part)
            eng.ingest(part)
            want, got = O.sort_records(km.evict()), O.sort_records(eng.evict())
            assert want.shape == got.shape and np.array_equal(want, got), (lo, hi)
            assert eng.live_flows() == 0
            n_sp = km.spilled()
            if ringbuf:
                gs = eng.read_spilled()
                assert len(gs) == n_sp
                if n_sp:
                    ws = km.spilled_records(n_sp)
                    assert np.array_equal(ws[np.lexsort(ws.T[::-1])], gs[np.lexsort(gs.T[::-1])])
        assert len(eng.evict()) == 0
        st = eng.stats()
    assert st["observed_intf_missed"] == km.intf_missed and st["hashmap_fail_create"] == km.fail_create
    assert st["spills"] == 0 and st["ringbuf_dropped"] == 0 and st["evictions"] == len(cuts)


def test_messy_stream_generations_on_the_emulation(engine_emul, kmap_impl):
    check_generations(messy_stream(51, 2_400, 120, n_ifaces=9), 1 << 9, 1_024, [0, 700, 1_500, 2_400])
    full = messy_stream(52, 2_000, 400, tls=False)                                  # the map fills in every generation
    check_generations(full, 150, 1_024, [0, 900, 2_000], ringbuf=True)
    check_generations(full, 150, 1_024, [0, 900, 2_000], ringbuf=False)


@pytest.mark.gpu
def test_messy_stream_generations_gpu(kmap_impl):
    check_generations(messy_stream(11, 60_000, 300), 1 << 12, 997, [0, 10_000, 35_000, 60_000])
    check_generations(messy_stream(42, 400_000, 50_000, n_ifaces=3), 1 << 16, 1 << 16, [0, 150_000, 400_000])
    full = messy_stream(31, 30_000, 2_000, tls=False)
    check_generations(full, 500, 4_096, [0, 12_000, 30_000], ringbuf=True)
    check_generations(full, 500, 4_096, [0, 12_000, 30_000], ringbuf=False)


# ------------------------------------------------------------------------------------------------- 3. feature folds
def check_feature_generations(n_pk, n_keys, n_feat, max_entries, max_batch, on_gpu):
    """KERNEL_MAP + RTT + DNS + PKT_DROP with packets and samples interleaved and an eviction between calls: every
    generation's six blocks equal O.FlowMap over the same calls.  Samples of flows that get their first packet in a later
    call (or never) come first; generations alternate host, device and mixed output pointers."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(81)
    pk = messy_stream(81, n_pk, n_keys, n_ifaces=5)
    allk = np.concatenate([np.unique(pk[:, :40], axis=0), keys_of(82, max(n_keys // 5, 3))])
    add, dns, drops = make_add(rng, allk, n_feat), make_dns(rng, allk, n_feat), make_drops(rng, allk, n_feat)
    h, p1, p2 = n_feat // 2, n_pk // 3, 2 * n_pk // 3
    calls = [                                              # (engine method, FlowMap method, data), eviction after each group
        [("ingest_additional", "fold_additional", add[:h]), ("ingest", "packets_kmap", pk[:p1]), ("ingest_dns", "fold_dns", dns[:h]),
         ("ingest_pkt_drops", "fold_drops", drops[:h])],
        [("ingest_pkt_drops", "fold_drops", drops[h:]), ("ingest", "packets_kmap", pk[p1:p2]), ("ingest_additional", "fold_additional", add[h:])],
        [("ingest_dns", "fold_dns", dns[h:])],             # feature-only generation
        [("ingest", "packets_kmap", pk[p2:])],
    ]
    outputs = [(0,) * 6, (1,) * 6, (0, 1, 1, 1, 1, 1), (1, 0, 0, 0, 0, 0)]
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP | fa.FA_F_RINGBUF_FALLBACK
    om, missed = O.FlowMap(), 0
    with kmap_engine(max_entries, flags, max_batch=max_batch) as eng:
        for gi, (group, device) in enumerate(zip(calls, outputs)):
            for meth, ometh, data in group:
                getattr(eng, meth)(data)
                r = getattr(om, ometh)(data)
                missed += r if ometh == "packets_kmap" else 0
            want = om.evict_ex()
            got = evict_ex_to(eng, max(len(want[0]), 1), device, on_gpu)
            assert_same_blocks(got, want, f"generation {gi}")
            assert len(got[0]) > 0 and eng.live_flows() == 0
        st = eng.stats()
    assert st["observed_intf_missed"] == missed and st["pkt_drops_ingested"] == n_feat and st["evictions"] == len(calls)


def test_feature_generations_on_the_emulation(engine_emul, kmap_impl):
    check_feature_generations(n_pk=3_000, n_keys=150, n_feat=900, max_entries=1 << 10, max_batch=1_024, on_gpu=False)


@pytest.mark.gpu
def test_feature_generations_gpu(kmap_impl):
    check_feature_generations(n_pk=60_000, n_keys=2_000, n_feat=20_000, max_entries=1 << 15, max_batch=16_384, on_gpu=True)


# ------------------------------------------------------------------------------------------------- 4. DNS correlation
def check_dns_across_evictions(stream_len, max_entries, max_batch):
    """dns_flows is not part of the swap: a query ingested before an eviction and answered after it gives its latency
    sample in the next generation, exactly as O.DnsCorrelator does; purge_stale_dns keeps working after swaps."""
    import netobserv_ebpf_agent_b200 as fa
    with kmap_engine(max_entries, fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_RTT, max_batch=max_batch) as eng:
        # hand case: the query in generation 1, its response in generation 2
        pk = gen_host(seed=91, n=500, n_keys=40)
        eng.ingest(pk); eng.ingest_dns_packets(query(1_000, 77))
        assert len(eng.evict()) == len(np.unique(pk[:, :40], axis=0))
        assert eng.stats()["dns_queries_pending"] == 1
        eng.ingest_dns_packets(response(1_450, 77))
        recs, dns, _, _, _, pres = eng.evict_ex()
        assert len(recs) == 1 and pres[0] == 1
        d = dns.view(O.DNS_DTYPE).reshape(-1)[0]
        assert (d["latency"], d["id"], d["errno"]) == (450, 77, 0)
        assert bytes(recs[0, :40]) == bytes(response(0, 0)["id"][0])
        # a messy stream cut into batches, an eviction after each one and a purge in between
        s = dns_stream(7, stream_len, n_clients=30, n_ids=4)
        corr, om = O.DnsCorrelator(), O.FlowMap()
        corr.packets(np.concatenate([query(1_000, 77), response(1_450, 77)]))
        cuts = [0, stream_len // 4, stream_len // 2, 3 * stream_len // 4, stream_len]
        for k, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
            eng.ingest_dns_packets(s[lo:hi])
            om.fold_dns(corr.packets(s[lo:hi]))
            if k == 1:
                now, timeout = int(s[hi - 1]["dns"]["end"]), 100
                eng.purge_stale_dns(now, timeout)
                gone = corr.purge(now, timeout)
                assert gone > 0 and eng.stats()["dns_queries_purged"] == gone
            assert eng.stats()["dns_queries_pending"] == corr.pending()
            assert_same_blocks(eng.evict_ex(), om.evict_ex(), f"batch {k}")


def test_dns_correlation_across_evictions_on_the_emulation(engine_emul, kmap_impl):
    check_dns_across_evictions(2_000, 1 << 12, 1_024)


@pytest.mark.gpu
def test_dns_correlation_across_evictions_gpu(kmap_impl):
    check_dns_across_evictions(40_000, 1 << 16, 1 << 14)


# ------------------------------------------------------------------------------------------------- 5. concurrent
def refold(gens):
    """Fold evicted generations in generation order into one view per flow.  The base is AccumulateBase over the
    generations that saw packets, adopted whole from the first of them (a generation where the flow only had feature
    samples contributes its start / end only); feature blocks merge as AccumulateDNS / AccumulateDrops /
    AccumulateAdditional do (first sample's timestamps and name, max latency / RTT, last non-zero id, cause and state,
    last errno, OR of flags, saturating drop counters); rtt_min is the smallest non-zero value; present is OR-ed."""
    acc = {}
    for g in gens:
        recs, dns, add, drops, rmin, pres = g
        for i in range(len(recs)):
            k = recs[i, :40].tobytes()
            row = [recs[i].copy(), dns[i].copy(), add[i].copy(), drops[i].copy(), int(rmin[i]), int(pres[i])]
            if k not in acc:
                acc[k] = row
                continue
            cur = acc[k]
            p, o = cur[0].view(O.REC_DTYPE)[0], row[0].view(O.REC_DTYPE)[0]
            start = min([x for x in (int(p["start"]), int(o["start"])) if x] or [0])
            end = max(int(p["end"]), int(o["end"]))
            if p["packets"] == 0:
                cur[0] = row[0].copy()
            elif o["packets"] != 0:
                cur[0][40:] = O.accumulate_base(cur[0][40:], row[0][40:])
            r = cur[0].view(O.REC_DTYPE)[0]
            r["start"], r["end"] = start, end
            if row[5] & 1:
                if cur[5] & 1:
                    a, b = cur[1].view(O.DNS_DTYPE)[0], row[1].view(O.DNS_DTYPE)[0]
                    a["flags"] |= b["flags"]; a["errno"] = b["errno"]; a["latency"] = max(a["latency"], b["latency"])
                    a["id"] = b["id"] if b["id"] else a["id"]
                else:
                    cur[1] = row[1].copy()
            if row[5] & 2:
                if cur[5] & 2:
                    a, b = cur[2].view(O.ADD_DTYPE)[0], row[2].view(O.ADD_DTYPE)[0]
                    a["rtt"] = max(a["rtt"], b["rtt"])
                else:
                    cur[2] = row[2].copy()
            if row[5] & 4:
                if cur[5] & 4:
                    a, b = cur[3].view(O.DROP_DTYPE)[0], row[3].view(O.DROP_DTYPE)[0]
                    a["bytes"] = min(65_535, int(a["bytes"]) + int(b["bytes"]))
                    a["packets"] = min(65_535, int(a["packets"]) + int(b["packets"]))
                    a["flags"] |= b["flags"]
                    a["cause"] = b["cause"] if b["cause"] else a["cause"]
                    a["state"] = b["state"] if b["state"] else a["state"]
                else:
                    cur[3] = row[3].copy()
            cur[4] = min([x for x in (cur[4], row[4]) if x] or [0])
            cur[5] |= row[5]
    rows = list(acc.values())
    return (np.array([r[0] for r in rows], np.uint8).reshape(-1, 144), np.array([r[1] for r in rows], np.uint8).reshape(-1, 64),
            np.array([r[2] for r in rows], np.uint8).reshape(-1, 32), np.array([r[3] for r in rows], np.uint8).reshape(-1, 32),
            np.array([r[4] for r in rows], np.uint64), np.array([r[5] for r in rows], np.uint8))


def check_concurrent(n, n_keys, n_feat, max_entries, max_batch, chunk):
    """An evictor thread loops on evict_ex(cap=max_entries) while this thread feeds packets and RTT / DNS / drop samples
    in chunks.  Whatever the interleaving, the generations folded in order (refold) equal the oracle's fold of the
    whole stream, because the streams are built so that generations compose: descriptors are constant per key and every
    key has one non-zero interface (no observed-interface list, no last-writer field that differs between records),
    packet timestamps increase with the record index (the map's "last writer" end is the maximum), the samples carry no
    Ethernet protocol (a feature-only generation cannot set the base's) and no IPsec fields, and max_entries covers every
    key (no record meets a full map).  Timing is not asserted."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(5)
    pk = gen_host(seed=44, n=n, n_keys=n_keys, dist=1)
    allk = np.concatenate([np.unique(pk[:, :40], axis=0), keys_of(45, max(n_keys // 10, 3))])
    assert len(allk) <= max_entries
    add, dns, drops = make_add(rng, allk, n_feat), make_dns(rng, allk, n_feat), make_drops(rng, allk, n_feat)
    add["add"]["eth"] = 0; add["add"]["ipsec_ret"] = 0; add["add"]["ipsec_enc"] = 0
    dns["dns"]["eth"] = 0; drops["drop"]["eth"] = 0
    feats = [("ingest_additional", add), ("ingest_dns", dns), ("ingest_pkt_drops", drops)]
    n_chunks = -(-n // chunk)
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP | fa.FA_F_RINGBUF_FALLBACK
    evicted, errors, stop = [], [], threading.Event()
    with kmap_engine(max_entries, flags, max_batch=max_batch) as eng:
        def evictor():
            try:
                while not stop.is_set():
                    evicted.append(eng.evict_ex(cap=max_entries))
            except Exception as ex:                                 # reported by the main thread
                errors.append(ex)
        t = threading.Thread(target=evictor)
        t.start()
        try:
            for c in range(n_chunks):
                rc, took = eng.ingest(pk[c * chunk:(c + 1) * chunk])
                assert rc == 0 and took == min(chunk, n - c * chunk)
                for meth, data in feats:
                    lo, hi = c * len(data) // n_chunks, (c + 1) * len(data) // n_chunks
                    getattr(eng, meth)(data[lo:hi])
        finally:
            stop.set(); t.join()
        assert not errors, errors
        evicted.append(eng.evict_ex())
        st = eng.stats()
        assert len(eng.read_spilled()) == 0
    assert st["records_ingested"] == n and st["flows_evicted"] == sum(len(g[0]) for g in evicted)
    assert st["pkt_drops_ingested"] == n_feat and st["dns_ingested"] == n_feat and st["additional_ingested"] == n_feat
    assert sum(1 for g in evicted if len(g[0])) >= 2                 # the evictor really ran during the ingest
    om = O.FlowMap()
    om.packets_kmap(pk); om.fold_additional(add); om.fold_dns(dns); om.fold_drops(drops)
    assert_same_blocks(refold(evicted), om.evict_ex(), "union of the generations")


def test_ingest_while_evicting_on_the_emulation(engine_emul, kmap_impl):
    check_concurrent(n=8_000, n_keys=300, n_feat=1_500, max_entries=1 << 10, max_batch=1_024, chunk=500)


@pytest.mark.gpu
def test_ingest_while_evicting_gpu(kmap_impl):
    check_concurrent(n=1_000_000, n_keys=20_000, n_feat=100_000, max_entries=1 << 15, max_batch=1 << 17, chunk=1 << 16)
