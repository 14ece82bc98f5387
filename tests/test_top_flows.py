"""fa_top_flows: the exact top-k live flows by bytes or packets, ranked on the device without evicting.

Rank order (include/flowagg.h): metric descending, then ascending slot hash (oracle_slot_hash), then ascending key
bytes.  Ranking cases compare the rows with the oracle's flows sorted by that order, bit for bit; the other cases compare
every block of the peek with the fa_evict_ex row of the same flow taken right after, and check that nothing changed.

Every case runs on the engine emulation (`engine_emul`, small, CPU suite) and on the device (`gpu`, 10^5 to 10^6
flows, k up to 10^5)."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_adversarial_parity import DevBuf, key_families, pre_aggregate, table_slots
from test_dns_correlate import query, response
from test_evict_blocks import BLOCKS, WIDTHS
from test_gpu_features import keys_of, make_add, make_dns
from test_pktdrop import make_drops

pytestmark = pytest.mark.timeout(900)


# ---------------------------------------------------------------------------------------------------- ranking helper
def top_order(recs, by):
    """Permutation that ranks (n, 144) records as fa_top_flows does: metric descending, slot hash ascending, key bytes
    ascending."""
    r = np.ascontiguousarray(recs).view(np.uint8).reshape(-1, O.REC)
    v = r.view(O.REC_DTYPE).reshape(-1)
    m = v["bytes"].astype(np.uint64) if by == "bytes" else v["packets"].astype(np.uint64)
    h = np.array([O.lib().oracle_slot_hash(O._p(np.ascontiguousarray(k))) for k in r[:, :O.ID]], dtype=np.uint64)
    return np.lexsort([r[:, c] for c in range(O.ID - 1, -1, -1)] + [h, ~m])


def ranked(recs, by, k):
    r = np.ascontiguousarray(recs).view(np.uint8).reshape(-1, O.REC)
    return r[top_order(r, by)[:k]]


def oracle_flows(batches, max_entries):
    acc = O.Accounter(max_entries)
    for b in batches:
        acc.account(b)
    out = acc.evict()
    acc.close()
    return out


def rows(blocks):
    return [np.ascontiguousarray(b).view(np.uint8).reshape(len(b), -1) for b in blocks]


def assert_rows_equal(got, want, what=""):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} rows differ, first at rank {int(bad[0])}")


def same_as_eviction(peek, evicted, by):
    """Every block row of the peek equals the eviction's row of the same flow, and the peek is the eviction's top."""
    peek, evicted = rows(peek), rows(evicted)
    order = top_order(evicted[0], by)[: len(peek[0])]
    for name, p, e in zip(BLOCKS, peek, evicted):
        assert_rows_equal(p, e[order], name)


# ---------------------------------------------------------------------------------------------------- 1. ranking
def check_ranking(n, n_keys, dist, varying, ks):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=11 + dist + 2 * varying, n=n, n_keys=n_keys, dist=dist, varying=varying)
    max_entries = 2 * n_keys
    want = oracle_flows([recs], max_entries)
    live = len(want)
    with fa.FlowAggEngine(max_entries) as eng:
        assert eng.ingest(recs) == (fa.FA_OK, n)
        for by in ("bytes", "packets"):
            for k in ks(live):
                got = eng.top_flows(k, by)[0]
                assert_rows_equal(got, ranked(want, by, k), f"{by} k={k}")
        assert eng.live_flows() == live


def ks_of(live):
    return sorted({1, 17, 1000, live - 1, live, live + 5})


@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
@pytest.mark.parametrize("varying", [0, 1])
def test_ranking_emul(engine_emul, dist, varying):
    check_ranking(3_000, 1_200, dist, varying, ks_of)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
@pytest.mark.parametrize("varying", [0, 1])
def test_ranking_gpu(dist, varying):
    check_ranking(600_000, 150_000, dist, varying, lambda live: sorted({1, 17, 1000, 100_000, live - 1, live, live + 5}))


# The emulation's tables fit the default scratch (k + 4096 entries), so the select would stop before its first digit
# pass.  FA_TOP_SLACK=0 shrinks the scratch to a power of two >= max(k, 1024): the digit passes, the stop test and the
# compaction at a resolved prefix then run on small tables too (and over more passes on the device).
@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
def test_ranking_digit_passes_emul(engine_emul, monkeypatch, dist):
    monkeypatch.setenv("FA_TOP_SLACK", "0")
    check_ranking(6_000, 3_000, dist, 1, lambda live: [1, 17, 1000])


@pytest.mark.gpu
@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
def test_ranking_digit_passes_gpu(monkeypatch, dist):
    monkeypatch.setenv("FA_TOP_SLACK", "0")
    check_ranking(600_000, 150_000, dist, 1, lambda live: [1, 17, 1000, 100_000])


def test_ties_digit_passes_emul(engine_emul, monkeypatch):
    monkeypatch.setenv("FA_TOP_SLACK", "0")
    check_ties(1_500, 4_000)


# ---------------------------------------------------------------------------------------------------- 2. non-destructive
def check_non_destructive(n, n_keys):
    import netobserv_ebpf_agent_b200 as fa
    a = gen_host(seed=21, n=n, n_keys=n_keys, dist=1)
    b = gen_host(seed=22, n=n, n_keys=n_keys, dist=1, first=n)
    max_entries = 4 * n_keys
    with fa.FlowAggEngine(max_entries) as eng:
        eng.ingest(a)
        live = eng.live_flows()
        first = eng.top_flows(50)
        assert eng.live_flows() == live
        assert_rows_equal(first[0], ranked(oracle_flows([a], max_entries), "bytes", 50), "after A")
        eng.ingest(b)
        live = eng.live_flows()
        p1, p2 = eng.top_flows(live + 5, "packets"), eng.top_flows(live + 5, "packets")
        assert eng.live_flows() == live
        for x, y in zip(p1, p2):
            assert np.array_equal(x, y)
        want = oracle_flows([a, b], max_entries)
        assert_rows_equal(p1[0], ranked(want, "packets", live), "after A + B")
        assert_rows_equal(O.sort_records(eng.evict()), O.sort_records(want), "eviction")


def test_non_destructive_emul(engine_emul):
    check_non_destructive(2_000, 600)


@pytest.mark.gpu
def test_non_destructive_gpu():
    check_non_destructive(500_000, 100_000)


# ---------------------------------------------------------------------------------------------------- 3. feature folds
def feature_engine(n, n_keys, seed):
    """An engine with RTT + DNS + packet-drop folds, samples for flows with and without base records, DNS latency samples
    from fa_ingest_dns_packets."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(seed)
    recs = gen_host(seed=seed, n=n, n_keys=n_keys, dist=1)
    keys = np.concatenate([np.unique(recs[:, :40], axis=0), keys_of(seed + 1, 16)])    # 16 feature-only flows
    eng = fa.FlowAggEngine(4 * n_keys, flags=fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP)
    eng.ingest(recs)
    eng.ingest_additional(make_add(rng, keys, n // 4))
    eng.ingest_dns(make_dns(rng, keys, n // 8))
    eng.ingest_pkt_drops(make_drops(rng, keys, n // 8))
    eng.ingest_dns_packets(np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001),
                                           response(9000, 9, sport=40001)]))
    return eng


def check_features(n, n_keys, ks):
    eng = feature_engine(n, n_keys, 31)
    try:
        live = eng.live_flows()
        peeks = [(k, by, eng.top_flows(k, by)) for k in ks(live) for by in ("bytes", "packets")]
        assert eng.live_flows() == live
        evicted = eng.evict_ex()
        assert len(evicted[0]) == live and (rows(evicted)[5] != 0).any()
        for k, by, p in peeks:
            assert len(p[0]) == min(k, live)
            same_as_eviction(p, evicted, by)
    finally:
        eng.close()


def test_feature_rows_emul(engine_emul):
    check_features(1_500, 400, lambda live: [17, live + 5])


@pytest.mark.gpu
def test_feature_rows_gpu():
    check_features(400_000, 100_000, lambda live: [17, 100_000, live + 5])


# ---------------------------------------------------------------------------------------------------- 4. ties
def check_ties(n_bg, slots_for):
    """Keys with one identical premix and equal metrics (the key bytes decide), in a background of one-record flows
    (every flow has one packet: by packets the whole table is one tie set, and k falls in its middle)."""
    import netobserv_ebpf_agent_b200 as fa
    bg = gen_host(seed=41, n=n_bg, n_keys=n_bg * 8, dist=0)
    bg = bg[np.unique(bg[:, :40], axis=0, return_index=True)[1]]
    full = key_families(43, table_slots(slots_for), n_full=64)["full"]
    tie = np.repeat(bg[:1], len(full), axis=0)
    tie[:, :40] = full
    recs = np.concatenate([bg, tie])
    recs.view(O.REC_DTYPE)["packets"] = 1
    v = recs.view(O.REC_DTYPE).reshape(-1)
    v["bytes"][-len(full):] = v["bytes"].max() + 1              # the premix family ties at the top by bytes
    max_entries = 2 * len(recs)
    want = oracle_flows([recs], max_entries)
    live = len(want)
    with fa.FlowAggEngine(max_entries) as eng:
        eng.ingest(recs)
        for by, k in (("bytes", 1), ("bytes", 17), ("bytes", 64), ("bytes", 70), ("packets", live // 2), ("packets", 1),
                      ("packets", live)):
            assert_rows_equal(eng.top_flows(k, by)[0], ranked(want, by, k), f"{by} k={k}")


def test_ties_emul(engine_emul):
    check_ties(1_500, 4_000)


@pytest.mark.gpu
def test_ties_gpu():
    check_ties(300_000, 1_000_000)


# ---------------------------------------------------------------------------------------------------- 5. wrap
def check_wrap(n, n_keys):
    import netobserv_ebpf_agent_b200 as fa
    recs = pre_aggregate(gen_host(seed=51, n=n, n_keys=n_keys, dist=1), np.random.default_rng(52))
    max_entries = 2 * n_keys
    want = oracle_flows([recs], max_entries)
    with fa.FlowAggEngine(max_entries) as eng:
        eng.ingest(recs)
        for by in ("bytes", "packets"):
            for k in (1, 17, len(want)):
                assert_rows_equal(eng.top_flows(k, by)[0], ranked(want, by, k), f"{by} k={k}")


def test_wrap_emul(engine_emul):
    check_wrap(2_000, 500)


@pytest.mark.gpu
def test_wrap_gpu():
    check_wrap(400_000, 100_000)


# ---------------------------------------------------------------------------------------------------- 6. KERNEL_MAP
def check_kernel_map(n, n_keys, max_entries, ringbuf, rtt):
    """Records of every flow arrive on two interfaces (packets on the second one do not count); with max_entries below
    the key count the map fills and the rest goes to the fallback ring, which is not ranked."""
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=61, n=n, n_keys=n_keys, dist=1)
    v = recs.view(O.REC_DTYPE).reshape(-1)
    other = np.random.default_rng(62).random(n) < 0.3
    v["if_index"] = np.where(other, 7, 3)
    flags = (fa.FA_F_RINGBUF_FALLBACK if ringbuf else 0) | (fa.FA_F_ENABLE_RTT if rtt else 0)
    with fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=flags) as eng:
        eng.ingest(recs)
        if rtt:
            eng.ingest_additional(make_add(np.random.default_rng(63), np.concatenate([recs[:50, :40], keys_of(64, 8)]), n // 8))
        live = eng.live_flows()
        peeks = [(k, by, eng.top_flows(k, by)) for k in (1, 17, live + 5) for by in ("bytes", "packets")]
        assert eng.live_flows() == live
        evicted = eng.evict_ex()
        assert len(evicted[0]) == live
        if ringbuf:
            assert len(eng.read_spilled()) > 0
        for k, by, p in peeks:
            same_as_eviction(p, evicted, by)


@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_emul(engine_emul, monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kernel_map(2_000, 600, 300 if ringbuf else 2_000, ringbuf, rtt=not ringbuf)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_gpu(monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kernel_map(400_000, 100_000, 20_000 if ringbuf else 200_000, ringbuf, rtt=not ringbuf)


# ---------------------------------------------------------------------------------------------------- 7. non-blocking
def check_nonblocking(n, n_keys, mode):
    import netobserv_ebpf_agent_b200 as fa
    a = gen_host(seed=71, n=n, n_keys=n_keys, dist=1)
    b = gen_host(seed=72, n=n, n_keys=n_keys, dist=1, first=n)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_NONBLOCKING_EVICT) as eng, \
            fa.FlowAggEngine(4 * n_keys, mode=mode) as ref:
        eng.ingest(a)
        eng.evict()
        eng.ingest(b)
        ref.ingest(b)
        live = eng.live_flows()
        got = eng.top_flows(live + 5, "packets")
        want = ref.evict_ex()
        same_as_eviction(got, want, "packets")
        if mode == fa.FA_MODE_ACCOUNTER:
            assert_rows_equal(got[0], ranked(oracle_flows([b], 4 * n_keys), "packets", live), "oracle")
        assert O.sort_records(eng.evict()).shape == (live, O.REC)


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_nonblocking_emul(engine_emul, mode):
    check_nonblocking(1_500, 500, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_nonblocking_gpu(mode):
    check_nonblocking(400_000, 100_000, mode)


# ---------------------------------------------------------------------------------------------------- 8. placement
def top_filled(eng, by, k, device, on_gpu):
    """fa_top_flows into blocks pre-filled with 0xFF, each in host memory or, where device[i] is set, in device memory
    -> the six blocks as (n, width) uint8 arrays."""
    from netobserv_ebpf_agent_b200._lib import FA_TOP_BYTES, FA_TOP_PACKETS, EvictOut, check, lib
    bufs, ptrs = [], []
    for w, dev in zip(WIDTHS, device):
        if not dev:
            b = np.full(k * w, 0xFF, np.uint8); p = b.ctypes.data
        elif on_gpu:
            import torch
            b = torch.full((k * w,), 0xFF, dtype=torch.uint8, device="cuda"); p = b.data_ptr()
        else:
            b = C.c_void_p(); check(lib().fa_device_alloc(eng._h, k * w, C.byref(b))); p = b.value
            C.memset(p, 0xFF, k * w)
        bufs.append(b); ptrs.append(p)
    got = C.c_size_t(0)
    check(lib().fa_top_flows(eng._h, FA_TOP_BYTES if by == "bytes" else FA_TOP_PACKETS, k, C.byref(EvictOut(*ptrs)),
                             C.byref(got)))
    out = []
    for b, w in zip(bufs, WIDTHS):
        if isinstance(b, C.c_void_p):
            a = np.frombuffer(C.string_at(b.value, k * w), np.uint8).copy()
            check(lib().fa_device_free(eng._h, b))
        elif isinstance(b, np.ndarray):
            a = b
        else:
            a = b.cpu().numpy()
        assert (a[got.value * w:] == 0xFF).all()                     # rows past n_out are not written
        out.append(a[: got.value * w].reshape(got.value, w))
    return out


PLACEMENTS = [(False,) * 6, (True,) * 6] + [tuple(i == j for j in range(6)) for i in range(6)]


def check_placement(n, n_keys, k, mode, rtt, on_gpu):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=81, n=n, n_keys=n_keys, dist=1)
    keys = np.concatenate([np.unique(recs[:, :40], axis=0), keys_of(82, 8)])
    produced = {"records", "additional", "rtt_min", "present"} if rtt else {"records"}
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_ENABLE_RTT if rtt else 0) as eng:
        eng.ingest(recs)
        if rtt:
            eng.ingest_additional(make_add(np.random.default_rng(83), keys, n // 4))
        want = rows(eng.top_flows(k))
        for device in PLACEMENTS:
            got = top_filled(eng, "bytes", k, device, on_gpu)
            for name, g, w in zip(BLOCKS, got, want):
                if name not in produced:
                    assert not g.any(), (device, name)
                assert np.array_equal(g, w), (device, name)


@pytest.mark.parametrize("mode,rtt", [(0, False), (0, True), (1, False), (1, True)])
def test_placement_emul(engine_emul, mode, rtt):
    check_placement(1_000, 300, 40, mode, rtt, on_gpu=False)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtt", [(0, False), (0, True), (1, False), (1, True)])
def test_placement_gpu(mode, rtt):
    check_placement(300_000, 80_000, 100_000, mode, rtt, on_gpu=True)


# ---------------------------------------------------------------------------------------------------- 9. errors
def check_errors(n, n_keys):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_INVAL, EvictOut, lib
    recs = gen_host(seed=91, n=n, n_keys=n_keys, dist=1)
    out = np.zeros((4, O.REC), np.uint8)
    got = C.c_size_t(7)
    with fa.FlowAggEngine(4 * n_keys) as eng:
        eng.ingest(recs)
        live = eng.live_flows()
        before = eng.stats()
        good, no_rec = EvictOut(records=out.ctypes.data), EvictOut()
        cases = [(None, 0, 4, C.byref(good), C.byref(got)), (eng._h, 0, 4, None, C.byref(got)),
                 (eng._h, 0, 4, C.byref(no_rec), C.byref(got)), (eng._h, 0, 4, C.byref(good), None),
                 (eng._h, 2, 4, C.byref(good), C.byref(got)), (eng._h, 0, 0, C.byref(good), C.byref(got)),
                 (eng._h, 0, fa.FA_TOP_MAX_K + 1, C.byref(good), C.byref(got))]
        for c in cases:
            assert lib().fa_top_flows(*c) == FA_E_INVAL, c
            assert got.value == 0
        assert eng.stats() == before
        assert eng.live_flows() == live
        assert not out.any()
        assert_rows_equal(O.sort_records(eng.evict()), O.sort_records(oracle_flows([recs], 4 * n_keys)), "eviction")


def test_errors_emul(engine_emul):
    check_errors(1_000, 300)


@pytest.mark.gpu
def test_errors_gpu():
    check_errors(200_000, 50_000)


# ---------------------------------------------------------------------------------------------------- device outputs
@pytest.mark.gpu
def test_device_outputs_and_device_ingest_gpu():
    """Device-resident input and device-resident records block, k = 10^5 over 10^6 flows."""
    import netobserv_ebpf_agent_b200 as fa
    import torch
    from netobserv_ebpf_agent_b200._lib import FA_TOP_BYTES, EvictOut, check, lib
    recs = gen_host(seed=101, n=2_000_000, n_keys=1_500_000, dist=0)
    max_entries = 2_000_000
    want = oracle_flows([recs], max_entries)
    k = 100_000
    with fa.FlowAggEngine(max_entries) as eng:
        buf = DevBuf(eng, recs.size, None)
        buf.write(recs)
        assert eng.ingest(buf.ptr, len(recs)) == (fa.FA_OK, len(recs))
        out = torch.zeros(k * O.REC, dtype=torch.uint8, device="cuda")
        got = C.c_size_t(0)
        check(lib().fa_top_flows(eng._h, FA_TOP_BYTES, k, C.byref(EvictOut(records=out.data_ptr())), C.byref(got)))
        assert got.value == k
        assert_rows_equal(out.cpu().numpy().reshape(k, O.REC), ranked(want, "bytes", k), "device records")
