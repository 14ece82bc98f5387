"""fa_group_flows: exact roll-ups of the live flows by a key mask (subnet, port, protocol), on the device, without
evicting.

The expected side groups flow rows on the host with numpy: the 40 key bytes ANDed with the mask (byte 39 cleared),
np.unique over a void view, np.add.at on uint64 for flows / bytes / packets (bytes wrap mod 2^64 the same way), the
smallest non-zero start, np.maximum.at for end and np.bitwise_or.at for flags.  The rows are the oracle's flows, or the
fa_evict_ex rows taken right after the call.  Both sides are sorted by key and compared as 88-byte rows, bit for bit,
for every mask of masks().  Every case runs on the engine emulation (`engine_emul`, a few thousand flows, CPU suite) and
on the device (`gpu`, 10^5 to 2·10^6 flows)."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_adversarial_parity import key_families, pre_aggregate, table_slots, uptime_times
from test_dns_correlate import query, response
from test_expire_flows import Replay
from test_gpu_features import keys_of, make_add, make_dns
from test_pktdrop import make_drops

pytestmark = pytest.mark.timeout(1200)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0 = 1_000_000
CHANGED_BY_GROUPING = ("kernel_launches", "d2h_bytes")


# ---------------------------------------------------------------------------------------------------- masks, expected side
def masks():
    """name -> 40-byte mask: one group, one group per flow, src /120 (an IPv4 /24), dst /112 + dst port, proto + dst port,
    a mask with byte 39 set, and three seeded random masks (sparse bits in every byte: word and byte order)."""
    import netobserv_ebpf_agent_b200 as fa
    m = {"zero": fa.group_mask(), "ones": np.full(40, 0xFF, np.uint8), "src120": fa.group_mask(src_prefix=120),
         "dst112_dport": fa.group_mask(dst_prefix=112, dst_port=True), "proto_dport": fa.group_mask(proto=True, dst_port=True)}
    b39 = fa.group_mask(src_prefix=124, proto=True, icmp=True)
    b39[39] = 0xFF
    m["byte39"] = b39
    rng = np.random.default_rng(4242)
    for i in range(3):
        bits = (rng.random((40, 8)) < 0.12).astype(np.uint8)
        m[f"random{i}"] = np.packbits(bits, axis=1).reshape(40)
    return m


def as_rows(recs):
    return np.ascontiguousarray(recs).view(np.uint8).reshape(-1, O.REC)


def group_rows(recs, mask):
    """The expected fa_group_flows result for flow rows `recs` (n, 144), sorted by key."""
    from netobserv_ebpf_agent_b200 import GROUP_DTYPE
    r = as_rows(recs)
    v = r.view(O.REC_DTYPE).reshape(-1)
    k = r[:, :O.ID] & np.asarray(mask, np.uint8)[None, :]
    k[:, 39] = 0
    uk, inv = np.unique(np.ascontiguousarray(k).view("V40").ravel(), return_inverse=True)
    inv = inv.ravel()
    out = np.zeros(len(uk), GROUP_DTYPE)
    out["key"] = np.frombuffer(uk.tobytes(), np.uint8).reshape(-1, 40)
    for f, x in (("flows", np.ones(len(r), np.uint64)), ("bytes", v["bytes"].astype(np.uint64)),
                 ("packets", v["packets"].astype(np.uint64))):
        acc = np.zeros(len(uk), np.uint64)
        np.add.at(acc, inv, x)
        out[f] = acc
    start = v["start"].astype(np.uint64)
    lo = np.full(len(uk), np.iinfo(np.uint64).max, np.uint64)
    np.minimum.at(lo, inv, np.where(start == 0, np.iinfo(np.uint64).max, start))
    out["start_mono_time_ts"] = np.where(lo == np.iinfo(np.uint64).max, 0, lo)
    end = np.zeros(len(uk), np.uint64)
    np.maximum.at(end, inv, v["end"].astype(np.uint64))
    out["end_mono_time_ts"] = end
    flags = np.zeros(len(uk), np.uint16)
    np.bitwise_or.at(flags, inv, v["flags"].astype(np.uint16))
    out["flags"] = flags
    return out


def by_key(g):
    g = np.ascontiguousarray(g)
    return g[np.argsort(np.ascontiguousarray(g["key"]).view("V40").ravel(), kind="stable")]


def assert_groups(got, want, what=""):
    g = by_key(got).view(np.uint8).reshape(-1, 88)
    w = by_key(want).view(np.uint8).reshape(-1, 88)
    assert len(g) == len(w), (what, len(g), len(w))
    if not np.array_equal(g, w):
        bad = np.nonzero((g != w).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(g)} groups differ, first at {int(bad[0])}")


def check_masks(eng, flows, what, which=None):
    """Every mask (or those named in `which`) against the grouping of the flow rows `flows`."""
    for name, m in masks().items():
        if which is None or name in which:
            assert_groups(eng.group_flows(m), group_rows(flows, m), f"{what} / {name}")


# ---------------------------------------------------------------------------------------------------- 1. oracle parity
def check_oracle(n, n_keys, mode, dist, varying, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=2101 + dist + 2 * varying + 4 * mode, n=n, n_keys=n_keys, dist=dist, varying=varying, t0=T0)
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        for part in np.array_split(recs, 2):
            eng.ingest(part)
            rep.add("base", part)
            flows = rep.state()[0]
            assert eng.live_flows() == len(flows)
            check_masks(eng, flows, "oracle")
        ev = eng.evict_ex()
        assert len(ev[0]) == len(flows)
        assert_groups(group_rows(ev[0], masks()["ones"]), group_rows(flows, masks()["ones"]), "eviction")


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
@pytest.mark.parametrize("varying", [0, 1])
def test_oracle_emul(engine_emul, mode, dist, varying):
    check_oracle(3_000, 1_000, mode, dist, varying, max_batch=700)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
@pytest.mark.parametrize("varying", [0, 1])
def test_oracle_gpu(mode, dist, varying):
    check_oracle(1_000_000, 300_000, mode, dist, varying, max_batch=1 << 17)


# ---------------------------------------------------------------------------------------------------- 2. wrap and time
ZERO_NET = bytes(10) + b"\xff\xff" + bytes([10, 99, 99])        # ::ffff:10.99.99.0/24: every start of its flows is 0


def check_wrap(n, n_keys, max_batch):
    """Pre-aggregated records at uptime scale: the all-zero group's byte sum wraps mod 2^64 and its packet sum passes
    2^32; one source /24 has only zero starts."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(2201)
    recs = pre_aggregate(uptime_times(gen_host(seed=2201, n=n, n_keys=n_keys, dist=1), rng), rng)
    zero = recs[: max(n // 50, 40)].copy()
    zero[:, 0:15] = np.frombuffer(ZERO_NET, np.uint8)
    zero[:, 15] = np.arange(len(zero)) % 256
    zero.view(O.REC_DTYPE)["start"] = 0
    recs = np.concatenate([recs, zero])
    rep = Replay()
    rep.add("base", recs)
    flows = rep.state()[0]
    v = flows.view(O.REC_DTYPE).reshape(-1)
    assert int(v["bytes"].astype(object).sum()) >= 1 << 64 and int(v["packets"].astype(np.uint64).sum()) > 1 << 32
    with fa.FlowAggEngine(2 * n_keys + len(zero), max_batch=max_batch) as eng:
        eng.ingest(recs)
        check_masks(eng, flows, "wrap")
        g = eng.group_flows(fa.group_mask(src_prefix=120))
        z = g[(g["key"][:, :15] == np.frombuffer(ZERO_NET, np.uint8)).all(axis=1)]
        assert len(z) == 1 and z["flows"][0] > 1 and z["start_mono_time_ts"][0] == 0 and z["end_mono_time_ts"][0] != 0
        one = eng.group_flows(fa.group_mask())
        assert len(one) == 1 and int(one["packets"][0]) > 1 << 32 and one["flows"][0] == len(flows)


def test_wrap_emul(engine_emul):
    check_wrap(3_000, 800, max_batch=700)


@pytest.mark.gpu
def test_wrap_gpu():
    check_wrap(800_000, 200_000, max_batch=1 << 17)


# ---------------------------------------------------------------------------------------------------- 3. colliding keys
def check_colliding(n_bg, max_batch):
    """Key families built against the group table's size: the identical-premix and the shared-low-32-bit families
    collide whatever the size, the chains share a home slot.  Identical-premix keys also sit in neighbouring flow-table
    slots, so they meet in one warp round: a peer set matched on the hash alone would merge them."""
    import netobserv_ebpf_agent_b200 as fa
    bg = gen_host(seed=2301, n=n_bg, n_keys=n_bg // 2, dist=1, t0=T0)
    rep0 = Replay()
    rep0.add("base", bg)
    live_guess = len(rep0.state()[0])
    fam = key_families(2302, table_slots(live_guess + 500), n_full=64, n_chain=300, n_way=32)
    fk = np.concatenate([fam["full"], fam["chain_last"], fam["chain_mid"], fam["way"], fam["elect"]])
    fr = np.repeat(bg[:1], len(fk), axis=0)
    fr[:, :40] = fk
    fr.view(O.REC_DTYPE).reshape(-1)["bytes"] = np.arange(1, len(fk) + 1, dtype=np.uint64) << np.uint64(20)
    recs = np.concatenate([bg, fr, fr[::3]])
    recs = recs[np.random.default_rng(2303).permutation(len(recs))]
    rep = Replay()
    rep.add("base", recs)
    flows = rep.state()[0]
    with fa.FlowAggEngine(2 * len(flows), max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.live_flows() == len(flows)
        assert table_slots(len(flows)) == table_slots(live_guess + 500)      # the chains hit the group table as built
        coarse = fa.group_mask(src_prefix=128, dst_prefix=128, proto=True)
        for name, m in (("ones", masks()["ones"]), ("coarse", coarse)):
            got = eng.group_flows(m)
            assert_groups(got, group_rows(flows, m), f"colliding / {name}")
        got = eng.group_flows(masks()["ones"])
        assert np.isin(np.ascontiguousarray(fk).view("V40").ravel(), np.ascontiguousarray(got["key"]).view("V40").ravel()).all()


def test_colliding_emul(engine_emul):
    check_colliding(2_000, max_batch=1_000)


@pytest.mark.gpu
def test_colliding_gpu():
    check_colliding(400_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 4. feature folds
def check_features(n, n_keys, max_batch):
    """RTT, DNS and packet-drop samples, feature-only flows (their start / end come from the feature lines) and DNS
    latency from fa_ingest_dns_packets.  The all-zero mask and a proto mask put feature-only flows and base flows in
    one group."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(2401)
    recs = gen_host(seed=2401, n=n, n_keys=n_keys, dist=1, t0=T0)
    keys = np.concatenate([np.unique(recs[:, :40], axis=0), keys_of(2402, 64)])        # 64 feature-only flows
    add, dns, drops = make_add(rng, keys, n // 4), make_dns(rng, keys, n // 8), make_drops(rng, keys, n // 8)
    rep = Replay()
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP
    with fa.FlowAggEngine(4 * n_keys, flags=flags, max_batch=max_batch) as eng:
        eng.ingest_additional(add[: len(add) // 2]); rep.add("add", add[: len(add) // 2])
        eng.ingest(recs); rep.add("base", recs)
        eng.ingest_dns(dns); rep.add("dns", dns)
        eng.ingest_pkt_drops(drops); rep.add("drop", drops)
        eng.ingest_additional(add[len(add) // 2:]); rep.add("add", add[len(add) // 2:])
        st = rep.state()
        only = np.isin(np.ascontiguousarray(st[0][:, :40]).view("V40").ravel(), np.ascontiguousarray(keys[-64:]).view("V40").ravel())
        assert only.sum() > 32
        check_masks(eng, st[0], "features, oracle")
        eng.ingest_dns_packets(np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001),
                                               response(9000, 9, sport=40001)]))
        got = {name: eng.group_flows(m) for name, m in masks().items()}
        evicted = eng.evict_ex()
        assert (evicted[5] != 0).any() and len(evicted[0]) >= len(st[0])
        for name, m in masks().items():
            assert_groups(got[name], group_rows(evicted[0], m), f"features, eviction / {name}")


def test_features_emul(engine_emul):
    check_features(2_000, 500, max_batch=600)


@pytest.mark.gpu
def test_features_gpu():
    check_features(600_000, 150_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 5. nothing changes
def check_nothing_changes(n, n_keys, max_batch):
    """With the sketch and the DNS correlation table in use: the stats (but launches and copies), the sketch, the
    pending DNS queries and a later eviction are those of a twin engine that never grouped; calls in a row, a call after
    FA_E_2BIG and a call after the group table had to grow are exact."""
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, GROUP_DTYPE, lib
    from test_adversarial_parity import SKETCH_SEED
    recs = gen_host(seed=2501, n=n, n_keys=n_keys, dist=1, t0=T0)
    small = recs[:300]
    kw = dict(flags=fa.FA_F_ENABLE_SKETCH | fa.FA_F_ENABLE_DNS, cms_log2_width=12, cms_depth=4, hll_precision=10,
              sketch_seed=SKETCH_SEED, max_batch=max_batch)
    pkts = np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001)])     # one query stays pending
    ms = masks()
    with fa.FlowAggEngine(4 * n_keys, **kw) as eng, fa.FlowAggEngine(4 * n_keys, **kw) as ref:
        for x in (eng, ref):
            x.ingest(small); x.ingest_dns_packets(pkts)
        live0 = eng.live_flows()
        assert live0 < 768                                          # the first group table has 1024 slots
        before = eng.stats()
        check_masks(eng, ref.top_flows(live0)[0], "small", ("zero", "ones", "src120"))   # the twin's rows, read in place
        after = eng.stats()
        for k in before:
            if k not in CHANGED_BY_GROUPING:
                assert after[k] == before[k], k
        assert after["kernel_launches"] > before["kernel_launches"] and after["d2h_bytes"] > before["d2h_bytes"]
        for x in (eng, ref):
            x.ingest(recs)
        flows = ref.top_flows(ref.live_flows())[0]
        assert len(flows) > 768                                     # the group table grows
        # FA_E_2BIG first: the table must come out of it all zero
        m = ms["src120"]
        n_want = len(group_rows(flows, m))
        out = np.full((n_want - 1) * 88, 0xA5, np.uint8)
        got = C.c_size_t(0)
        assert lib().fa_group_flows(eng._h, m.ctypes.data, out.ctypes.data, n_want - 1, C.byref(got)) == FA_E_2BIG
        assert got.value == n_want and (out == 0xA5).all()
        for name in ("proto_dport", "ones", "zero", "src120", "random1"):      # calls in a row, different masks
            assert_groups(eng.group_flows(ms[name]), group_rows(flows, ms[name]), f"in a row / {name}")
        s_eng, s_ref = eng.stats(), ref.stats()
        assert s_ref["dns_queries_pending"] == 1
        for k in s_ref:
            if k not in CHANGED_BY_GROUPING:
                assert s_eng[k] == s_ref[k], k
        for a, b in zip(eng.sketch_export(12, 4, 10), ref.sketch_export(12, 4, 10)):
            assert np.array_equal(a, b)
        assert eng.hll_estimate() == ref.hll_estimate()
        a, b = eng.evict_ex(), ref.evict_ex()
        for x, y in zip(a, b):
            x, y = as_rows_any(x), as_rows_any(y)
            assert np.array_equal(x[O.sort_perm(a[0])], y[O.sort_perm(b[0])])
        assert len(eng.group_flows(ms["zero"])) == 0 and GROUP_DTYPE.itemsize == 88


def as_rows_any(b):
    return np.ascontiguousarray(b).view(np.uint8).reshape(len(b), -1)


def test_nothing_changes_emul(engine_emul):
    check_nothing_changes(12_000, 4_000, 2_000)


@pytest.mark.gpu
def test_nothing_changes_gpu():
    check_nothing_changes(800_000, 200_000, 1 << 16)


# ---------------------------------------------------------------------------------------------------- 6. KERNEL_MAP
def check_kernel_map(n, n_keys, max_entries, ringbuf, max_batch):
    """Packets on a second interface (not counted in the first-seen interface's row); max_entries below the key count:
    the map fills, and with the fallback ring the records that did not enter are not grouped."""
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=2601 + ringbuf, n=n, n_keys=n_keys, dist=1, t0=T0)
    v = recs.view(O.REC_DTYPE).reshape(-1)
    v["if_index"] = np.where(np.random.default_rng(2602).random(n) < 0.3, 7, 3)
    rep = Replay(kmap=True, max_entries=max_entries, ringbuf=ringbuf)
    with fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=fa.FA_F_RINGBUF_FALLBACK if ringbuf else 0,
                          max_batch=max_batch) as eng:
        for part in np.array_split(recs, 2):
            eng.ingest(part)
            rep.add("base", part)
        flows = rep.state()[0]
        assert eng.live_flows() == len(flows) == max_entries
        if ringbuf:
            assert len(eng.read_spilled()) > 0
        check_masks(eng, flows, f"kmap ringbuf={ringbuf}")
        ev = eng.evict_ex()
        assert_groups(group_rows(ev[0], masks()["ones"]), group_rows(flows, masks()["ones"]), "eviction")
    assert (rep.spilled if ringbuf else rep.fail_create)


@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_emul(engine_emul, monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kernel_map(3_000, 1_000, 300, ringbuf, max_batch=700)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_gpu(monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kernel_map(600_000, 200_000, 50_000, ringbuf, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 7. full table
def check_physically_full(max_entries, n, max_batch):
    """FA_F_NO_FULL_CUT with more distinct keys than slots: every slot of the flow table is live."""
    import netobserv_ebpf_agent_b200 as fa
    slots = table_slots(max_entries)
    recs = gen_host(seed=2701, n=n, n_keys=1 << 30, dist=0, t0=T0)
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NO_FULL_CUT, max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.stats()["spills"] > 0 and eng.live_flows() == slots
        got = {name: eng.group_flows(m) for name, m in masks().items()}
        ev = eng.evict_ex()
        assert len(ev[0]) == slots
        for name, m in masks().items():
            assert_groups(got[name], group_rows(ev[0], m), f"full table / {name}")


def test_physically_full_emul(engine_emul):
    check_physically_full(700, 1_100, max_batch=600)                 # 1024 slots


@pytest.mark.gpu
def test_physically_full_gpu():
    check_physically_full(180_000, 600_000, max_batch=1 << 16)        # 2^18 slots


# ---------------------------------------------------------------------------------------------------- 8. non-blocking
def check_nonblocking_sequential(n, n_keys, mode):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=2801 + mode, n=n, n_keys=n_keys, dist=1, t0=T0)
    a, b = recs[: n // 2], recs[n // 2:]
    kmap = mode == fa.FA_MODE_KERNEL_MAP
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_NONBLOCKING_EVICT) as eng:
        eng.ingest(a)
        ra = Replay(kmap=kmap); ra.add("base", a)
        check_masks(eng, ra.state()[0], "first window", ("zero", "src120", "ones"))
        first = eng.evict_ex()
        assert len(first[0]) == len(ra.state()[0])
        assert len(eng.group_flows(masks()["zero"])) == 0              # the retired table is not grouped
        eng.ingest(b)
        rb = Replay(kmap=kmap); rb.add("base", b)
        check_masks(eng, rb.state()[0], "second window")
        assert_groups(group_rows(eng.evict_ex()[0], masks()["ones"]), group_rows(rb.state()[0], masks()["ones"]), "eviction")


def check_nonblocking_concurrent(n, n_keys, max_entries, max_batch, chunk):
    """An evictor thread against a thread that alternates ingest and group_flows: every call is consistent (the
    per-flow mask gives distinct keys with flows = 1, the one-group mask sums them), and the generations, re-folded,
    equal the oracle's fold of the stream."""
    import netobserv_ebpf_agent_b200 as fa
    from test_nonblocking_evict import refold
    recs = gen_host(seed=2803, n=n, n_keys=n_keys, dist=1, t0=T0)
    out, stop = [], threading.Event()
    ones, zero = masks()["ones"], masks()["zero"]
    calls = 0
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NONBLOCKING_EVICT, max_batch=max_batch) as eng:
        def evictor():
            while not stop.is_set():
                out.append(eng.evict(cap=max_entries).copy())
        t = threading.Thread(target=evictor)
        t.start()
        for lo in range(0, n, chunk):
            rc, took = eng.ingest(recs[lo:lo + chunk])
            assert rc == 0 and took == min(chunk, n - lo)
            g = eng.group_flows(ones if calls % 2 == 0 else zero, cap=max_entries)
            if calls % 2 == 0:
                assert (g["flows"] == 1).all()
                assert len(np.unique(np.ascontiguousarray(g["key"]).view("V40"))) == len(g)
            else:
                assert len(g) <= 1 and (len(g) == 0 or 0 < g["flows"][0] <= max_entries)
            calls += 1
        stop.set(); t.join()
        out.append(eng.evict().copy())
        st = eng.stats()
    assert st["records_ingested"] == n and st["flows_evicted"] == sum(len(p) for p in out)
    assert sum(1 for p in out if len(p)) >= 2
    assert np.array_equal(refold(out), refold([recs]))


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_nonblocking_emul(engine_emul, mode):
    check_nonblocking_sequential(2_000, 600, mode)


def test_nonblocking_concurrent_emul(engine_emul):
    check_nonblocking_concurrent(8_000, 400, 1 << 11, 1_024, 1_000)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_nonblocking_gpu(mode):
    check_nonblocking_sequential(800_000, 200_000, mode)


@pytest.mark.gpu
def test_nonblocking_concurrent_gpu():
    check_nonblocking_concurrent(2_000_000, 300_000, 1 << 20, 1 << 17, 1 << 16)


# ---------------------------------------------------------------------------------------------------- 9. placement, errors
class Out:
    """n_rows x 88 B of output filled with 0xA5: host pageable, pinned (fa_host_alloc) or device memory (a CUDA tensor
    on the GPU, fa_device_alloc memory on the emulation)."""

    def __init__(self, eng, kind, n_rows, on_gpu):
        from netobserv_ebpf_agent_b200._lib import check, lib
        self.eng, self.kind, self.nb = eng, kind, max(n_rows, 1) * 88
        if kind == "pageable":
            self.buf = np.full(self.nb, 0xA5, np.uint8)
            self.ptr = self.buf.ctypes.data
        elif kind == "pinned":
            p = C.c_void_p()
            check(lib().fa_host_alloc(self.nb, C.byref(p)))
            C.memset(p.value, 0xA5, self.nb)
            self.p, self.ptr = p, p.value
        elif on_gpu:
            import torch
            self.buf = torch.full((self.nb,), 0xA5, dtype=torch.uint8, device="cuda")
            self.ptr = self.buf.data_ptr()
        else:
            p = C.c_void_p()
            check(lib().fa_device_alloc(eng._h, self.nb, C.byref(p)))
            C.memset(p.value, 0xA5, self.nb)
            self.p, self.ptr = p, p.value

    def read(self):
        from netobserv_ebpf_agent_b200 import GROUP_DTYPE
        if self.kind == "pageable":
            b = self.buf.copy()
        elif hasattr(self, "buf"):
            b = self.buf.cpu().numpy()
        else:
            b = np.frombuffer(C.string_at(self.ptr, self.nb), np.uint8).copy()
        return b, b[: self.nb // 88 * 88].view(GROUP_DTYPE)

    def free(self):
        from netobserv_ebpf_agent_b200._lib import check, lib
        if self.kind == "pinned":
            check(lib().fa_host_free(self.p))
        elif hasattr(self, "p"):
            check(lib().fa_device_free(self.eng._h, self.p))


def check_placement(n, n_keys, mode, on_gpu, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, FA_E_INVAL, FA_OK, lib
    recs = gen_host(seed=2901, n=n, n_keys=n_keys, dist=1, t0=T0)
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        got = C.c_size_t(7)
        m = masks()["dst112_dport"]
        assert lib().fa_group_flows(eng._h, m.ctypes.data, None, 0, C.byref(got)) == FA_OK and got.value == 0   # empty engine
        eng.ingest(recs); rep.add("base", recs)
        want = group_rows(rep.state()[0], m)
        n_g = len(want)
        assert n_g > 2
        for kind in ("pageable", "pinned", "device"):
            for cap in (n_g, n_g + 5, n_g - 1):
                o = Out(eng, kind, cap, on_gpu)
                got.value = 7
                rc = lib().fa_group_flows(eng._h, m.ctypes.data, o.ptr, cap, C.byref(got))
                raw, rows = o.read()
                o.free()
                assert got.value == n_g, (kind, cap)
                if cap < n_g:
                    assert rc == FA_E_2BIG and (raw == 0xA5).all(), (kind, cap)     # nothing written
                else:
                    assert rc == FA_OK
                    assert_groups(rows[:n_g], want, f"{kind} cap={cap}")
                    assert (raw[n_g * 88:] == 0xA5).all()                             # nothing past the groups
        got.value = 7
        assert lib().fa_group_flows(eng._h, m.ctypes.data, None, 0, C.byref(got)) == FA_E_2BIG and got.value == n_g  # count
        out = np.zeros(n_g, fa.GROUP_DTYPE)
        for args in ((None, m.ctypes.data, out.ctypes.data, n_g, C.byref(got)), (eng._h, None, out.ctypes.data, n_g, C.byref(got)),
                     (eng._h, m.ctypes.data, out.ctypes.data, n_g, None), (eng._h, m.ctypes.data, None, 1, C.byref(got))):
            got.value = 7
            assert lib().fa_group_flows(*args) == FA_E_INVAL, args
            assert got.value == 0 or args[-1] is None
        assert_groups(eng.group_flows(m), want, "after the errors")


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_placement_emul(engine_emul, mode):
    check_placement(1_500, 400, mode, on_gpu=False, max_batch=256)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_placement_gpu(mode):
    check_placement(600_000, 200_000, mode, on_gpu=True, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 10. layout
PROBE = r'''
#include <stdio.h>
#include <stddef.h>
#include "flowagg.h"
#define P(f) printf(#f " %zu\n", offsetof(fa_flow_group, f))
int main(void) {
  printf("sizeof %zu\n", sizeof(fa_flow_group));
  P(key); P(flows); P(bytes); P(packets); P(start_mono_time_ts); P(end_mono_time_ts); P(flags); P(pad_);
  return 0;
}
'''


def test_group_layout_matches_dtype():
    from netobserv_ebpf_agent_b200 import GROUP_DTYPE
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(c, "w").write(PROBE)
        subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-o", exe, c, "-I" + os.path.join(ROOT, "include")], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = {k: int(v) for k, v in (ln.split() for ln in out.strip().splitlines())}
    want = {"sizeof": GROUP_DTYPE.itemsize}
    want.update({f: GROUP_DTYPE.fields[f][1] for f in GROUP_DTYPE.names})
    assert got == want


def test_group_mask():
    import netobserv_ebpf_agent_b200 as fa
    m = fa.group_mask(src_prefix=120, dst_prefix=100, src_port=True, proto=True, icmp=True)
    assert m[:15].tolist() == [0xFF] * 15 and m[15] == 0
    assert m[16:28].tolist() == [0xFF] * 12 and m[28] == 0xF0 and not m[29:32].any()
    assert m[32:34].tolist() == [0xFF, 0xFF] and not m[34:36].any() and m[36:39].tolist() == [0xFF] * 3 and m[39] == 0
    assert not fa.group_mask().any()
