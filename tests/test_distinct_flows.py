"""fa_distinct_flows: exact per-group distinct counts of a second key mask (port scans, fan-out, clients per service),
on the device, without evicting.

The expected side is numpy over the 40-byte keys of flow rows: np.unique over key & (G | D) (a void view, byte 39
cleared) gives the distinct (group, value) pairs, grouping those by & G and counting gives `distinct`, and np.unique over
key & G with counts gives `flows`.  The rows are the oracle's flows, or the fa_evict_ex rows taken right after the call.
Both sides are sorted by key and compared as 56-byte rows, bit for bit, for every mask pair of pairs().  Every case runs
on the engine emulation (`engine_emul`, a few thousand flows, CPU suite) and on the device (`gpu`, 10^5 to 2·10^6
flows)."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_adversarial_parity import key_families, table_slots
from test_dns_correlate import query, response
from test_expire_flows import Replay
from test_gpu_features import keys_of, make_add, make_dns
from test_group_flows import as_rows, as_rows_any, assert_groups, group_rows
from test_histogram_flows import PROM_NS, assert_hist, hist_rows
from test_pktdrop import make_drops

pytestmark = pytest.mark.timeout(1200)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0 = 1_000_000
U64_MAX = (1 << 64) - 1
CHANGED_BY_DISTINCT = ("kernel_launches", "d2h_bytes")
ROW = 56


# ---------------------------------------------------------------------------------------------------- mask pairs, expected side
def pairs():
    """name -> (group mask G, distinct mask D)."""
    import netobserv_ebpf_agent_b200 as fa
    gm = fa.group_mask
    ones = np.full(40, 0xFF, np.uint8)
    p = {"scan": (gm(src_prefix=128), gm(dst_port=True)),
         "fanout": (gm(src_prefix=128), gm(dst_prefix=128)),
         "clients": (gm(proto=True, dst_port=True), gm(src_prefix=128)),
         "dst120_src": (gm(dst_prefix=120), gm(src_prefix=128)),
         "zero_dst": (gm(), gm(dst_prefix=128)),
         "ones_ones": (ones, ones.copy()),
         "src120_zero": (gm(src_prefix=120), gm()),
         "src120_subset": (gm(src_prefix=120), gm(src_prefix=100))}
    g39, d39 = gm(src_prefix=124, proto=True), gm(dst_prefix=128, icmp=True)
    g39[39] = d39[39] = 0xFF
    p["byte39"] = (g39, d39)
    rng = np.random.default_rng(5151)
    for i in range(3):
        g, d = ((rng.random((40, 8)) < 0.12).astype(np.uint8) for _ in range(2))
        p[f"random{i}"] = (np.packbits(g, axis=1).reshape(40), np.packbits(d, axis=1).reshape(40))
    return p


def masked(keys, mask):
    k = keys & np.asarray(mask, np.uint8)[None, :]
    k[:, 39] = 0
    return np.ascontiguousarray(k).view("V40").ravel()


def distinct_rows(recs, g, d):
    """The expected fa_distinct_flows result (min_distinct = 0) for flow rows `recs` (n, 144)."""
    from netobserv_ebpf_agent_b200 import DISTINCT_DTYPE
    keys = as_rows(recs)[:, :O.ID]
    u = np.asarray(g, np.uint8) | np.asarray(d, np.uint8)
    pk = np.frombuffer(np.unique(masked(keys, u)).tobytes(), np.uint8).reshape(-1, 40)
    uk, distinct = np.unique(masked(pk, g), return_counts=True)
    fk, flows = np.unique(masked(keys, g), return_counts=True)
    assert np.array_equal(uk, fk)
    out = np.zeros(len(uk), DISTINCT_DTYPE)
    out["key"] = np.frombuffer(uk.tobytes(), np.uint8).reshape(-1, 40)
    out["flows"], out["distinct"] = flows, distinct
    return out


def sorted_rows(x):
    x = np.ascontiguousarray(x)
    r = x.view(np.uint8).reshape(-1, ROW)
    return r[np.argsort(np.ascontiguousarray(x["key"]).view("V40").ravel(), kind="stable")]


def assert_distinct(got, want, what=""):
    g, w = sorted_rows(got), sorted_rows(want)
    assert len(g) == len(w), (what, len(g), len(w))
    if not np.array_equal(g, w):
        bad = np.nonzero((g != w).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(g)} groups differ, first at {int(bad[0])}")


def check_pairs(eng, flows, what, which=None):
    """Every pair (or those named in `which`) against the flow rows `flows`, and the invariants against fa_group_flows:
    the same keys and flows as group_flows(G), and the distinct counts summing to the groups of group_flows(G | D)."""
    got = {}
    for name, (g, d) in pairs().items():
        if which is not None and name not in which:
            continue
        got[name] = r = eng.distinct_flows(g, d)
        assert_distinct(r, distinct_rows(flows, g, d), f"{what} / {name}")
        grp = eng.group_flows(g)
        assert len(grp) == len(r) and (r["distinct"] >= 1).all()
        assert np.array_equal(sorted_rows(r)[:, :48], np.ascontiguousarray(sorted_by_key(grp)).view(np.uint8).reshape(-1, 88)[:, :48])
        assert int(r["distinct"].sum()) == len(eng.group_flows(g | d))
    return got


def sorted_by_key(g):
    return g[np.argsort(np.ascontiguousarray(g["key"]).view("V40").ravel(), kind="stable")]


# ---------------------------------------------------------------------------------------------------- 1. oracle parity
def check_oracle(n, n_keys, mode, dist, varying, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=5101 + dist + 2 * varying + 4 * mode, n=n, n_keys=n_keys, dist=dist, varying=varying, t0=T0)
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        for part in np.array_split(recs, 2):
            eng.ingest(part)
            rep.add("base", part)
            flows = rep.state()[0]
            assert eng.live_flows() == len(flows)
            got = check_pairs(eng, flows, "oracle")
        ev = eng.evict_ex()
        assert len(ev[0]) == len(flows)
        for name, (g, d) in pairs().items():
            assert_distinct(got[name], distinct_rows(ev[0], g, d), f"eviction / {name}")


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


# ---------------------------------------------------------------------------------------------------- 2. crafted fan-out, 4. threshold
def addr(v6, host):
    """A 16-byte address: ::ffff:10.77.h.h or 2001:db8::h."""
    a = np.zeros(16, np.uint8)
    if v6:
        a[:4] = (0x20, 0x01, 0x0D, 0xB8)
        a[12:16] = np.frombuffer(int(host).to_bytes(4, "big"), np.uint8)
    else:
        a[10:12] = 0xFF
        a[12:16] = (10, 77, (host >> 8) & 0xFF, host & 0xFF)
    return a


def crafted_keys(ns):
    """For each N and address family: a source scanning N destination ports of one host (TCP), and a host fanning out
    to N peers on port 22.  -> (keys (m, 40), {(kind, v6, N): source address})."""
    keys, src = [], {}
    host = 1
    for n in ns:
        for v6 in (False, True):
            for kind in ("scan", "fanout"):
                s = addr(v6, host); host += 1
                k = np.zeros((n, 40), np.uint8)
                k[:, 0:16] = s
                if kind == "scan":
                    k[:, 16:32] = addr(v6, 60000)
                    port = 1 + np.arange(n, dtype=np.uint32)
                else:
                    k[:, 16:32] = np.stack([addr(v6, 100000 + i) for i in range(n)])
                    port = np.full(n, 22, np.uint32)
                k[:, 32:34] = np.frombuffer((np.full(n, 50000, ">u2")).tobytes(), np.uint8).reshape(n, 2)
                k[:, 34:36] = np.frombuffer(port.astype(">u2").tobytes(), np.uint8).reshape(n, 2)
                k[:, 36] = 6
                keys.append(k)
                src[(kind, v6, n)] = s
                host += 1
    return np.concatenate(keys), src


def check_crafted(n_bg, ns, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, FA_OK, lib
    bg = gen_host(seed=5201, n=n_bg, n_keys=n_bg // 2, dist=1, t0=T0)
    ck, src = crafted_keys(ns)
    fr = np.repeat(bg[:1], len(ck), axis=0)
    fr[:, :40] = ck
    recs = np.concatenate([bg, fr, fr[::7]])
    recs = recs[np.random.default_rng(5202).permutation(len(recs))]
    rep = Replay()
    rep.add("base", recs)
    flows = rep.state()[0]
    p = pairs()
    with fa.FlowAggEngine(2 * len(flows), max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.live_flows() == len(flows)
        got = check_pairs(eng, flows, "crafted", ("scan", "fanout", "clients", "zero_dst", "ones_ones"))
        for (kind, v6, n), s in src.items():
            r = got[kind]
            row = r[(r["key"][:, :16] == s).all(axis=1)]
            assert len(row) == 1 and row["distinct"][0] == n and row["flows"][0] == n, (kind, v6, n)
        # the threshold: the full result filtered, for every crafted N and the edges
        for name in ("scan", "fanout"):
            g, d = p[name]
            full = got[name]
            for t in sorted({0, 1, 2, U64_MAX} | {x for n in ns for x in (n, n + 1)} | {int(full["distinct"].max()) + 1}):
                want = full[full["distinct"] >= max(t, 1)]
                assert_distinct(eng.distinct_flows(g, d, min_distinct=t), want, f"{name} min_distinct={t}")
                cnt = C.c_size_t(7)
                assert lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, t, None, 0, C.byref(cnt)) == \
                    (FA_E_2BIG if len(want) else FA_OK)
                assert cnt.value == len(want)
                if len(want) > 1:                                     # FA_E_2BIG reports the passing count
                    out = np.full((len(want) - 1) * ROW, 0xA5, np.uint8)
                    assert lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, t, out.ctypes.data, len(want) - 1,
                                                   C.byref(cnt)) == FA_E_2BIG
                    assert cnt.value == len(want) and (out == 0xA5).all()
            assert len(eng.distinct_flows(g, d, min_distinct=int(full["distinct"].max()) + 1)) == 0
        ev = eng.evict_ex()
        for name in ("scan", "fanout"):
            assert_distinct(got[name], distinct_rows(ev[0], *p[name]), f"crafted, eviction / {name}")


def test_crafted_emul(engine_emul):
    check_crafted(2_000, (1, 31, 32, 33, 1024), max_batch=1_000)


@pytest.mark.gpu
def test_crafted_gpu():
    check_crafted(400_000, (1, 31, 32, 33, 1024, 65535), max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 5. colliding keys
def check_colliding(n_bg, max_batch):
    """Key families built against the group tables' size (both levels are sized from the live count with an all-ones
    group mask): the identical-premix and shared-low-32-bit families collide whatever the size, the chains share a home
    slot, and identical-premix keys meet in one warp round at both levels."""
    import netobserv_ebpf_agent_b200 as fa
    bg = gen_host(seed=5301, n=n_bg, n_keys=n_bg // 2, dist=1, t0=T0)
    rep0 = Replay()
    rep0.add("base", bg)
    live_guess = len(rep0.state()[0])
    fam = key_families(5302, table_slots(live_guess + 500), n_full=64, n_chain=300, n_way=32)
    fk = np.concatenate([fam["full"], fam["chain_last"], fam["chain_mid"], fam["way"], fam["elect"]])
    fr = np.repeat(bg[:1], len(fk), axis=0)
    fr[:, :40] = fk
    recs = np.concatenate([bg, fr, fr[::3]])
    recs = recs[np.random.default_rng(5303).permutation(len(recs))]
    rep = Replay()
    rep.add("base", recs)
    flows = rep.state()[0]
    ones, zero = np.full(40, 0xFF, np.uint8), fa.group_mask()
    coarse = fa.group_mask(src_prefix=128, dst_prefix=128, proto=True)
    with fa.FlowAggEngine(2 * len(flows), max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.live_flows() == len(flows)
        assert table_slots(len(flows)) == table_slots(live_guess + 500)
        for name, (g, d) in (("ones/ones", (ones, ones)), ("ones/zero", (ones, zero)), ("coarse/ones", (coarse, ones)),
                             ("zero/ones", (zero, ones))):
            assert_distinct(eng.distinct_flows(g, d), distinct_rows(flows, g, d), f"colliding / {name}")
        r = eng.distinct_flows(ones, zero)
        assert np.isin(np.ascontiguousarray(fk).view("V40").ravel(), np.ascontiguousarray(r["key"]).view("V40").ravel()).all()


def test_colliding_emul(engine_emul):
    check_colliding(2_000, max_batch=1_000)


@pytest.mark.gpu
def test_colliding_gpu():
    check_colliding(400_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 6. feature folds
def check_features(n, n_keys, max_batch):
    """Flows first seen through RTT, DNS or drop samples are live flows and count, in flows and in distinct."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(5401)
    recs = gen_host(seed=5401, n=n, n_keys=n_keys, dist=1, t0=T0)
    keys = np.concatenate([np.unique(recs[:, :40], axis=0), keys_of(5402, 64)])        # 64 feature-only flows
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
        check_pairs(eng, st[0], "features, oracle")
        eng.ingest_dns_packets(np.concatenate([query(1000, 7), response(5000, 7)]))
        got = {name: eng.distinct_flows(g, d) for name, (g, d) in pairs().items()}
        evicted = eng.evict_ex()
        assert len(evicted[0]) >= len(st[0])
        for name, (g, d) in pairs().items():
            assert_distinct(got[name], distinct_rows(evicted[0], g, d), f"features, eviction / {name}")


def test_features_emul(engine_emul):
    check_features(2_000, 500, max_batch=600)


@pytest.mark.gpu
def test_features_gpu():
    check_features(600_000, 150_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 7. KERNEL_MAP, full tables
def check_kernel_map(n, n_keys, max_entries, ringbuf, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=5501 + ringbuf, n=n, n_keys=n_keys, dist=1, t0=T0)
    v = recs.view(O.REC_DTYPE).reshape(-1)
    v["if_index"] = np.where(np.random.default_rng(5502).random(n) < 0.3, 7, 3)
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
        check_pairs(eng, flows, f"kmap ringbuf={ringbuf}")
    assert (rep.spilled if ringbuf else rep.fail_create)


@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_emul(engine_emul, ringbuf):
    check_kernel_map(3_000, 1_000, 300, ringbuf, max_batch=700)


@pytest.mark.gpu
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_gpu(ringbuf):
    check_kernel_map(600_000, 200_000, 50_000, ringbuf, max_batch=1 << 16)


def check_physically_full(max_entries, n, max_batch):
    """FA_F_NO_FULL_CUT with more distinct keys than slots: every slot of the flow table is live."""
    import netobserv_ebpf_agent_b200 as fa
    slots = table_slots(max_entries)
    recs = gen_host(seed=5601, n=n, n_keys=1 << 30, dist=0, t0=T0)
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NO_FULL_CUT, max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.stats()["spills"] > 0 and eng.live_flows() == slots
        got = {name: eng.distinct_flows(g, d) for name, (g, d) in pairs().items()}
        ev = eng.evict_ex()
        assert len(ev[0]) == slots
        for name, (g, d) in pairs().items():
            assert_distinct(got[name], distinct_rows(ev[0], g, d), f"full table / {name}")


def test_physically_full_emul(engine_emul):
    check_physically_full(700, 1_100, max_batch=600)                 # 1024 slots


@pytest.mark.gpu
def test_physically_full_gpu():
    check_physically_full(180_000, 600_000, max_batch=1 << 16)        # 2^18 slots


# ---------------------------------------------------------------------------------------------------- 8. non-blocking
def check_nonblocking_sequential(n, n_keys, mode):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=5701 + mode, n=n, n_keys=n_keys, dist=1, t0=T0)
    a, b = recs[: n // 2], recs[n // 2:]
    kmap = mode == fa.FA_MODE_KERNEL_MAP
    g, d = pairs()["zero_dst"]
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_NONBLOCKING_EVICT) as eng:
        eng.ingest(a)
        ra = Replay(kmap=kmap); ra.add("base", a)
        check_pairs(eng, ra.state()[0], "first window", ("zero_dst", "fanout", "clients"))
        assert len(eng.evict_ex()[0]) == len(ra.state()[0])
        assert len(eng.distinct_flows(g, d)) == 0                      # the retired table is not counted
        eng.ingest(b)
        rb = Replay(kmap=kmap); rb.add("base", b)
        check_pairs(eng, rb.state()[0], "second window")


def check_nonblocking_concurrent(n, n_keys, max_entries, max_batch, chunk):
    """An evictor thread against a thread that alternates ingest and distinct_flows: every call is consistent (an
    all-ones distinct mask gives distinct == flows; the window's distinct keys are its flows), and the generations,
    re-folded, equal the oracle's fold of the stream."""
    import netobserv_ebpf_agent_b200 as fa
    from test_nonblocking_evict import refold
    recs = gen_host(seed=5703, n=n, n_keys=n_keys, dist=1, t0=T0)
    out, stop = [], threading.Event()
    ones, zero, src = np.full(40, 0xFF, np.uint8), fa.group_mask(), fa.group_mask(src_prefix=120)
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
            if calls % 2 == 0:
                r = eng.distinct_flows(src, ones, cap=max_entries)
                assert (r["distinct"] == r["flows"]).all()
            else:
                r = eng.distinct_flows(zero, ones, cap=max_entries)
                assert len(r) <= 1 and (len(r) == 0 or 0 < r["distinct"][0] == r["flows"][0] <= max_entries)
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


# ---------------------------------------------------------------------------------------------------- 9. nothing changes
def check_nothing_changes(n, n_keys, max_batch):
    """With the sketch, RTT, DNS and the DNS correlation table in use: the stats (but launches and copies), the sketch,
    the pending DNS queries and a later eviction are those of a twin engine that never called it; fa_distinct_flows,
    fa_group_flows and fa_histogram_flows interleaved on one engine stay exact (so both group tables come back all
    zero), also after FA_E_2BIG and after the tables had to grow."""
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, lib
    from test_adversarial_parity import SKETCH_SEED
    rng = np.random.default_rng(5801)
    recs = gen_host(seed=5801, n=n, n_keys=n_keys, dist=1, t0=T0)
    small = recs[:300]
    keys = np.unique(recs[:, :40], axis=0)
    add, dns = make_add(rng, keys, n // 4), make_dns(rng, keys, n // 8)
    kw = dict(flags=fa.FA_F_ENABLE_SKETCH | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_RTT, cms_log2_width=12, cms_depth=4,
              hll_precision=10, sketch_seed=SKETCH_SEED, max_batch=max_batch)
    pkts = np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001)])     # one query stays pending
    p = pairs()
    src120 = fa.group_mask(src_prefix=120)
    with fa.FlowAggEngine(4 * n_keys, **kw) as eng, fa.FlowAggEngine(4 * n_keys, **kw) as ref:
        for x in (eng, ref):
            x.ingest(small); x.ingest_dns_packets(pkts)
        assert eng.live_flows() < 768                               # the first group tables have 1024 slots
        before = eng.stats()
        flows = ref.top_flows(ref.live_flows())[0]
        for name in ("fanout", "ones_ones", "zero_dst"):
            assert_distinct(eng.distinct_flows(*p[name]), distinct_rows(flows, *p[name]), f"small / {name}")
        after = eng.stats()
        for k in before:
            if k not in CHANGED_BY_DISTINCT:
                assert after[k] == before[k], k
        assert after["kernel_launches"] > before["kernel_launches"] and after["d2h_bytes"] > before["d2h_bytes"]
        for x in (eng, ref):
            x.ingest(recs); x.ingest_additional(add); x.ingest_dns(dns)
        blocks = ref.top_flows(ref.live_flows())
        flows = blocks[0]
        assert len(flows) > 768                                     # the group tables grow
        g, d = p["fanout"]
        n_want = len(distinct_rows(flows, g, d))
        out = np.full((n_want - 1) * ROW, 0xA5, np.uint8)
        got = C.c_size_t(0)
        assert lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, 0, out.ctypes.data, n_want - 1, C.byref(got)) == FA_E_2BIG
        assert got.value == n_want and (out == 0xA5).all()
        for name in ("clients", "ones_ones", "zero_dst", "scan", "random1", "byte39"):      # interleaved, different masks
            assert_distinct(eng.distinct_flows(*p[name]), distinct_rows(flows, *p[name]), f"in a row / {name}")
            assert_groups(eng.group_flows(p[name][0]), group_rows(flows, p[name][0]), f"group_flows after / {name}")
            assert_hist(eng.histogram_flows(src120, fa.FA_HIST_RTT, PROM_NS), hist_rows(blocks, src120, "rtt", PROM_NS),
                        f"histogram_flows after / {name}")
        s_eng, s_ref = eng.stats(), ref.stats()
        assert s_ref["dns_queries_pending"] == 1
        for k in s_ref:
            if k not in CHANGED_BY_DISTINCT:
                assert s_eng[k] == s_ref[k], k
        for a, b in zip(eng.sketch_export(12, 4, 10), ref.sketch_export(12, 4, 10)):
            assert np.array_equal(a, b)
        assert eng.hll_estimate() == ref.hll_estimate()
        a, b = eng.evict_ex(), ref.evict_ex()
        for x, y in zip(a, b):
            x, y = as_rows_any(x), as_rows_any(y)
            assert np.array_equal(x[O.sort_perm(a[0])], y[O.sort_perm(b[0])])
        assert len(eng.distinct_flows(*p["zero_dst"])) == 0


def test_nothing_changes_emul(engine_emul):
    check_nothing_changes(12_000, 4_000, 2_000)


@pytest.mark.gpu
def test_nothing_changes_gpu():
    check_nothing_changes(800_000, 200_000, 1 << 16)


# ---------------------------------------------------------------------------------------------------- 10. placement, errors
class Out:
    """n_rows x 56 B of output filled with 0xA5: host pageable, pinned (fa_host_alloc) or device memory (a CUDA tensor
    on the GPU, fa_device_alloc memory on the emulation), at byte offset `shift`."""

    def __init__(self, eng, kind, n_rows, on_gpu, shift=0):
        from netobserv_ebpf_agent_b200._lib import check, lib
        self.eng, self.kind, self.nb, self.shift = eng, kind, max(n_rows, 1) * ROW, shift
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
            self.buf = torch.full((self.nb + shift,), 0xA5, dtype=torch.uint8, device="cuda")
            self.ptr = self.buf.data_ptr() + shift
        else:
            p = C.c_void_p()
            check(lib().fa_device_alloc(eng._h, self.nb + shift, C.byref(p)))
            C.memset(p.value, 0xA5, self.nb + shift)
            self.p, self.ptr = p, p.value + shift

    def read(self):
        from netobserv_ebpf_agent_b200 import DISTINCT_DTYPE
        if self.kind == "pageable":
            b = self.buf.copy()
        elif hasattr(self, "buf"):
            b = self.buf.cpu().numpy()[self.shift:]
        else:
            b = np.frombuffer(C.string_at(self.ptr, self.nb), np.uint8).copy()
        return b, b[: self.nb // ROW * ROW].view(DISTINCT_DTYPE)

    def free(self):
        from netobserv_ebpf_agent_b200._lib import check, lib
        if self.kind == "pinned":
            check(lib().fa_host_free(self.p))
        elif hasattr(self, "p"):
            check(lib().fa_device_free(self.eng._h, self.p))


def check_placement(n, n_keys, mode, on_gpu, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, FA_E_INVAL, FA_OK, lib
    recs = gen_host(seed=5901, n=n, n_keys=n_keys, dist=1, t0=T0)
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    g, d = pairs()["clients"]
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        got = C.c_size_t(7)
        assert lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, 0, None, 0, C.byref(got)) == FA_OK and got.value == 0
        eng.ingest(recs); rep.add("base", recs)
        want = distinct_rows(rep.state()[0], g, d)
        n_g = len(want)
        assert n_g > 2
        for kind in ("pageable", "pinned", "device"):
            for cap in (n_g, n_g + 5, n_g - 1):
                o = Out(eng, kind, cap, on_gpu)
                got.value = 7
                rc = lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, 0, o.ptr, cap, C.byref(got))
                raw, rows = o.read()
                o.free()
                assert got.value == n_g, (kind, cap)
                if cap < n_g:
                    assert rc == FA_E_2BIG and (raw == 0xA5).all(), (kind, cap)     # nothing written
                else:
                    assert rc == FA_OK
                    assert_distinct(rows[:n_g], want, f"{kind} cap={cap}")
                    assert (raw[n_g * ROW:] == 0xA5).all()                            # nothing past the groups
        got.value = 7
        assert lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, 0, None, 0, C.byref(got)) == FA_E_2BIG
        assert got.value == n_g                                                        # a count query
        o = Out(eng, "device", n_g, on_gpu, shift=4)
        got.value = 7
        assert lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, 0, o.ptr, n_g, C.byref(got)) == FA_E_INVAL
        raw, _ = o.read()
        o.free()
        assert got.value == 0 and (raw == 0xA5).all()
        out = np.zeros(n_g, fa.DISTINCT_DTYPE)
        gp, dp, op = g.ctypes.data, d.ctypes.data, out.ctypes.data
        for args in ((None, gp, dp, 0, op, n_g, C.byref(got)), (eng._h, None, dp, 0, op, n_g, C.byref(got)),
                     (eng._h, gp, None, 0, op, n_g, C.byref(got)), (eng._h, gp, dp, 0, op, n_g, None),
                     (eng._h, gp, dp, 0, None, 1, C.byref(got))):
            got.value = 7
            assert lib().fa_distinct_flows(*args) == FA_E_INVAL, args
            assert got.value == 0 or args[-1] is None
        assert_distinct(eng.distinct_flows(g, d), want, "after the errors")


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_placement_emul(engine_emul, mode):
    check_placement(1_500, 400, mode, on_gpu=False, max_batch=256)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_placement_gpu(mode):
    check_placement(600_000, 200_000, mode, on_gpu=True, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 11. layout
PROBE = r'''
#include <stdio.h>
#include <stddef.h>
#include "flowagg.h"
int main(void) {
  printf("sizeof %zu\nkey %zu\nflows %zu\ndistinct %zu\n", sizeof(fa_distinct_group), offsetof(fa_distinct_group, key),
         offsetof(fa_distinct_group, flows), offsetof(fa_distinct_group, distinct));
  return 0;
}
'''


def test_distinct_layout_matches_dtype():
    from netobserv_ebpf_agent_b200 import DISTINCT_DTYPE
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(c, "w").write(PROBE)
        subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-o", exe, c, "-I" + os.path.join(ROOT, "include")], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = {k: int(v) for k, v in (ln.split() for ln in out.strip().splitlines())}
    want = {"sizeof": DISTINCT_DTYPE.itemsize}
    want.update({f: DISTINCT_DTYPE.fields[f][1] for f in DISTINCT_DTYPE.names})
    assert got == want == {"sizeof": 56, "key": 0, "flows": 40, "distinct": 48}
