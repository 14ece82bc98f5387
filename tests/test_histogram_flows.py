"""fa_histogram_flows: exact per-group histograms of flow size, duration, RTT and DNS latency over the live flows, on
the device, without evicting.

The expected side is numpy over flow rows: the groups of test_group_flows (key bytes ANDed with the mask, byte 39
cleared, np.unique over a void view), each flow's value under the decoder's presence rules, the bucket by
np.searchsorted(bounds, v, side="left") (Prometheus `le`: v <= bounds[b]), np.add.at for flows / count / sum (uint64,
wrapping) / bucket counts, np.minimum.at / np.maximum.at for min / max.  The rows are the oracle's flows, or the
fa_evict_ex rows taken right after the call.  Both sides are sorted by key and compared bit for bit.  Every case runs on
the engine emulation (`engine_emul`, a few thousand flows, CPU suite) and on the device (`gpu`, 10^5 to 2·10^6 flows)."""
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
from test_group_flows import Out, as_rows, as_rows_any, assert_groups, by_key, group_rows, masks

pytestmark = pytest.mark.timeout(1200)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0 = 1_000_000
U64_MAX = (1 << 64) - 1
CHANGED_BY_HISTOGRAM = ("kernel_launches", "d2h_bytes")
BASE_VALUES = ("bytes", "packets", "duration")


def hist_consts():
    import netobserv_ebpf_agent_b200 as fa
    return {"bytes": fa.FA_HIST_BYTES, "packets": fa.FA_HIST_PACKETS, "duration": fa.FA_HIST_DURATION,
            "rtt": fa.FA_HIST_RTT, "dns": fa.FA_HIST_DNS_LATENCY}


# ---------------------------------------------------------------------------------------------------- expected side
def flow_values(blocks, value):
    """(values u64, has) of every flow row: blocks = the evict_ex blocks (records, dns, additional, ...) or (records,)."""
    v = as_rows(blocks[0]).view(O.REC_DTYPE).reshape(-1)
    n = len(v)
    if value == "bytes":
        return v["bytes"].astype(np.uint64), np.ones(n, bool)
    if value == "packets":
        return v["packets"].astype(np.uint64), np.ones(n, bool)
    if value == "duration":
        s, e = v["start"].astype(np.uint64), v["end"].astype(np.uint64)
        return np.where(e >= s, e - s, np.uint64(0)).astype(np.uint64), s != 0
    if value == "rtt":                                   # additional.flow_rtt, exported only when != 0
        rtt = np.ascontiguousarray(as_rows_any(blocks[2])).view(O.ADD_DTYPE).reshape(-1)["rtt"].astype(np.uint64)
        return rtt, rtt != 0
    d = np.ascontiguousarray(as_rows_any(blocks[1])).view(O.DNS_DTYPE).reshape(-1)   # dns.latency, only with dns.id != 0
    return d["latency"].astype(np.uint64), d["id"] != 0


def hist_rows(blocks, mask, value, bounds):
    """The expected fa_histogram_flows result for flow rows `blocks`."""
    import netobserv_ebpf_agent_b200 as fa
    bounds = np.asarray(bounds, np.uint64)
    r = as_rows(blocks[0])
    k = r[:, :O.ID] & np.asarray(mask, np.uint8)[None, :]
    k[:, 39] = 0
    uk, inv = np.unique(np.ascontiguousarray(k).view("V40").ravel(), return_inverse=True)
    inv = inv.ravel()
    g = len(uk)
    out = np.zeros(g, fa.hist_dtype(len(bounds)))
    out["key"] = np.frombuffer(uk.tobytes(), np.uint8).reshape(-1, 40)
    flows = np.zeros(g, np.uint64)
    np.add.at(flows, inv, np.uint64(1))
    out["flows"] = flows
    vals, has = flow_values(blocks, value)
    iv, x = inv[has], vals[has]
    cnt, sm, hi = np.zeros(g, np.uint64), np.zeros(g, np.uint64), np.zeros(g, np.uint64)
    lo = np.full(g, U64_MAX, np.uint64)
    np.add.at(cnt, iv, np.uint64(1))
    np.add.at(sm, iv, x)                                 # wraps mod 2^64
    np.minimum.at(lo, iv, x)
    np.maximum.at(hi, iv, x)
    counts = np.zeros((g, len(bounds) + 1), np.uint64)
    np.add.at(counts, (iv, np.searchsorted(bounds, x, side="left")), np.uint64(1))
    out["count"], out["sum"], out["max"], out["counts"] = cnt, sm, hi, counts
    out["min"] = np.where(cnt > 0, lo, np.uint64(0))
    return out


def assert_hist(got, want, what=""):
    w = want.dtype.itemsize
    assert got.dtype.itemsize == w, (what, got.dtype, want.dtype)
    g = by_key(got).view(np.uint8).reshape(-1, w)
    x = by_key(want).view(np.uint8).reshape(-1, w)
    assert len(g) == len(x), (what, len(g), len(x))
    if not np.array_equal(g, x):
        bad = np.nonzero((g != x).any(axis=1))[0]
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {len(g)} rows differ, first at {i}:\n got  {by_key(got)[i]}\n want {by_key(want)[i]}")


POW2 = np.array([1 << i for i in range(63)], np.uint64)                                        # 2^0 .. 2^62
PROM_NS = np.array([int(s * 1e9) for s in (1e-4, 2.5e-4, 5e-4, 1e-3, 2.5e-3, 5e-3, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5,
                                            1, 2.5, 5, 10)], np.uint64)                         # 100 us .. 10 s


def bound_sets(blocks, value):
    """name -> bounds: powers of two, a Prometheus-style ns set, one bound, bounds placed on values of the data (so
    that <= and < differ), and the same with a last bound of 2^64 - 1."""
    vals, has = flow_values(blocks, value)
    u = np.unique(vals[has]) if has.any() else np.array([5], np.uint64)
    on = np.unique(u[np.linspace(0, len(u) - 1, min(len(u), 40)).astype(np.int64)])
    return {"pow2": POW2, "prom": PROM_NS, "one": u[len(u) // 2: len(u) // 2 + 1], "on_data": on,
            "on_data_top": np.unique(np.append(on[:62], np.uint64(U64_MAX)))}


def check_values(eng, blocks, what, values=BASE_VALUES, which=None):
    """Every value of `values` over every mask (or those named in `which`), the bound sets in rotation, and every bound
    set for two masks."""
    c = hist_consts()
    ms = masks()
    for vi, value in enumerate(values):
        sets = bound_sets(blocks, value)
        names = list(sets)
        for mi, (mname, m) in enumerate(ms.items()):
            if which is not None and mname not in which:
                continue
            chosen = names if mname in ("src120", "ones") else [names[(mi + vi) % len(names)]]
            for bname in chosen:
                got = eng.histogram_flows(m, c[value], sets[bname])
                assert_hist(got, hist_rows(blocks, m, value, sets[bname]), f"{what} / {value} / {mname} / {bname}")


# ---------------------------------------------------------------------------------------------------- 1. oracle parity
def check_oracle(n, n_keys, mode, dist, varying, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=3101 + dist + 2 * varying + 4 * mode, n=n, n_keys=n_keys, dist=dist, varying=varying, t0=T0)
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        for i, part in enumerate(np.array_split(recs, 2)):
            eng.ingest(part)
            rep.add("base", part)
            st = rep.state()
            assert eng.live_flows() == len(st[0])
            check_values(eng, st[:1], f"oracle, part {i}", which=("zero", "src120", "ones") if i == 0 else None)
        ev = eng.evict_ex()
        assert len(ev[0]) == len(st[0])


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


# ---------------------------------------------------------------------------------------------------- 2. feature folds
def check_features(n, n_keys, mode, max_batch):
    """RTT and DNS latency (and duration, whose start / end the feature lines patch) against the fa_evict_ex rows taken
    right after the calls, and against the oracle before them.  Feature-only flows; flows whose additional samples all
    have rtt 0 (IPsec only); flows whose DNS samples all have id 0 and an errno; DNS latency from
    fa_ingest_dns_packets (a matched query and an unanswered response)."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(3201 + mode)
    recs = gen_host(seed=3201 + mode, n=n, n_keys=n_keys, dist=1, t0=T0)
    base_keys = np.unique(recs[:, :40], axis=0)
    only = keys_of(3202, 96)                                            # feature-only flows
    keys = np.concatenate([base_keys, only])
    add, dns = make_add(rng, keys, n // 4), make_dns(rng, keys, n // 8)
    ipsec = make_add(rng, np.concatenate([base_keys[:40], only[:16]]), 200)
    ipsec["add"]["rtt"] = 0
    ipsec["add"]["ipsec_ret"] = rng.integers(1, 4, len(ipsec))
    errno = make_dns(rng, np.concatenate([base_keys[40:80], only[16:32]]), 200)
    errno["dns"]["id"] = 0
    errno["dns"]["errno"] = rng.integers(1, 100, len(errno))
    errno_keys = np.ascontiguousarray(errno["id"]).view("V40").ravel()
    add = add[~np.isin(np.ascontiguousarray(add["id"]).view("V40").ravel(), np.ascontiguousarray(ipsec["id"]).view("V40").ravel())]
    dns = dns[~np.isin(np.ascontiguousarray(dns["id"]).view("V40").ravel(), errno_keys)]
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=flags, max_batch=max_batch) as eng:
        for kind, x in (("add", add[: len(add) // 2]), ("add", ipsec), ("base", recs), ("dns", dns), ("dns", errno),
                        ("add", add[len(add) // 2:])):
            {"add": eng.ingest_additional, "base": eng.ingest, "dns": eng.ingest_dns}[kind](x)
            rep.add(kind, x)
        if mode == fa.FA_MODE_ACCOUNTER:                                    # the replay folds features in this mode
            st = rep.state()
            check_values(eng, st, "features, oracle", values=("rtt", "dns", "duration"))
        eng.ingest_dns_packets(np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001),
                                               response(9000, 9, sport=40001), response(9500, 11, sport=40002)]))
        c = hist_consts()
        got = {}
        for value in ("rtt", "dns", "duration", "bytes"):
            for mname in ("zero", "src120", "ones", "proto_dport"):
                got[value, mname] = eng.histogram_flows(masks()[mname], c[value], PROM_NS if value != "bytes" else POW2)
        evicted = eng.evict_ex()
        pres = evicted[5]
        assert (pres == 0).any() and (pres & 1).any() and (pres & 2).any()
        assert ((pres & 2) != 0).sum() > flow_values(evicted, "rtt")[1].sum() > 0     # IPsec-only samples: a block, no RTT
        assert ((pres & 1) != 0).sum() > flow_values(evicted, "dns")[1].sum() > 0     # errno-only samples: a block, no id
        v = as_rows(evicted[0]).view(O.REC_DTYPE).reshape(-1)
        assert ((pres != 0) & (v["bytes"] == 0)).any()                                  # feature-only flows
        for (value, mname), g in got.items():
            want = hist_rows(evicted, masks()[mname], value, PROM_NS if value != "bytes" else POW2)
            assert_hist(g, want, f"features, eviction / {value} / {mname}")
        d = as_rows_any(evicted[1]).view(O.DNS_DTYPE).reshape(-1)
        assert ((d["id"] == 7) & (d["latency"] == 4000)).any()              # the packet-correlated sample is counted


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_features_emul(engine_emul, mode):
    check_features(2_000, 500, mode, max_batch=600)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_features_gpu(mode):
    check_features(600_000, 150_000, mode, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 3. wrap
def check_wrap(n, n_keys, max_batch):
    """Pre-aggregated records at uptime scale: the byte sum of the one-group mask wraps mod 2^64, packet values sit
    near 2^32, durations cross 2^32 boundaries."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(3301)
    recs = pre_aggregate(uptime_times(gen_host(seed=3301, n=n, n_keys=n_keys, dist=1), rng), rng)
    rep = Replay()
    rep.add("base", recs)
    st = rep.state()
    v = as_rows(st[0]).view(O.REC_DTYPE).reshape(-1)
    assert int(v["bytes"].astype(object).sum()) >= 1 << 64 and int(v["packets"].max()) > 0xFFFF0000
    top = np.array([1 << 32, (1 << 63) + 5, U64_MAX - 0x1000, U64_MAX], np.uint64)
    c = hist_consts()
    with fa.FlowAggEngine(2 * n_keys, max_batch=max_batch) as eng:
        eng.ingest(recs)
        check_values(eng, st[:1], "wrap")
        for value in ("bytes", "packets"):
            for mname in ("zero", "src120"):
                got = eng.histogram_flows(masks()[mname], c[value], top)
                assert_hist(got, hist_rows(st[:1], masks()[mname], value, top), f"wrap / {value} / {mname} / top")
        one = eng.histogram_flows(masks()["zero"], c["bytes"], top)
        assert len(one) == 1 and one["count"][0] == len(st[0])
        assert int(one["sum"][0]) == int(v["bytes"].astype(object).sum()) % (1 << 64)


def test_wrap_emul(engine_emul):
    check_wrap(3_000, 800, max_batch=700)


@pytest.mark.gpu
def test_wrap_gpu():
    check_wrap(800_000, 200_000, max_batch=1 << 17)


# ---------------------------------------------------------------------------------------------------- 4. colliding keys
def check_colliding(n_bg, max_batch):
    """Key families built against the group table's size (test_group_flows): identical-premix keys are distinct groups
    under the all-ones mask and sit in neighbouring flow-table slots, so they meet in one warp round."""
    import netobserv_ebpf_agent_b200 as fa
    bg = gen_host(seed=3401, n=n_bg, n_keys=n_bg // 2, dist=1, t0=T0)
    rep0 = Replay()
    rep0.add("base", bg)
    live_guess = len(rep0.state()[0])
    fam = key_families(3402, table_slots(live_guess + 500), n_full=64, n_chain=300, n_way=32)
    fk = np.concatenate([fam["full"], fam["chain_last"], fam["chain_mid"], fam["way"], fam["elect"]])
    fr = np.repeat(bg[:1], len(fk), axis=0)
    fr[:, :40] = fk
    fr.view(O.REC_DTYPE).reshape(-1)["bytes"] = np.arange(1, len(fk) + 1, dtype=np.uint64) << np.uint64(20)
    recs = np.concatenate([bg, fr, fr[::3]])
    recs = recs[np.random.default_rng(3403).permutation(len(recs))]
    rep = Replay()
    rep.add("base", recs)
    st = rep.state()
    c = hist_consts()
    with fa.FlowAggEngine(2 * len(st[0]), max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.live_flows() == len(st[0])
        assert table_slots(len(st[0])) == table_slots(live_guess + 500)
        coarse = fa.group_mask(src_prefix=128, dst_prefix=128, proto=True)
        for name, m in (("ones", masks()["ones"]), ("coarse", coarse)):
            for value in ("bytes", "duration"):
                got = eng.histogram_flows(m, c[value], POW2)
                assert_hist(got, hist_rows(st[:1], m, value, POW2), f"colliding / {name} / {value}")
        got = eng.histogram_flows(masks()["ones"], c["bytes"], POW2)
        full = np.isin(np.ascontiguousarray(got["key"]).view("V40").ravel(), np.ascontiguousarray(fam["full"]).view("V40").ravel())
        assert full.sum() == len(fam["full"]) and (got["flows"][full] == 1).all()


def test_colliding_emul(engine_emul):
    check_colliding(2_000, max_batch=1_000)


@pytest.mark.gpu
def test_colliding_gpu():
    check_colliding(400_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 5. KERNEL_MAP
def check_kernel_map(n, n_keys, max_entries, ringbuf, max_batch):
    """Packets on a second interface; max_entries below the key count: the map fills, and with the fallback ring the
    records that did not enter are not binned."""
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=3501 + ringbuf, n=n, n_keys=n_keys, dist=1, t0=T0)
    v = recs.view(O.REC_DTYPE).reshape(-1)
    v["if_index"] = np.where(np.random.default_rng(3502).random(n) < 0.3, 7, 3)
    rep = Replay(kmap=True, max_entries=max_entries, ringbuf=ringbuf)
    with fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=fa.FA_F_RINGBUF_FALLBACK if ringbuf else 0,
                          max_batch=max_batch) as eng:
        for part in np.array_split(recs, 2):
            eng.ingest(part)
            rep.add("base", part)
        st = rep.state()
        assert eng.live_flows() == len(st[0]) == max_entries
        if ringbuf:
            assert len(eng.read_spilled()) > 0
        check_values(eng, st[:1], f"kmap ringbuf={ringbuf}")
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


# ---------------------------------------------------------------------------------------------------- 6. full table
def check_physically_full(max_entries, n, max_batch):
    """FA_F_NO_FULL_CUT with more distinct keys than slots: every slot of the flow table is live."""
    import netobserv_ebpf_agent_b200 as fa
    slots = table_slots(max_entries)
    recs = gen_host(seed=3601, n=n, n_keys=1 << 30, dist=0, t0=T0)
    c = hist_consts()
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NO_FULL_CUT, max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.stats()["spills"] > 0 and eng.live_flows() == slots
        got = {(v, name): eng.histogram_flows(m, c[v], POW2) for v in ("bytes", "duration") for name, m in masks().items()}
        ev = eng.evict_ex()
        assert len(ev[0]) == slots
        for (v, name), g in got.items():
            assert_hist(g, hist_rows(ev, masks()[name], v, POW2), f"full table / {v} / {name}")


def test_physically_full_emul(engine_emul):
    check_physically_full(700, 1_100, max_batch=600)                 # 1024 slots


@pytest.mark.gpu
def test_physically_full_gpu():
    check_physically_full(180_000, 600_000, max_batch=1 << 16)        # 2^18 slots


# ---------------------------------------------------------------------------------------------------- 7. non-blocking
def check_nonblocking_sequential(n, n_keys, mode):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=3701 + mode, n=n, n_keys=n_keys, dist=1, t0=T0)
    a, b = recs[: n // 2], recs[n // 2:]
    kmap = mode == fa.FA_MODE_KERNEL_MAP
    c = hist_consts()
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_NONBLOCKING_EVICT) as eng:
        eng.ingest(a)
        ra = Replay(kmap=kmap); ra.add("base", a)
        check_values(eng, ra.state()[:1], "first window", which=("zero", "src120", "ones"))
        first = eng.evict_ex()
        assert len(first[0]) == len(ra.state()[0])
        assert len(eng.histogram_flows(masks()["zero"], c["bytes"], POW2)) == 0     # the retired table is not binned
        eng.ingest(b)
        rb = Replay(kmap=kmap); rb.add("base", b)
        check_values(eng, rb.state()[:1], "second window")


def check_nonblocking_concurrent(n, n_keys, max_entries, max_batch, chunk):
    """An evictor thread against a thread that alternates ingest and histogram_flows: every call is consistent (per
    group, the bucket counts sum to count; the one-group mask's count is the live flows it saw), and the generations,
    re-folded, equal the oracle's fold of the stream."""
    import netobserv_ebpf_agent_b200 as fa
    from test_nonblocking_evict import refold
    recs = gen_host(seed=3703, n=n, n_keys=n_keys, dist=1, t0=T0)
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
            g = eng.histogram_flows(ones if calls % 2 == 0 else zero, fa.FA_HIST_BYTES, POW2, cap=max_entries)
            assert (g["counts"].sum(axis=1) == g["count"]).all() and (g["count"] == g["flows"]).all()
            assert ((g["min"] <= g["max"]) & (g["min"] > 0)).all()
            if calls % 2 == 0:
                assert (g["flows"] == 1).all() and (g["sum"] == g["min"]).all()
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


# ---------------------------------------------------------------------------------------------------- 8. nothing changes
def check_nothing_changes(n, n_keys, max_batch):
    """With the sketch, RTT, DNS and the DNS correlation table in use: the stats (but launches and copies), the
    sketch, the pending DNS queries and a later eviction are those of a twin engine that never called it; a
    fa_group_flows call after it returns what one before it did; two calls in a row give identical rows; a call after
    FA_E_2BIG and one after the group table had to grow are exact."""
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, lib
    from test_adversarial_parity import SKETCH_SEED
    rng = np.random.default_rng(3801)
    recs = gen_host(seed=3801, n=n, n_keys=n_keys, dist=1, t0=T0)
    small = recs[:300]
    keys = np.unique(recs[:, :40], axis=0)
    add, dns = make_add(rng, keys, n // 4), make_dns(rng, keys, n // 8)
    kw = dict(flags=fa.FA_F_ENABLE_SKETCH | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_RTT, cms_log2_width=12, cms_depth=4,
              hll_precision=10, sketch_seed=SKETCH_SEED, max_batch=max_batch)
    pkts = np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001)])     # one query stays pending
    ms, c = masks(), hist_consts()
    with fa.FlowAggEngine(4 * n_keys, **kw) as eng, fa.FlowAggEngine(4 * n_keys, **kw) as ref:
        for x in (eng, ref):
            x.ingest(small); x.ingest_dns_packets(pkts)
        assert eng.live_flows() < 768                               # the first group table has 1024 slots
        before = eng.stats()
        g0 = eng.group_flows(ms["src120"])
        h1 = eng.histogram_flows(ms["src120"], c["duration"], PROM_NS)
        h2 = eng.histogram_flows(ms["src120"], c["duration"], PROM_NS)
        assert by_key(h1).tobytes() == by_key(h2).tobytes()         # identical rows (in unspecified order)
        assert_groups(eng.group_flows(ms["src120"]), g0, "group_flows after histogram_flows")
        after = eng.stats()
        for k in before:
            if k not in CHANGED_BY_HISTOGRAM:
                assert after[k] == before[k], k
        assert after["kernel_launches"] > before["kernel_launches"] and after["d2h_bytes"] > before["d2h_bytes"]
        for x in (eng, ref):
            x.ingest(recs); x.ingest_additional(add); x.ingest_dns(dns)
        blocks = ref.top_flows(ref.live_flows())
        assert len(blocks[0]) > 768                                 # the group table grows
        m = ms["src120"]
        n_want = len(group_rows(blocks[0], m))
        row = fa.hist_dtype(len(PROM_NS)).itemsize
        out = np.full((n_want - 1) * row, 0xA5, np.uint8)
        got = C.c_size_t(0)
        b = np.ascontiguousarray(PROM_NS)
        assert lib().fa_histogram_flows(eng._h, m.ctypes.data, c["rtt"], b.ctypes.data, len(b), out.ctypes.data, n_want - 1,
                                        C.byref(got)) == FA_E_2BIG
        assert got.value == n_want and (out == 0xA5).all()
        g_before = eng.group_flows(ms["proto_dport"])
        for name in ("proto_dport", "ones", "zero", "src120", "random1"):       # calls in a row, different masks
            for value in ("rtt", "dns", "bytes"):
                assert_hist(eng.histogram_flows(ms[name], c[value], PROM_NS), hist_rows(blocks, ms[name], value, PROM_NS),
                            f"in a row / {name} / {value}")
        assert_groups(eng.group_flows(ms["proto_dport"]), g_before, "group_flows after the calls")
        s_eng, s_ref = eng.stats(), ref.stats()
        assert s_ref["dns_queries_pending"] == 1
        for k in s_ref:
            if k not in CHANGED_BY_HISTOGRAM:
                assert s_eng[k] == s_ref[k], k
        for a, b in zip(eng.sketch_export(12, 4, 10), ref.sketch_export(12, 4, 10)):
            assert np.array_equal(a, b)
        assert eng.hll_estimate() == ref.hll_estimate()
        a, b = eng.evict_ex(), ref.evict_ex()
        for x, y in zip(a, b):
            x, y = as_rows_any(x), as_rows_any(y)
            assert np.array_equal(x[O.sort_perm(a[0])], y[O.sort_perm(b[0])])
        assert len(eng.histogram_flows(ms["zero"], c["bytes"], POW2)) == 0


def test_nothing_changes_emul(engine_emul):
    check_nothing_changes(12_000, 4_000, 2_000)


@pytest.mark.gpu
def test_nothing_changes_gpu():
    check_nothing_changes(800_000, 200_000, 1 << 16)


# ---------------------------------------------------------------------------------------------------- 9. placement, errors
def check_placement(n, n_keys, mode, on_gpu, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, FA_E_INVAL, FA_OK, lib
    recs = gen_host(seed=3901, n=n, n_keys=n_keys, dist=1, t0=T0)
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    bounds = np.ascontiguousarray(PROM_NS)
    nb = len(bounds)
    row = fa.hist_dtype(nb).itemsize
    assert row == 80 + 8 * (nb + 1)
    B = bounds.ctypes.data
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        got = C.c_size_t(7)
        m = masks()["dst112_dport"]
        assert lib().fa_histogram_flows(eng._h, m.ctypes.data, fa.FA_HIST_DURATION, B, nb, None, 0, C.byref(got)) == FA_OK
        assert got.value == 0                                                      # empty engine
        eng.ingest(recs); rep.add("base", recs)
        want = hist_rows(rep.state()[:1], m, "duration", bounds)
        n_g = len(want)
        assert n_g > 2
        for kind in ("pageable", "pinned", "device"):
            for cap in (n_g, n_g + 5, n_g - 1):
                o = Out(eng, kind, cap * row // 88 + 1, on_gpu)                    # Out counts 88-byte rows
                got.value = 7
                rc = lib().fa_histogram_flows(eng._h, m.ctypes.data, fa.FA_HIST_DURATION, B, nb, o.ptr, cap, C.byref(got))
                raw, _ = o.read()
                o.free()
                assert got.value == n_g, (kind, cap)
                if cap < n_g:
                    assert rc == FA_E_2BIG and (raw == 0xA5).all(), (kind, cap)     # nothing written
                else:
                    assert rc == FA_OK
                    assert_hist(raw[: n_g * row].view(fa.hist_dtype(nb)), want, f"{kind} cap={cap}")
                    assert (raw[n_g * row:] == 0xA5).all()                           # nothing past the rows
        got.value = 7
        assert lib().fa_histogram_flows(eng._h, m.ctypes.data, fa.FA_HIST_DURATION, B, nb, None, 0, C.byref(got)) == FA_E_2BIG
        assert got.value == n_g                                                     # a count query
        out = np.zeros(n_g, fa.hist_dtype(nb))
        O_ = out.ctypes.data
        flat = np.array([5, 5], np.uint64)
        down = np.array([9, 3], np.uint64)
        many = np.arange(1, 65, dtype=np.uint64)
        bad = [(None, m.ctypes.data, 0, B, nb, O_, n_g), (eng._h, None, 0, B, nb, O_, n_g), (eng._h, m.ctypes.data, 0, None, nb, O_, n_g),
               (eng._h, m.ctypes.data, 0, B, nb, None, 1), (eng._h, m.ctypes.data, 5, B, nb, O_, n_g),
               (eng._h, m.ctypes.data, 0, B, 0, O_, n_g), (eng._h, m.ctypes.data, 0, many.ctypes.data, 64, O_, n_g),
               (eng._h, m.ctypes.data, 0, flat.ctypes.data, 2, O_, n_g), (eng._h, m.ctypes.data, 0, down.ctypes.data, 2, O_, n_g),
               (eng._h, m.ctypes.data, fa.FA_HIST_RTT, B, nb, O_, n_g), (eng._h, m.ctypes.data, fa.FA_HIST_DNS_LATENCY, B, nb, O_, n_g)]
        for args in bad:
            got.value = 7
            assert lib().fa_histogram_flows(*args, C.byref(got)) == FA_E_INVAL, args
            assert got.value == 0
        assert lib().fa_histogram_flows(eng._h, m.ctypes.data, 0, B, nb, O_, n_g, None) == FA_E_INVAL
        if on_gpu:                                                                  # a misaligned device out
            import torch
            t = torch.zeros(n_g * row + 16, dtype=torch.uint8, device="cuda")
            got.value = 7
            assert lib().fa_histogram_flows(eng._h, m.ctypes.data, 0, B, nb, t.data_ptr() + 4, n_g, C.byref(got)) == FA_E_INVAL
        else:
            p = C.c_void_p()
            assert lib().fa_device_alloc(eng._h, n_g * row + 16, C.byref(p)) == FA_OK
            got.value = 7
            assert lib().fa_histogram_flows(eng._h, m.ctypes.data, 0, B, nb, p.value + 4, n_g, C.byref(got)) == FA_E_INVAL
            assert lib().fa_device_free(eng._h, p) == FA_OK
        assert got.value == 0
        assert_hist(eng.histogram_flows(m, fa.FA_HIST_DURATION, bounds), want, "after the errors")
        one = np.array([U64_MAX], np.uint64)                                        # every value lands in bucket 0
        h = eng.histogram_flows(m, fa.FA_HIST_BYTES, one)
        assert (h["counts"][:, 1] == 0).all() and (h["counts"][:, 0] == h["flows"]).all()


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
#define P(f) printf(#f " %zu\n", offsetof(fa_hist_row, f))
int main(void) {
  printf("sizeof %zu\n", sizeof(fa_hist_row));
  printf("row7 %u\n", (unsigned)FA_HIST_ROW_BYTES(7));
  printf("values %u %u %u %u %u %u\n", FA_HIST_BYTES, FA_HIST_PACKETS, FA_HIST_DURATION, FA_HIST_RTT, FA_HIST_DNS_LATENCY,
         FA_HIST_MAX_BOUNDS);
  P(key); P(flows); P(count); P(sum); P(min); P(max);
  return 0;
}
'''


def test_hist_layout_matches_dtype():
    import netobserv_ebpf_agent_b200 as fa
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(c, "w").write(PROBE)
        subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-o", exe, c, "-I" + os.path.join(ROOT, "include")], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    lines = dict(ln.split(" ", 1) for ln in out.strip().splitlines())
    dt = fa.hist_dtype(7)
    assert int(lines["sizeof"]) == dt.fields["counts"][1] == 80
    assert int(lines["row7"]) == dt.itemsize == 80 + 8 * 8
    assert [int(x) for x in lines["values"].split()] == [fa.FA_HIST_BYTES, fa.FA_HIST_PACKETS, fa.FA_HIST_DURATION,
                                                         fa.FA_HIST_RTT, fa.FA_HIST_DNS_LATENCY, fa.FA_HIST_MAX_BOUNDS]
    for f in ("key", "flows", "count", "sum", "min", "max"):
        assert int(lines[f]) == dt.fields[f][1], f
    assert fa.hist_dtype(63).itemsize == 80 + 8 * 64 == 592
