"""fa_expire_flows: evict only the flows past an idle or active timeout, and keep the rest live.

The expected side is an independent restatement on top of the CPU oracle (`Replay`): the live flows are the keys whose
records since their creation are kept, in stream order; the table's rows are the oracle's fold of those records (folds
are per key, so the fold of some keys' records gives those keys' rows); an expiry applies the predicate of
include/flowagg.h to those rows and drops the expired keys' records.  Outputs are compared as sets sorted by key, every
block bit for bit.  Every case runs on the engine emulation (`engine_emul`, small, CPU suite) and on the device (`gpu`,
10^5 to 2·10^6 flows)."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_adversarial_parity import key_families, table_slots
from test_dns_correlate import query, response
from test_evict_blocks import BLOCKS, WIDTHS
from test_gpu_features import keys_of, make_add, make_dns
from test_pktdrop import make_drops
from test_top_flows import rows

pytestmark = pytest.mark.timeout(1200)

T0 = 1_000_000                                   # the generator's ts(i) = T0 + i
CHANGED_BY_EXPIRY = ("flows_evicted", "evictions", "live_flows", "kernel_launches", "d2h_bytes")


# ---------------------------------------------------------------------------------------------------- the oracle
def kid(keys):
    """(m, >= 40) uint8 rows -> (m,) 40-byte void keys (padding byte 39 zeroed), for np.isin / np.unique."""
    a = np.asarray(keys, np.uint8)
    k = np.ascontiguousarray((a if a.ndim == 2 else a.reshape(len(a), -1))[:, :O.ID]).copy()
    k[:, 39] = 0
    return k.view("V40").ravel()


def due(ts, now, timeout):
    if timeout == 0:
        return np.zeros(len(ts), bool)
    return (np.uint64(now) - ts.astype(np.uint64)).view(np.int64) >= np.int64(timeout)


def expired_mask(recs, now, idle, active):
    v = np.ascontiguousarray(recs).view(np.uint8).reshape(-1, O.REC).view(O.REC_DTYPE).reshape(-1)
    return due(v["end"], now, idle) | due(v["start"], now, active)


class Replay:
    """The flows an engine holds, as the records that made them (kind, rows) in stream order.  KERNEL_MAP with a map
    that can fill: which records enter is decided by the oracle's map at the time of each batch."""
    FOLD = {"base": "account", "add": "fold_additional", "dns": "fold_dns", "drop": "fold_drops"}

    def __init__(self, kmap=False, max_entries=0, ringbuf=False):
        self.kmap, self.max_entries, self.ringbuf = kmap, max_entries, ringbuf
        self.hist, self.spilled, self.fail_create = [], [], 0

    def _kmap(self, max_entries, ringbuf):
        km = O.KernelMap(max_entries, ringbuf_fallback=ringbuf)
        for _, r in self.hist:
            km.packets(r)
        return km

    def add(self, kind, recs):
        r = np.ascontiguousarray(recs).view(np.uint8).reshape(len(recs), -1)
        if self.kmap and self.max_entries:
            km = self._kmap(self.max_entries, self.ringbuf)        # the live flows only: the replay never fills the map
            assert km.fail_create == 0
            km.packets(r)
            self.fail_create += km.fail_create
            n_sp = km.spilled()
            if n_sp:
                self.spilled.append(km.spilled_records(n_sp))
            live = kid(km.evict())
            km.close()
            r = r[np.isin(kid(r), live)]                            # spilled records are not part of any flow
        self.hist.append((kind, r))

    def state(self):
        """The six evict_ex blocks of every live flow."""
        if self.kmap:
            km = self._kmap(max(self.max_entries, sum(len(r) for _, r in self.hist), 1), False)
            recs = km.evict()
            km.close()
            m = len(recs)
            return recs, np.zeros((m, 64), np.uint8), np.zeros((m, 32), np.uint8), np.zeros((m, 32), np.uint8), \
                np.zeros(m, np.uint64), np.zeros(m, np.uint8)
        fm = O.FlowMap()
        for kind, r in self.hist:
            getattr(fm, self.FOLD[kind])(r)
        out = fm.evict_ex()
        fm.close()
        return out

    def live_keys(self):
        return kid(self.state()[0])

    def expire(self, now, idle, active):
        st = self.state()
        m = expired_mask(st[0], now, idle, active)
        gone = kid(st[0][m])
        self.hist = [(k, r[~np.isin(kid(r), gone)]) for k, r in self.hist]
        return tuple(np.asarray(b)[m] for b in st)

    def evict(self):
        st = self.state()
        self.hist = []
        return st


def sorted_rows(blocks):
    b = rows(blocks)
    p = O.sort_perm(b[0])
    return [x[p] for x in b]


def assert_same(got, want, what=""):
    g, w = sorted_rows(got), sorted_rows(want)
    assert len(g[0]) == len(w[0]), (what, len(g[0]), len(w[0]))
    for name, a, b in zip(BLOCKS, g, w):
        if not np.array_equal(a, b):
            bad = np.nonzero((a != b).any(axis=1))[0]
            raise AssertionError(f"{what} {name}: {len(bad)} of {len(a)} rows differ, first at {int(bad[0])}")


def times_of(blocks):
    v = rows(blocks)[0].view(O.REC_DTYPE).reshape(-1)
    return v["start"].astype(np.uint64), v["end"].astype(np.uint64)


def idle_cut(rep, q, now):
    """An idle timeout that expires about a fraction q of the replay's flows at `now` (a timestamp quantile)."""
    _, end = times_of(rep.state())
    return max(int(now) - int(np.quantile(end.astype(np.float64), q)), 1)


def active_cut(rep, q, now):
    start, _ = times_of(rep.state())
    s = start[start != 0].astype(np.float64)
    return max(int(now) - int(np.quantile(s, q)), 1) if len(s) else 1


def expire_both(eng, rep, now, idle, active, what):
    got = eng.expire_flows(now, idle, active)
    want = rep.expire(now, idle, active)
    assert_same(got, want, what)
    return got


# ---------------------------------------------------------------------------------------------------- 1. oracle parity
def check_oracle(n, n_keys, mode, dist, varying, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    kmap = mode == fa.FA_MODE_KERNEL_MAP
    recs = gen_host(seed=1101 + dist + 2 * varying + 4 * mode, n=n, n_keys=n_keys, dist=dist, varying=varying, t0=T0)
    parts = np.array_split(recs, 4)
    rep = Replay(kmap=kmap)
    total = 0
    with fa.FlowAggEngine(4 * n_keys, mode=mode, max_batch=max_batch) as eng:
        for i, part in enumerate(parts):
            eng.ingest(part)
            rep.add("base", part)
            now = T0 + sum(len(p) for p in parts[: i + 1])
            if i == 0:
                idle, active = idle_cut(rep, 0.3, now), 0
            elif i == 1:
                idle, active = 0, active_cut(rep, 0.5, now)
            elif i == 2:
                idle, active = idle_cut(rep, 0.2, now), active_cut(rep, 0.2, now)
            else:
                break
            got = expire_both(eng, rep, now, idle, active, f"expiry {i}")
            assert 0 < len(got[0]) < len(rep.state()[0]) + len(got[0])
            total += len(got[0])
            assert eng.live_flows() == len(rep.state()[0])
        assert_same(eng.evict_ex(), rep.evict(), "final eviction")
        assert eng.stats()["flows_evicted"] >= total


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


# ---------------------------------------------------------------------------------------------------- 2. survivors
def family_records(fam_keys, template, t_old, t_new):
    """One record per key; alternate members of each family get old timestamps."""
    out = []
    for keys in fam_keys:
        r = np.repeat(template[:1], len(keys), axis=0)
        r[:, :40] = keys
        v = r.view(O.REC_DTYPE).reshape(-1)
        old = (np.arange(len(keys)) % 2) == 1
        v["start"] = np.where(old, t_old, t_new)
        v["end"] = np.where(old, t_old + 5, t_new + 5)
        out.append(r)
    return np.concatenate(out)


def check_survivors(n_bg, max_entries, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    fam = key_families(1201, table_slots(max_entries), n_full=64, n_chain=300, n_way=32)
    bg = gen_host(seed=1202, n=n_bg, n_keys=n_bg // 2, dist=1, t0=T0)
    t_new = T0 + n_bg
    fr = family_records([fam["full"], fam["chain_last"], fam["chain_mid"], fam["way"]], bg, T0 // 2, t_new)
    recs = np.concatenate([bg, fr])
    recs = recs[np.random.default_rng(1203).permutation(len(recs))]
    rep = Replay()
    with fa.FlowAggEngine(max_entries, max_batch=max_batch) as eng:
        eng.ingest(recs)
        rep.add("base", recs)
        now = t_new + 10
        idle = now - (T0 // 2 + 5)                                 # every old family member and the older background
        idle = min(idle, idle_cut(rep, 0.5, now))
        survivors_before = rep.state()
        keep = ~expired_mask(survivors_before[0], now, idle, 0)
        live_keys = rows(survivors_before)[0][keep][:, :40].copy()
        before = eng.lookup_flows(live_keys)
        got = expire_both(eng, rep, now, idle, 0, "colliding families")
        assert len(got[0]) > len(fr) // 3
        after = eng.lookup_flows(live_keys)
        assert after[6].all()
        for name, a, b in zip(BLOCKS, rows(before[:6]), rows(after[:6])):
            assert np.array_equal(a, b), name
        assert not eng.lookup_flows(got[0][:, :40].copy())[6].any()     # expired keys miss
        more = gen_host(seed=1204, n=n_bg // 2, n_keys=n_bg, dist=0, t0=t_new + 100)
        again = np.repeat(more[:1], len(fr), axis=0)
        again[:, :40] = fr[:, :40]
        again.view(O.REC_DTYPE)["start"] = t_new + 200
        again.view(O.REC_DTYPE)["end"] = t_new + 300
        tail = np.concatenate([more, again])
        eng.ingest(tail)
        rep.add("base", tail)
        final = eng.evict_ex()
        assert len(np.unique(kid(final[0]))) == len(final[0])           # no key twice
        assert_same(final, rep.evict(), "after re-ingest")


def test_survivors_emul(engine_emul):
    check_survivors(2_000, 4_000, max_batch=1_000)


@pytest.mark.gpu
def test_survivors_gpu():
    check_survivors(400_000, 1_000_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 3. feature folds
def check_features(n, n_keys, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(1301)
    recs = gen_host(seed=1301, n=n, n_keys=n_keys, dist=1, t0=T0)
    # one home-slot chain: alternate members are old and carry feature samples (timeless, so the base decides), the
    # survivors move back along the chain, and the chain's later keys are created afterwards in the slots they vacated
    chain = key_families(1304, table_slots(4 * n_keys), n_chain=160)["chain_mid"]
    old_c, new_c = chain[:24], chain[24:]
    keys = np.concatenate([np.unique(recs[:, :40], axis=0), keys_of(1302, 64)])     # 64 feature-only flows
    add, dns, drops = make_add(rng, keys, n // 4), make_dns(rng, keys, n // 8), make_drops(rng, keys, n // 8)
    recs = np.concatenate([recs, family_records([old_c], recs, T0 // 2, 1 << 42)])   # 1 << 42: after every sample
    c_add, c_dns = make_add(rng, old_c, 96), make_dns(rng, old_c, 48)
    for blk, f in ((c_add.view(O.ADDREC_DTYPE), "add"), (c_dns.view(O.DNSREC_DTYPE), "dns")):
        blk[f]["start"] = 0
        blk[f]["end"] = 0
    add, dns = np.concatenate([add, c_add]), np.concatenate([dns, c_dns])
    rep = Replay()
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP
    with fa.FlowAggEngine(4 * n_keys, flags=flags, max_batch=max_batch) as eng:
        eng.ingest_additional(add[: len(add) // 2]); rep.add("add", add[: len(add) // 2])
        eng.ingest(recs); rep.add("base", recs)
        eng.ingest_dns(dns); rep.add("dns", dns)
        eng.ingest_pkt_drops(drops); rep.add("drop", drops)
        eng.ingest_additional(add[len(add) // 2:]); rep.add("add", add[len(add) // 2:])
        st = rep.state()
        only = np.isin(kid(st[0]), kid(keys[-64:]))
        assert only.any() and rows(st)[5][only].all()
        _, end = times_of(st)
        now = int(end.max()) + 1
        for q in (0.3, 0.6):
            idle = idle_cut(rep, q, now)
            got = expire_both(eng, rep, now, idle, 0, f"features q={q}")
            assert (rows(got)[5] != 0).any() and len(got[0])
            if q == 0.3:                                          # the chain's new keys go where its survivors were
                live_now = rep.live_keys()
                assert not np.isin(kid(old_c[1::2]), live_now).any() and np.isin(kid(old_c[0::2]), live_now).all()
                nc = family_records([new_c], recs, now - 3, now - 3)
                eng.ingest(nc); rep.add("base", nc)
        # the feature-only flows' patched times decide: some of them expired, some are still live
        gone = kid(keys[-64:])
        live_now = rep.live_keys()
        assert 0 < np.isin(gone, live_now).sum() < 64
        fresh = gen_host(seed=1303, n=n // 2, n_keys=n_keys, dist=0, t0=now + 10)     # new flows, some in freed slots
        eng.ingest(fresh); rep.add("base", fresh)
        final = eng.evict_ex()
        assert_same(final, rep.evict(), "new flows in freed slots")
        new = ~np.isin(kid(final[0]), np.concatenate([kid(keys), kid(chain)]))
        assert new.any() and not rows(final)[5][new].any()           # no stray feature blocks


def test_features_emul(engine_emul):
    check_features(2_000, 500, max_batch=600)


@pytest.mark.gpu
def test_features_gpu():
    check_features(600_000, 150_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 4. KERNEL_MAP full map
def check_kmap_full(n, n_keys, max_entries, ringbuf, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=1401 + ringbuf, n=n, n_keys=n_keys, dist=0, t0=T0)     # uniform: every part fills the map
    v = recs.view(O.REC_DTYPE).reshape(-1)
    v["if_index"] = np.where(np.random.default_rng(1402).random(n) < 0.3, 7, 3)
    parts = np.array_split(recs, 3)
    rep = Replay(kmap=True, max_entries=max_entries, ringbuf=ringbuf)
    spilled = []
    with fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=fa.FA_F_RINGBUF_FALLBACK if ringbuf else 0,
                          max_batch=max_batch) as eng:
        for i, part in enumerate(parts):
            eng.ingest(part)
            rep.add("base", part)
            if ringbuf:
                spilled.append(eng.read_spilled())
            assert eng.live_flows() == len(rep.state()[0])
            now = T0 + sum(len(p) for p in parts[: i + 1])
            if i < 2:
                got = expire_both(eng, rep, now, idle_cut(rep, 0.5, now), 0, f"kmap expiry {i}")
                assert len(got[0])
        assert_same(eng.evict_ex(), rep.evict(), "final eviction")
        st = eng.stats()
    assert st["hashmap_fail_create"] == rep.fail_create
    assert (rep.spilled if ringbuf else rep.fail_create)          # the map filled
    if ringbuf:
        g, w = np.concatenate(spilled), np.concatenate(rep.spilled)
        assert st["ringbuf_spilled"] == len(w) == len(g)
        assert np.array_equal(g[np.lexsort(g.T[::-1])], w[np.lexsort(w.T[::-1])])    # whole rows: a key can spill twice
    else:
        assert st["ringbuf_spilled"] == 0


@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_full_emul(engine_emul, monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kmap_full(3_000, 1_000, 300, ringbuf, max_batch=700)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf", [False, True])
def test_kernel_map_full_gpu(monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kmap_full(600_000, 200_000, 50_000, ringbuf, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 5. ACCOUNTER FA_FULL
def accounter_cut(live, recs, max_entries):
    """Index of the first record whose key is new while the cache holds max_entries flows, or len(recs)."""
    ids = kid(recs)
    new = np.nonzero(~np.isin(ids, live))[0]
    _, first = np.unique(ids[new], return_index=True)
    firsts = np.sort(new[first])
    room = max_entries - len(live)
    return int(firsts[room]) if len(firsts) > room else len(recs)


def check_full_cut(n, n_keys, max_entries, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=1501, n=n, n_keys=n_keys, dist=0, t0=T0)
    rep = Replay()
    done, gens = 0, 0
    with fa.FlowAggEngine(max_entries, max_batch=max_batch) as eng:
        while done < n:
            rc, took = eng.ingest(recs[done:])
            assert took == accounter_cut(rep.live_keys(), recs[done:], max_entries)
            rep.add("base", recs[done:done + took])
            done += took
            if rc == fa.FA_FULL:
                assert eng.live_flows() == max_entries
                now = T0 + done
                got = expire_both(eng, rep, now, idle_cut(rep, 0.5, now), 0, f"generation {gens}")
                assert 0 < len(got[0]) < max_entries
                gens += 1
        assert_same(eng.evict_ex(), rep.evict(), "final eviction")
        st = eng.stats()
    assert gens >= 3 and st["full_cuts"] == gens


def test_full_cut_emul(engine_emul):
    check_full_cut(30_000, 20_000, 5_000, max_batch=4_096)


@pytest.mark.gpu
def test_full_cut_gpu():
    check_full_cut(400_000, 200_000, 5_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 6. full table
def check_physically_full(max_entries, n, max_batch):
    """FA_F_NO_FULL_CUT with more distinct keys than slots: no EMPTY slot, so no cluster bound (the one-thread
    backward-shift path).  The expected rows come from the engine's own top-k snapshot of the whole table."""
    import netobserv_ebpf_agent_b200 as fa
    slots = table_slots(max_entries)
    recs = gen_host(seed=1601, n=n, n_keys=1 << 30, dist=0, t0=T0)
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NO_FULL_CUT, max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.stats()["spills"] > 0 and eng.live_flows() == slots
        snap = eng.top_flows(slots)
        now = T0 + n
        idle = idle_cut_of(snap, 0.4, now)
        m = expired_mask(snap[0], now, idle, 0)
        survivors = rows(snap)[0][~m]
        before = eng.lookup_flows(survivors[:, :40].copy())
        got = eng.expire_flows(now, idle)
        assert_same(got, tuple(np.asarray(b)[m] for b in snap), "expired")
        after = eng.lookup_flows(survivors[:, :40].copy())
        assert after[6].all() and np.array_equal(before[0], after[0])
        assert not eng.lookup_flows(got[0][:, :40].copy())[6].any()
        fresh = gen_host(seed=1602, n=int(m.sum()) // 2, n_keys=1 << 30, dist=0, t0=now)
        eng.ingest(fresh)
        assert eng.lookup_flows(fresh[:, :40].copy())[6].all()
        final = eng.evict_ex()
        assert len(np.unique(kid(final[0]))) == len(final[0]) == len(survivors) + len(np.unique(kid(fresh)))
        keep = np.isin(kid(final[0]), kid(survivors))
        assert_same(tuple(np.asarray(b)[keep] for b in final), tuple(np.asarray(b)[~m] for b in snap), "survivors")


def idle_cut_of(blocks, q, now):
    _, end = times_of(blocks)
    return max(int(now) - int(np.quantile(end.astype(np.float64), q)), 1)


def test_physically_full_emul(engine_emul):
    check_physically_full(700, 1_100, max_batch=600)                 # 1024 slots


@pytest.mark.gpu
def test_physically_full_gpu():
    check_physically_full(180_000, 600_000, max_batch=1 << 16)        # 2^18 slots


# ---------------------------------------------------------------------------------------------------- 7. non-blocking
def check_nonblocking_sequential(n, n_keys, mode):
    import netobserv_ebpf_agent_b200 as fa
    kmap = mode == fa.FA_MODE_KERNEL_MAP
    recs = gen_host(seed=1701 + mode, n=n, n_keys=n_keys, dist=1, t0=T0)
    a, b = recs[: n // 2], recs[n // 2:]
    rep = Replay(kmap=kmap)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_NONBLOCKING_EVICT) as eng:
        eng.ingest(a); rep.add("base", a)
        now = T0 + len(a)
        expire_both(eng, rep, now, idle_cut(rep, 0.4, now), 0, "first expiry")
        assert_same(eng.evict_ex(), rep.evict(), "first eviction")
        eng.ingest(b); rep.add("base", b)
        now = T0 + n
        expire_both(eng, rep, now, idle_cut(rep, 0.3, now), active_cut(rep, 0.3, now), "second expiry")
        assert_same(eng.evict_ex(), rep.evict(), "second eviction")
        assert eng.live_flows() == 0


def check_nonblocking_concurrent(n, n_keys, max_entries, max_batch, chunk):
    """An ingest thread and an evictor thread that alternates fa_expire_flows and fa_evict_ex: every record ends up in
    exactly one output, so the union of the outputs, re-folded, equals the oracle's fold of the stream."""
    import netobserv_ebpf_agent_b200 as fa
    from test_nonblocking_evict import refold
    recs = gen_host(seed=1703, n=n, n_keys=n_keys, dist=1, t0=T0)
    out, stop, progress = [], threading.Event(), [0]
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NONBLOCKING_EVICT, max_batch=max_batch) as eng:
        def evictor():
            k = 0
            while not stop.is_set():
                if k % 2 == 0:
                    now = T0 + progress[0]
                    out.append(eng.expire_flows(now, chunk // 2, chunk, cap=max_entries)[0].copy())
                else:
                    out.append(eng.evict(cap=max_entries).copy())
                k += 1
        t = threading.Thread(target=evictor)
        t.start()
        for lo in range(0, n, chunk):
            rc, took = eng.ingest(recs[lo:lo + chunk])
            assert rc == 0 and took == min(chunk, n - lo)
            progress[0] = lo + took
        stop.set(); t.join()
        out.append(eng.evict().copy())
        st = eng.stats()
    assert st["records_ingested"] == n and st["flows_evicted"] == sum(len(p) for p in out)
    assert sum(1 for p in out[:-1:2] if len(p)) >= 1 and sum(1 for p in out if len(p)) >= 2
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


# ---------------------------------------------------------------------------------------------------- 8. nothing else
def check_nothing_else(n, n_keys, max_batch):
    """With the sketch and the DNS correlation table in use: the sketch export, the pending DNS queries and every fa_stats
    field but the five an expiry moves are those of an engine that never expired."""
    import netobserv_ebpf_agent_b200 as fa
    from test_adversarial_parity import SKETCH_SEED
    recs = gen_host(seed=1801, n=n, n_keys=n_keys, dist=1, t0=T0)
    kw = dict(flags=fa.FA_F_ENABLE_SKETCH | fa.FA_F_ENABLE_DNS, cms_log2_width=12, cms_depth=4, hll_precision=10,
              sketch_seed=SKETCH_SEED, max_batch=max_batch)
    pkts = np.concatenate([query(1000, 7), response(5000, 7), query(6000, 9, sport=40001)])     # one query stays pending
    with fa.FlowAggEngine(4 * n_keys, **kw) as eng, fa.FlowAggEngine(4 * n_keys, **kw) as ref:
        for x in (eng, ref):
            x.ingest(recs[: n // 2]); x.ingest_dns_packets(pkts)
        got = eng.expire_flows(T0 + n // 2, n // 8)
        assert len(got[0])
        for x in (eng, ref):
            x.ingest(recs[n // 2:])
        s_eng, s_ref = eng.stats(), ref.stats()
        assert s_ref["dns_queries_pending"] == 1
        for k in s_ref:
            if k not in CHANGED_BY_EXPIRY:
                assert s_eng[k] == s_ref[k], k
        assert s_eng["flows_evicted"] == len(got[0]) and s_eng["evictions"] == 1
        assert s_eng["live_flows"] == eng.live_flows()
        for a, b in zip(eng.sketch_export(12, 4, 10), ref.sketch_export(12, 4, 10)):
            assert np.array_equal(a, b)
        assert eng.hll_estimate() == ref.hll_estimate()


def test_nothing_else_emul(engine_emul):
    check_nothing_else(2_000, 600, 500)


@pytest.mark.gpu
def test_nothing_else_gpu():
    check_nothing_else(800_000, 200_000, 1 << 16)


# ---------------------------------------------------------------------------------------------------- 9. placement, errors
def expire_filled(eng, now, idle, cap, device, on_gpu):
    """fa_expire_flows with every block pre-filled with 0xFF in host memory or, where device[i] is set, in device
    memory -> (blocks, n)."""
    from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib
    held, ptrs, reads = [], [], []
    for w, dev in zip(WIDTHS, device):
        if dev and on_gpu:
            import torch
            b = torch.full((cap * w,), 0xFF, dtype=torch.uint8, device="cuda"); held.append(b)
            ptrs.append(b.data_ptr()); reads.append(lambda b=b: b.cpu().numpy())
        elif dev:
            p = C.c_void_p(); check(lib().fa_device_alloc(eng._h, cap * w, C.byref(p))); C.memset(p.value, 0xFF, cap * w)
            held.append(p); ptrs.append(p.value)
            reads.append(lambda p=p, nb=cap * w: np.frombuffer(C.string_at(p.value, nb), np.uint8).copy())
        else:
            b = np.full(cap * w, 0xFF, np.uint8); held.append(b); ptrs.append(b.ctypes.data); reads.append(lambda b=b: b)
    got = C.c_size_t(0)
    check(lib().fa_expire_flows(eng._h, now, idle, 0, C.byref(EvictOut(*ptrs)), cap, C.byref(got)))
    g = got.value
    blocks = [r()[: g * w].reshape(g, w) for r, w in zip(reads, WIDTHS)]
    for b in held:
        if isinstance(b, C.c_void_p):
            check(lib().fa_device_free(eng._h, b))
    return blocks, g


PLACEMENTS = [(False,) * 6, (True,) * 6] + [tuple(i == j for j in range(6)) for i in range(6)]


def check_placement(n, n_keys, mode, rtt, on_gpu, max_batch):
    """Host and device blocks, unproduced blocks zeroed; each placement expires its own slice of the flows, against the
    oracle."""
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=1901, n=n, n_keys=n_keys, dist=0, t0=T0)
    keys = np.unique(recs[:, :40], axis=0)
    produced = {"records", "additional", "rtt_min", "present"} if rtt else {"records"}
    rep = Replay(kmap=mode == fa.FA_MODE_KERNEL_MAP)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_ENABLE_RTT if rtt else 0, max_batch=max_batch) as eng:
        eng.ingest(recs); rep.add("base", recs)
        if rtt:
            add = make_add(np.random.default_rng(1902), keys, n // 4)
            add.view(O.ADDREC_DTYPE)["add"]["end"] = 0                 # the base records' times decide
            eng.ingest_additional(add); rep.add("add", add)
        if mode == fa.FA_MODE_KERNEL_MAP and rtt:
            pytest.skip("the replay oracle restates KERNEL_MAP without feature folds")
        now = T0 + n
        for i, device in enumerate(PLACEMENTS):
            idle = n - (i + 1) * n // (len(PLACEMENTS) + 1)
            want = rep.expire(now, idle, 0)
            cap = len(want[0]) + 3
            blocks, g = expire_filled(eng, now, idle, cap, device, on_gpu)
            assert g == len(want[0]) and g > 0
            for name, b in zip(BLOCKS, blocks):
                if name not in produced:
                    assert not b.any(), (device, name)
            assert_same(blocks, want, f"placement {device}")


@pytest.mark.parametrize("mode,rtt", [(0, False), (0, True), (1, False)])
def test_placement_emul(engine_emul, mode, rtt):
    check_placement(1_500, 400, mode, rtt, on_gpu=False, max_batch=256)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtt", [(0, False), (0, True), (1, False)])
def test_placement_gpu(mode, rtt):
    check_placement(600_000, 200_000, mode, rtt, on_gpu=True, max_batch=1 << 16)


def check_errors(n, n_keys):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, FA_E_INVAL, EvictOut, lib
    recs = gen_host(seed=1951, n=n, n_keys=n_keys, dist=1, t0=T0)
    with fa.FlowAggEngine(4 * n_keys) as eng:
        assert len(eng.expire_flows(T0, 5)[0]) == 0                      # empty table: nothing expires, not an error
        assert eng.stats()["evictions"] == 1
        eng.ingest(recs)
        live = eng.live_flows()
        out = np.full((4, O.REC), 0xAB, np.uint8)
        good, no_rec = EvictOut(records=out.ctypes.data), EvictOut()
        got = C.c_size_t(7)
        before = eng.stats()
        big = 1 << 63
        cases = [(None, T0, 5, 0, C.byref(good), 4, C.byref(got)), (eng._h, T0, 5, 0, None, 4, C.byref(got)),
                 (eng._h, T0, 5, 0, C.byref(no_rec), 4, C.byref(got)), (eng._h, T0, 5, 0, C.byref(good), 4, None),
                 (eng._h, T0, 0, 0, C.byref(good), 4, C.byref(got)), (eng._h, T0, big, 0, C.byref(good), 4, C.byref(got)),
                 (eng._h, T0, 0, big, C.byref(good), 4, C.byref(got))]
        for c in cases:
            assert lib().fa_expire_flows(*c) == FA_E_INVAL, c
            assert got.value == 0 or c[-1] is None
            got.value = 7
        # nothing expires: the timestamps are all after now - timeout, or after now (skewed clocks)
        assert len(eng.expire_flows(T0 + n, n + 10)[0]) == 0
        assert len(eng.expire_flows(T0 - 10, 1, 1)[0]) == 0
        # FA_E_2BIG with the count; nothing changes
        now, idle = T0 + n, n // 2
        want = Replay(); want.add("base", recs)
        n_exp = int(expired_mask(want.state()[0], now, idle, 0).sum())
        assert n_exp > 4
        assert lib().fa_expire_flows(eng._h, now, idle, 0, C.byref(good), 4, C.byref(got)) == FA_E_2BIG
        assert got.value == n_exp and (out == 0xAB).all()
        assert eng.live_flows() == live
        after = eng.stats()
        for k in before:
            if k not in ("evictions", "kernel_launches", "d2h_bytes"):
                assert after[k] == before[k], k
        assert after["evictions"] == before["evictions"] + 2              # the two calls that expired nothing
        expired = eng.expire_flows(now, idle, cap=n_exp)
        assert_same(expired, want.expire(now, idle, 0), "after FA_E_2BIG")
        assert_same(eng.evict_ex(), want.evict(), "rest")


def test_errors_emul(engine_emul):
    check_errors(1_000, 300)


@pytest.mark.gpu
def test_errors_gpu():
    check_errors(200_000, 50_000)
