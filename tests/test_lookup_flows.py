"""fa_lookup_flows: exact point lookups of live flows by key, on the device, without evicting.

Row i of every block answers keys[i]: for a live flow it equals the fa_evict_ex row of that flow taken right after (or
the oracle's flow), bit for bit; for any other key it is all zero, and found[i] says which.  Every case runs on the
engine emulation (`engine_emul`, small, CPU suite) and on the device (`gpu`, 10^5 to 2·10^6 flows, up to 10^6
lookups).  A small max_batch makes the lookups cross chunk boundaries."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_adversarial_parity import DevBuf, key_families, table_slots
from test_evict_blocks import BLOCKS, WIDTHS
from test_gpu_features import keys_of, make_add
from test_top_flows import feature_engine, oracle_flows, rows

pytestmark = pytest.mark.timeout(900)

UNCHANGED_BY_LOOKUP = ("kernel_launches", "h2d_bytes", "d2h_bytes")


# ---------------------------------------------------------------------------------------------------- helpers
def keys_of_recs(recs):
    k = np.ascontiguousarray(np.ascontiguousarray(recs).view(np.uint8).reshape(-1, O.REC)[:, :O.ID]).copy()
    k[:, 39] = 0
    return k


def absent_keys(seed, n, live_keys):
    """n keys of a disjoint generator seed that are not live."""
    k = np.unique(keys_of_recs(gen_host(seed=seed, n=2 * n + 16, n_keys=1 << 32, dist=0)), axis=0)
    live = {bytes(x) for x in live_keys}
    k = np.array([x for x in k if bytes(x) not in live], dtype=np.uint8).reshape(-1, O.ID)
    return k[:n]


def query_of(live_keys, absent, rng, n_dup):
    """All live keys, the absent ones and n_dup duplicates of live keys, shuffled."""
    dup = live_keys[rng.integers(0, len(live_keys), n_dup)] if n_dup else np.zeros((0, O.ID), np.uint8)
    q = np.concatenate([live_keys, absent, dup])
    return q[rng.permutation(len(q))]


def expected(blocks, q):
    """The rows lookup must return for keys q, given the evict_ex blocks (or (records,)) of the same table."""
    blocks = rows(blocks)
    at = {bytes(k): i for i, k in enumerate(keys_of_recs(blocks[0]))}
    qn = np.ascontiguousarray(q).copy()
    qn[:, 39] = 0
    idx = np.array([at.get(k.tobytes(), -1) for k in qn], dtype=np.int64)
    out = []
    for b in blocks:
        w = np.zeros((len(q), b.shape[1]), np.uint8)
        w[idx >= 0] = b[idx[idx >= 0]]
        out.append(w)
    return out, (idx >= 0).astype(np.uint8)


def assert_rows_equal(got, want, what=""):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} rows differ, first at row {int(bad[0])}")


def check_lookup(got, want_blocks, want_found):
    *blocks, found = got
    got_rows = rows(blocks)
    for name, g, w in zip(BLOCKS, got_rows, want_blocks):
        assert_rows_equal(g, w, name)
    assert np.array_equal(found, want_found)


def lookup_raw(eng, keys, n=None, found=True):
    """fa_lookup_flows from a host key array or address -> (rc, n_found, found, records)."""
    from netobserv_ebpf_agent_b200._lib import EvictOut, lib
    n = len(keys) if n is None else n
    out = np.zeros((max(n, 1), O.REC), np.uint8)
    f = np.zeros(max(n, 1), np.uint8)
    got = C.c_size_t(0)
    kp = keys if isinstance(keys, int) or keys is None else keys.ctypes.data
    rc = lib().fa_lookup_flows(eng._h, kp, n, C.byref(EvictOut(records=out.ctypes.data)), f.ctypes.data if found else None,
                               C.byref(got))
    return rc, got.value, f[:n], out[:n]


# ---------------------------------------------------------------------------------------------------- 1. oracle
def check_oracle(n, n_keys, dist, varying, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(100 + dist + 2 * varying)
    recs = gen_host(seed=101 + dist + 2 * varying, n=n, n_keys=n_keys, dist=dist, varying=varying)
    max_entries = 2 * n_keys
    want = oracle_flows([recs], max_entries)
    live_keys = keys_of_recs(want)
    q = query_of(live_keys, absent_keys(7000 + dist, len(live_keys) // 2, live_keys), rng, len(live_keys) // 4)
    with fa.FlowAggEngine(max_entries, max_batch=max_batch) as eng:
        assert eng.ingest(recs) == (fa.FA_OK, n)
        got = eng.lookup_flows(q)
        wb, wf = expected((want,), q)
        assert_rows_equal(got[0], wb[0], "records")
        assert np.array_equal(got[6], wf)
        assert not any(b.any() for b in got[1:6])                # no feature folds: every feature block is zero
        rc, n_found, found, _ = lookup_raw(eng, q)
        assert rc == 0 and n_found == int(wf.sum()) and np.array_equal(found, wf)
        assert eng.live_flows() == len(want)


@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
@pytest.mark.parametrize("varying", [0, 1])
def test_oracle_emul(engine_emul, dist, varying):
    check_oracle(3_000, 1_000, dist, varying, max_batch=700)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", [0, 1], ids=["uniform", "zipf"])
@pytest.mark.parametrize("varying", [0, 1])
def test_oracle_gpu(dist, varying):
    check_oracle(1_000_000, 400_000, dist, varying, max_batch=1 << 17)


# ---------------------------------------------------------------------------------------------------- 2. colliding keys
def check_colliding(n_bg, max_entries, max_batch):
    """Keys of one identical premix, 300-key home-slot chains (one at the last slot: the walk wraps) and keys sharing the
    low 32 hash bits; every second key of each family is ingested, the others must miss after walking the chain."""
    import netobserv_ebpf_agent_b200 as fa
    fam = key_families(201, table_slots(max_entries), n_full=64, n_chain=300, n_way=32)
    bg = gen_host(seed=202, n=n_bg, n_keys=n_bg // 2, dist=1)
    present = np.concatenate([f[0::2] for f in fam.values()])
    absent = np.concatenate([f[1::2] for f in fam.values()])
    coll = np.repeat(bg[:1], len(present), axis=0)
    coll[:, :40] = present
    recs = np.concatenate([bg, coll])
    recs = recs[np.random.default_rng(203).permutation(len(recs))]
    want = oracle_flows([recs], max_entries)
    q = np.concatenate([present, absent, keys_of_recs(bg[:50])])
    with fa.FlowAggEngine(max_entries, max_batch=max_batch) as eng:
        eng.ingest(recs)
        got = eng.lookup_flows(q)
        wb, wf = expected((want,), q)
        assert wf[:len(present)].all() and not wf[len(present):len(present) + len(absent)].any()
        assert_rows_equal(got[0], wb[0], "records")
        assert np.array_equal(got[6], wf)


def test_colliding_emul(engine_emul):
    check_colliding(2_000, 4_000, max_batch=1_000)


@pytest.mark.gpu
def test_colliding_gpu():
    check_colliding(400_000, 1_000_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 3. nothing changes
def check_nothing_changes(n, n_keys, max_batch, sketch):
    import netobserv_ebpf_agent_b200 as fa
    a = gen_host(seed=301, n=n, n_keys=n_keys, dist=1)
    b = gen_host(seed=302, n=n, n_keys=n_keys, dist=1, first=n)
    flags = fa.FA_F_ENABLE_SKETCH if sketch else 0
    q = np.concatenate([keys_of_recs(a[:n // 4]), keys_of_recs(b[:n // 4])])
    with fa.FlowAggEngine(4 * n_keys, max_batch=max_batch, flags=flags) as eng, \
            fa.FlowAggEngine(4 * n_keys, max_batch=max_batch, flags=flags) as ref:
        for x in (a, b):
            eng.ingest(x); ref.ingest(x)
            for _ in range(3):
                eng.lookup_flows(q)
        s_eng, s_ref = eng.stats(), ref.stats()
        assert s_eng["kernel_launches"] > s_ref["kernel_launches"]
        for k in s_ref:
            if k not in UNCHANGED_BY_LOOKUP:
                assert s_eng[k] == s_ref[k], k
        if sketch:
            assert np.array_equal(eng.cms_query(q), ref.cms_query(q))
        got, want = eng.evict_ex(), ref.evict_ex()
        order_g, order_w = np.lexsort(rows(got)[0][:, :40].T[::-1]), np.lexsort(rows(want)[0][:, :40].T[::-1])
        for name, g, w in zip(BLOCKS, rows(got), rows(want)):
            assert_rows_equal(g[order_g], w[order_w], name)
        assert eng.lookup_flows(q)[6].sum() == 0                  # evicted: every key misses


@pytest.mark.parametrize("sketch", [False, True])
def test_nothing_changes_emul(engine_emul, sketch):
    check_nothing_changes(2_000, 600, 500, sketch)


@pytest.mark.gpu
@pytest.mark.parametrize("sketch", [False, True])
def test_nothing_changes_gpu(sketch):
    check_nothing_changes(800_000, 200_000, 1 << 16, sketch)


# ---------------------------------------------------------------------------------------------------- 4. feature blocks
def check_features(n, n_keys):
    eng = feature_engine(n, n_keys, 401)
    try:
        live = eng.live_flows()
        live_keys = keys_of_recs(eng.top_flows(live + 5)[0])       # base, feature-only and DNS-packet flows
        assert len(live_keys) == live
        q = query_of(live_keys, absent_keys(402, 100, live_keys), np.random.default_rng(403), 50)
        got = eng.lookup_flows(q)
        assert eng.live_flows() == live
        evicted = eng.evict_ex()
        assert (rows(evicted)[5] != 0).any() and (rows(evicted)[5] == 0).any()
        wb, wf = expected(evicted, q)
        check_lookup(got, wb, wf)
    finally:
        eng.close()


def test_feature_rows_emul(engine_emul):
    check_features(1_500, 400)


@pytest.mark.gpu
def test_feature_rows_gpu():
    check_features(400_000, 100_000)


# ---------------------------------------------------------------------------------------------------- 5. KERNEL_MAP
def check_kernel_map(n, n_keys, max_entries, ringbuf, rtt, max_batch):
    """Packets of every flow on two interfaces; with max_entries below the key count the map fills and the rest goes to
    the fallback ring (or only counts), and those keys miss."""
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=501, n=n, n_keys=n_keys, dist=1)
    v = recs.view(O.REC_DTYPE).reshape(-1)
    v["if_index"] = np.where(np.random.default_rng(502).random(n) < 0.3, 7, 3)
    flags = (fa.FA_F_RINGBUF_FALLBACK if ringbuf else 0) | (fa.FA_F_ENABLE_RTT if rtt else 0)
    all_keys = np.unique(keys_of_recs(recs), axis=0)
    with fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=flags, max_batch=max_batch) as eng:
        eng.ingest(recs)
        extra = keys_of(503, 8)
        if rtt:
            eng.ingest_additional(make_add(np.random.default_rng(504), np.concatenate([all_keys[:50], extra]), n // 8))
        q = query_of(np.concatenate([all_keys, extra]), absent_keys(505, 100, all_keys), np.random.default_rng(506), 40)
        live = eng.live_flows()
        got = eng.lookup_flows(q)
        assert eng.live_flows() == live
        evicted = eng.evict_ex()
        assert len(evicted[0]) == live
        wb, wf = expected(evicted, q)
        check_lookup(got, wb, wf)
        if max_entries < n_keys:
            assert len(evicted[0]) < len(all_keys)                  # the map filled: the other keys miss
        if ringbuf:
            spilled = {bytes(k) for k in keys_of_recs(eng.read_spilled())}
            assert spilled and not any(bytes(k) in spilled for k in q[wf == 1])


@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf,full", [(False, False), (False, True), (True, True)])
def test_kernel_map_emul(engine_emul, monkeypatch, impl, ringbuf, full):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kernel_map(2_000, 600, 300 if full else 2_000, ringbuf, rtt=not full, max_batch=700)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["1", "2"])
@pytest.mark.parametrize("ringbuf,full", [(False, False), (False, True), (True, True)])
def test_kernel_map_gpu(monkeypatch, impl, ringbuf, full):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    check_kernel_map(400_000, 100_000, 20_000 if full else 200_000, ringbuf, rtt=not full, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 6. full table
def check_physically_full(max_entries, n, n_keys, max_batch):
    """FA_F_NO_FULL_CUT with more distinct keys than slots: the table is physically full (spills > 0), so a miss walks
    every slot and must stop after mask + 1 of them."""
    import netobserv_ebpf_agent_b200 as fa
    slots = table_slots(max_entries)
    recs = gen_host(seed=601, n=n, n_keys=n_keys, dist=0)
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NO_FULL_CUT, max_batch=max_batch) as eng:
        eng.ingest(recs)
        assert eng.stats()["spills"] > 0
        all_keys = np.unique(keys_of_recs(recs), axis=0)
        assert len(all_keys) > slots
        q = np.concatenate([all_keys, absent_keys(602, 64, all_keys)])
        got = eng.lookup_flows(q)
        evicted = eng.evict_ex()
        assert len(evicted[0]) == slots
        wb, wf = expected(evicted, q)
        assert wf.sum() == slots and not wf[len(all_keys):].any()
        check_lookup(got, wb, wf)


def test_physically_full_emul(engine_emul):
    check_physically_full(700, 1_060, 1 << 20, max_batch=600)     # 1024 slots, ~1,059 keys


@pytest.mark.gpu
def test_physically_full_gpu():
    check_physically_full(180_000, 800_000, 400_000, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 7. non-blocking
def check_nonblocking_sequential(n, n_keys, mode):
    import netobserv_ebpf_agent_b200 as fa
    a = gen_host(seed=701, n=n, n_keys=n_keys, dist=1)
    b = gen_host(seed=702, n=n, n_keys=n_keys, dist=1, first=n)
    ka, kb = np.unique(keys_of_recs(a), axis=0), np.unique(keys_of_recs(b), axis=0)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_NONBLOCKING_EVICT) as eng:
        eng.ingest(a)
        assert eng.lookup_flows(ka)[6].all()
        first = eng.evict_ex()
        assert not eng.lookup_flows(ka)[6].any()                   # evicted keys miss once fa_evict returns
        eng.ingest(b)
        got = eng.lookup_flows(np.concatenate([kb, ka]))
        second = eng.evict_ex()
        wb, wf = expected(second, np.concatenate([kb, ka]))
        assert wf[:len(kb)].all()
        check_lookup(got, wb, wf)
        assert len(first[0]) == len(ka)


def check_nonblocking_concurrent(n, n_keys, max_entries, max_batch, chunk):
    """An evictor thread against a thread that alternates ingest and lookup: every lookup row is its key's flow or
    zero, and the generations, re-folded, equal the oracle's fold of the whole stream.  The last chunk is ingested
    after the evictor stops, so that its keys are found for certain and compared with the final eviction."""
    import netobserv_ebpf_agent_b200 as fa
    from test_nonblocking_evict import refold
    recs = gen_host(seed=703, n=n, n_keys=n_keys, dist=1)
    body, tail = recs[: n - chunk], recs[n - chunk:]
    evicted, stop = [], threading.Event()
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NONBLOCKING_EVICT, max_batch=max_batch) as eng:
        def evictor():
            while not stop.is_set():
                evicted.append(eng.evict(cap=max_entries).copy())
        t = threading.Thread(target=evictor)
        t.start()
        for lo in range(0, len(body), chunk):
            rc, took = eng.ingest(body[lo:lo + chunk])
            assert rc == 0 and took == min(chunk, len(body) - lo)
            q = np.unique(keys_of_recs(body[lo:lo + chunk]), axis=0)
            got = eng.lookup_flows(q)
            found = got[6] == 1
            assert not got[0][~found].any()
            assert np.array_equal(keys_of_recs(got[0][found]), q[found])
        stop.set(); t.join()
        eng.ingest(tail)
        q = np.unique(keys_of_recs(tail), axis=0)
        got = eng.lookup_flows(q)
        final = eng.evict_ex()
        wb, wf = expected(final, q)
        assert wf.all()
        check_lookup(got, wb, wf)
        evicted.append(final[0].copy())
    assert sum(1 for p in evicted if len(p)) >= 2
    assert np.array_equal(refold(evicted), refold([recs]))


@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_nonblocking_emul(engine_emul, mode):
    check_nonblocking_sequential(1_500, 500, mode)


def test_nonblocking_concurrent_emul(engine_emul):
    check_nonblocking_concurrent(8_000, 400, 1 << 11, 1_024, 1_000)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1], ids=["accounter", "kmap"])
def test_nonblocking_gpu(mode):
    check_nonblocking_sequential(600_000, 150_000, mode)


@pytest.mark.gpu
def test_nonblocking_concurrent_gpu():
    check_nonblocking_concurrent(2_000_000, 300_000, 1 << 20, 1 << 17, 1 << 16)


# ---------------------------------------------------------------------------------------------------- 8. placement
def lookup_filled(eng, keys, key_mem, device, found_mem, on_gpu):
    """fa_lookup_flows with keys in pageable / pinned / device memory, every block pre-filled with 0xFF in host memory or,
    where device[i] is set, in device memory, and found in host / device memory or NULL -> (blocks, found, n_found)."""
    from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib
    m = len(keys)
    held = []

    def dev_buf(nbytes, fill):
        if on_gpu:
            import torch
            b = torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda"); held.append(b)
            return b.data_ptr(), lambda: b.cpu().numpy()
        b = C.c_void_p(); check(lib().fa_device_alloc(eng._h, nbytes, C.byref(b))); C.memset(b.value, fill, nbytes)
        held.append(b)
        return b.value, lambda: np.frombuffer(C.string_at(b.value, nbytes), np.uint8).copy()

    if key_mem == "pageable":
        kp = keys.ctypes.data
    elif key_mem == "pinned":
        p = C.c_void_p(); check(lib().fa_host_alloc(keys.nbytes, C.byref(p))); C.memmove(p.value, keys.ctypes.data, keys.nbytes)
        kp = p.value
    else:
        kp, _ = dev_buf(keys.nbytes, 0)
        if on_gpu:
            import torch
            held[-1].copy_(torch.from_numpy(keys.reshape(-1).copy()))
        else:
            C.memmove(kp, keys.ctypes.data, keys.nbytes)
    ptrs, reads = [], []
    for w, dev in zip(WIDTHS, device):
        if dev:
            p, r = dev_buf(m * w, 0xFF)
        else:
            b = np.full(m * w, 0xFF, np.uint8); held.append(b); p = b.ctypes.data; r = (lambda b=b: b)
        ptrs.append(p); reads.append(r)
    fread = None
    if found_mem == "host":
        fb = np.full(m, 0xFF, np.uint8); held.append(fb); fp = fb.ctypes.data; fread = lambda: fb  # noqa: E731
    elif found_mem == "device":
        fp, fread = dev_buf(m, 0xFF)
    else:
        fp = None
    got = C.c_size_t(0)
    check(lib().fa_lookup_flows(eng._h, kp, m, C.byref(EvictOut(*ptrs)), fp, C.byref(got)))
    blocks = [r()[: m * w].reshape(m, w) for r, w in zip(reads, WIDTHS)]
    found = fread() if fread else None
    for b in held:
        if isinstance(b, C.c_void_p):
            check(lib().fa_device_free(eng._h, b))
    if key_mem == "pinned":
        lib().fa_host_free(kp)
    return blocks, found, got.value


PLACEMENTS = [(False,) * 6, (True,) * 6] + [tuple(i == j for j in range(6)) for i in range(6)]


def check_placement(n, n_keys, mode, rtt, on_gpu, max_batch):
    import netobserv_ebpf_agent_b200 as fa
    recs = gen_host(seed=801, n=n, n_keys=n_keys, dist=1)
    keys = np.unique(keys_of_recs(recs), axis=0)
    extra = keys_of(802, 8)
    produced = {"records", "additional", "rtt_min", "present"} if rtt else {"records"}
    rng = np.random.default_rng(803)
    q = query_of(np.concatenate([keys, extra]), absent_keys(804, len(keys) // 4, keys), rng, 20)
    q39 = q.copy()
    q39[:, 39] = rng.integers(1, 256, len(q), dtype=np.uint8)        # key byte 39 is padding: ignored
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=fa.FA_F_ENABLE_RTT if rtt else 0, max_batch=max_batch) as eng:
        eng.ingest(recs)
        if rtt:
            eng.ingest_additional(make_add(np.random.default_rng(805), np.concatenate([keys, extra]), n // 4))
        want = eng.lookup_flows(q)
        runs = [("pageable", PLACEMENTS[0], "host"), ("pinned", PLACEMENTS[1], "device"), ("device", PLACEMENTS[0], None)]
        runs += [(("pageable", "pinned", "device")[i % 3], d, ("host", "device", None)[i % 3]) for i, d in enumerate(PLACEMENTS)]
        for key_mem, device, found_mem in runs:
            for qq in (q, q39):
                blocks, found, n_found = lookup_filled(eng, qq, key_mem, device, found_mem, on_gpu)
                assert n_found == int(want[6].sum())
                if found is not None:
                    assert np.array_equal(found, want[6]), (key_mem, found_mem)
                for name, g, w in zip(BLOCKS, blocks, rows(want[:6])):
                    if name not in produced:
                        assert not g.any(), (device, name)
                    assert np.array_equal(g, w), (key_mem, device, name)
                    assert not g[want[6] == 0].any()


@pytest.mark.parametrize("mode,rtt", [(0, False), (0, True), (1, False), (1, True)])
def test_placement_emul(engine_emul, mode, rtt):
    check_placement(1_000, 300, mode, rtt, on_gpu=False, max_batch=256)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rtt", [(0, False), (0, True), (1, False), (1, True)])
def test_placement_gpu(mode, rtt):
    check_placement(600_000, 200_000, mode, rtt, on_gpu=True, max_batch=1 << 16)


# ---------------------------------------------------------------------------------------------------- 9. errors
def check_errors(n, n_keys, on_gpu):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_INVAL, EvictOut, lib
    recs = gen_host(seed=901, n=n, n_keys=n_keys, dist=1)
    keys = keys_of_recs(recs[:4])
    out = np.full((4, O.REC), 0xAB, np.uint8)
    found = np.full(4, 0xAB, np.uint8)
    got = C.c_size_t(7)
    with fa.FlowAggEngine(4 * n_keys) as eng:
        eng.ingest(recs)
        live = eng.live_flows()
        buf = DevBuf(eng, 4 * O.ID + 8, None if on_gpu else lib())
        buf.write(np.concatenate([np.zeros(4, np.uint8), keys.reshape(-1)]))
        before = eng.stats()
        good, no_rec = EvictOut(records=out.ctypes.data), EvictOut()
        kp, fp = keys.ctypes.data, found.ctypes.data
        cases = [(None, kp, 4, C.byref(good), fp, C.byref(got)), (eng._h, kp, 4, None, fp, C.byref(got)),
                 (eng._h, kp, 4, C.byref(no_rec), fp, C.byref(got)), (eng._h, kp, 4, C.byref(good), fp, None),
                 (eng._h, None, 4, C.byref(good), fp, C.byref(got)), (eng._h, buf.ptr + 4, 4, C.byref(good), fp, C.byref(got))]
        for c in cases:
            assert lib().fa_lookup_flows(*c) == FA_E_INVAL, c
            assert got.value == 7
        assert (out == 0xAB).all() and (found == 0xAB).all()
        assert lib().fa_lookup_flows(eng._h, None, 0, C.byref(good), fp, C.byref(got)) == 0 and got.value == 0
        assert lib().fa_lookup_flows(eng._h, kp, 0, C.byref(good), None, C.byref(got)) == 0 and got.value == 0
        assert (out == 0xAB).all() and (found == 0xAB).all()
        assert eng.stats() == before
        assert eng.live_flows() == live
        buf.free()
        assert lookup_raw(eng, keys)[1] == 4
        assert_rows_equal(O.sort_records(eng.evict()), O.sort_records(oracle_flows([recs], 4 * n_keys)), "eviction")


def test_errors_emul(engine_emul):
    check_errors(1_000, 300, on_gpu=False)


@pytest.mark.gpu
def test_errors_gpu():
    check_errors(200_000, 50_000, on_gpu=True)


# ---------------------------------------------------------------------------------------------------- large lookups
@pytest.mark.gpu
def test_device_keys_and_outputs_gpu():
    """10^6 device-resident keys (half of them absent) against 2·10^6 flows ingested from device memory, with device
    records and found blocks."""
    import netobserv_ebpf_agent_b200 as fa
    import torch
    from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib
    recs = gen_host(seed=1001, n=3_000_000, n_keys=2_500_000, dist=0)
    max_entries = 3_000_000
    want = oracle_flows([recs], max_entries)
    live_keys = keys_of_recs(want)
    rng = np.random.default_rng(1002)
    q = np.concatenate([live_keys[rng.choice(len(live_keys), 500_000, replace=False)], absent_keys(1003, 500_000, live_keys)])
    q = q[rng.permutation(len(q))]
    m = len(q)
    with fa.FlowAggEngine(max_entries) as eng:
        buf = DevBuf(eng, recs.size, None)
        buf.write(recs)
        assert eng.ingest(buf.ptr, len(recs)) == (fa.FA_OK, len(recs))
        dk = torch.from_numpy(q.reshape(-1).copy()).cuda()
        out = torch.full((m * O.REC,), 0xFF, dtype=torch.uint8, device="cuda")
        found = torch.full((m,), 0xFF, dtype=torch.uint8, device="cuda")
        got = C.c_size_t(0)
        check(lib().fa_lookup_flows(eng._h, dk.data_ptr(), m, C.byref(EvictOut(records=out.data_ptr())), found.data_ptr(),
                                    C.byref(got)))
        wb, wf = expected((want,), q)
        assert got.value == int(wf.sum()) == 500_000
        assert np.array_equal(found.cpu().numpy(), wf)
        assert_rows_equal(out.cpu().numpy().reshape(m, O.REC), wb[0], "device records")
