"""The two engine-level pieces of the multi-GPU sample exchange, on the CPU engine emulation (csrc/sharded.cu itself is
not emulated; tests/test_gpu_sharded_features.py runs it on the device):

  fa_route_peer_samples      the STABLE route: each sample lands once, in its owner's segment, in slice order;
  fa_ingest_samples_counted  the fold of a segment whose count lives in device memory: segments folded one after the
                             other give the rows fa_ingest_additional / _dns / _pkt_drops give for the samples
                             concatenated in segment order, bit for bit in every block."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_gpu_features import keys_of, make_add, make_dns
from test_pktdrop import compare_ex, make_drops

KINDS = {0: (O.ADDREC_DTYPE, 72), 1: (O.DNSREC_DTYPE, 104), 2: (O.DROPREC_DTYPE, 72)}
GUARD = 5                                   # samples of sentinel bytes after every segment


def _owners(samples, n_shards):
    from netobserv_ebpf_agent_b200.sharded import owner_of
    return owner_of(samples.view(np.uint8).reshape(len(samples), -1)[:, :40], n_shards)


def _route(eng, kind, samples, n_shards, self_shard, seg_cap, n_dev=None, max_n=None):
    """Route `samples` (host memory: the emulation's device memory) into n_shards fresh segments -> (segments as uint8
    arrays of seg_cap + GUARD samples, count words, overflow words)."""
    from netobserv_ebpf_agent_b200._lib import check, lib
    rb = KINDS[kind][1]
    segs = [np.full((seg_cap + GUARD) * rb, 0xEE, np.uint8) for _ in range(n_shards)]
    counts = [np.full(1, 0xDEAD, np.uint64) for _ in range(n_shards)]
    over = np.zeros(2, np.uint64)
    nd = None if n_dev is None else np.array([n_dev], np.uint64)
    bufs = (C.c_void_p * n_shards)(*[s.ctypes.data for s in segs])
    cnts = (C.c_void_p * n_shards)(*[c.ctypes.data for c in counts])
    raw = np.ascontiguousarray(samples).view(np.uint8)
    check(lib().fa_route_peer_samples(eng._h, kind, raw.ctypes.data, None if nd is None else nd.ctypes.data,
                                      len(samples) if max_n is None else max_n, n_shards, self_shard, bufs, cnts, seg_cap,
                                      over.ctypes.data))
    return segs, [int(c[0]) for c in counts], over


def _samples(kind, rng, keys, n):
    return (make_add, make_dns, make_drops)[kind](rng, keys, n)


# every sample size, 1 to 5 shards
@pytest.mark.parametrize("kind,n_shards", [(0, 1), (1, 2), (2, 3), (1, 4), (0, 5)])
def test_route_is_stable_and_exactly_once(engine_emul, kind, n_shards):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(100 + 10 * kind + n_shards)
    keys = keys_of(40 + kind, 37)
    rb = KINDS[kind][1]
    with fa.FlowAggEngine(1024, flags=fa.FA_F_NO_FULL_CUT, max_batch=2048) as eng:
        # counts below, at and above one tile of 256, not multiples of it; n_dev below max_n
        for n, n_dev in ((1, None), (255, None), (600, None), (700, 517), (700, 0)):
            s = _samples(kind, rng, keys, n)
            own = _owners(s, n_shards)
            eff = n if n_dev is None else n_dev
            segs, counts, over = _route(eng, kind, s, n_shards, n_shards - 1, seg_cap=n, n_dev=n_dev, max_n=n)
            assert over.tolist() == [0, 0]
            for o in range(n_shards):
                want = s[:eff][own[:eff] == o].view(np.uint8).reshape(-1)      # in slice order: arrays, not multisets
                assert counts[o] == len(want) // rb
                assert np.array_equal(segs[o][:len(want)], want), (n, n_dev, o)
                assert (segs[o][len(want):] == 0xEE).all()                     # nothing past the run
            assert sum(counts) == eff


@pytest.mark.parametrize("kind", [1, 2])
def test_route_guards_a_segment_that_would_overflow(engine_emul, kind):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(7 + kind)
    keys = keys_of(50, 3)
    rb = KINDS[kind][1]
    s = _samples(kind, rng, keys, 600)
    own = _owners(s, 2)
    seg_cap = 150
    with fa.FlowAggEngine(1024, flags=fa.FA_F_NO_FULL_CUT, max_batch=2048) as eng:
        segs, counts, over = _route(eng, kind, s, 2, 0, seg_cap=seg_cap)
    lost = 0
    for o in range(2):
        mine = s[own == o]
        assert counts[o] == len(mine)                                           # the count says what was sent ...
        keep = min(len(mine), seg_cap)
        lost += len(mine) - keep
        assert np.array_equal(segs[o][:keep * rb], mine[:keep].view(np.uint8).reshape(-1))   # ... the first seg_cap are stored
        assert (segs[o][seg_cap * rb:] == 0xEE).all()                           # nothing out of bounds
    assert lost > 0 and int(over[0]) == lost and int(over[1]) == 0


def test_route_counts_a_device_count_above_max_n(engine_emul):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(3)
    s = make_add(rng, keys_of(51, 9), 300)
    with fa.FlowAggEngine(1024, flags=fa.FA_F_NO_FULL_CUT, max_batch=2048) as eng:
        segs, counts, over = _route(eng, 0, s, 2, 1, seg_cap=300, n_dev=320, max_n=300)
    assert sum(counts) == 300 and int(over[0]) == 20


def test_route_and_fold_errors(engine_emul):
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import FA_E_INVAL, lib
    L = lib()
    buf = np.zeros(1024, np.uint64)
    bufs = (C.c_void_p * 2)(buf.ctypes.data, buf.ctypes.data)
    over = np.zeros(2, np.uint64)
    with fa.FlowAggEngine(1024, flags=fa.FA_F_NO_FULL_CUT | fa.FA_F_ENABLE_RTT, max_batch=512) as eng:
        p = buf.ctypes.data
        assert L.fa_route_peer_samples(eng._h, 3, p, None, 4, 2, 0, bufs, bufs, 8, over.ctypes.data) == FA_E_INVAL
        assert L.fa_route_peer_samples(eng._h, 0, p, None, 4, 2, 2, bufs, bufs, 8, over.ctypes.data) == FA_E_INVAL
        assert L.fa_route_peer_samples(eng._h, 0, p + 4, None, 4, 2, 0, bufs, bufs, 8, over.ctypes.data) == FA_E_INVAL
        assert L.fa_route_peer_samples(eng._h, 0, p, None, 4, 17, 0, bufs, bufs, 8, over.ctypes.data) == FA_E_INVAL
        assert L.fa_ingest_samples_counted(eng._h, 1, p, p, 4, 1) == FA_E_INVAL            # created without DNS
        assert b"FA_F_ENABLE_DNS" in L.fa_last_error()
        assert L.fa_ingest_samples_counted(eng._h, 0, p, p, 513, 1) == FA_E_INVAL          # past max_batch
        assert L.fa_ingest_samples_counted(eng._h, 0, p, None, 4, 1) == FA_E_INVAL
    with fa.FlowAggEngine(1024, flags=fa.FA_F_ENABLE_RTT, max_batch=512) as eng:
        assert L.fa_ingest_samples_counted(eng._h, 0, buf.ctypes.data, buf.ctypes.data, 4, 1) == FA_E_INVAL   # full cut on
        assert b"FA_F_NO_FULL_CUT" in L.fa_last_error()


def _fold_segments(eng, kind, segments, seg_cap):
    """Lay the segments into one buffer of len(segments) x seg_cap samples (the gaps full of junk) and fold them in order
    with fa_ingest_samples_counted; every count word is zeroed by the fold."""
    from netobserv_ebpf_agent_b200._lib import check, lib
    dt, rb = KINDS[kind]
    buf = np.frombuffer(np.random.default_rng(kind).integers(0, 256, len(segments) * seg_cap * rb, dtype=np.uint8).tobytes(), dtype=dt).copy()
    words = np.zeros(len(segments), np.uint64)
    for i, seg in enumerate(segments):
        buf[i * seg_cap:i * seg_cap + len(seg)] = seg
        words[i] = len(seg)
    raw = buf.view(np.uint8)
    for i in range(len(segments)):
        check(lib().fa_ingest_samples_counted(eng._h, kind, raw.ctypes.data + i * seg_cap * rb, words.ctypes.data + 8 * i, seg_cap, 1))
    assert (words == 0).all()


def test_counted_fold_of_segments_equals_one_stream(engine_emul):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(61)
    base = gen_host(seed=61, n=800, n_keys=60, dist=1)
    keys = np.concatenate([np.unique(base[:, :40], axis=0), keys_of(62, 15)])      # some flows only through features
    hot = keys[:1]
    seg_cap = 280
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP
    with fa.FlowAggEngine(1 << 12, flags=flags | fa.FA_F_NO_FULL_CUT, max_batch=1024) as seg_eng, \
            fa.FlowAggEngine(1 << 12, flags=flags, max_batch=1024) as one_eng:
        for eng in (seg_eng, one_eng):
            eng.ingest(base[:400])
        for rnd in range(2):
            for kind in (0, 1, 2):
                # uneven segments, an empty one, a full one; the hot flow in every non-empty segment
                sizes = [(120, 0, 280, 37), (280, 5, 0, 199)][rnd]
                segments = []
                for n in sizes:
                    seg = _samples(kind, rng, keys, n)
                    if n:
                        seg["id"][rng.integers(0, n, max(1, n // 8))] = hot
                    segments.append(seg)
                _fold_segments(seg_eng, kind, segments, seg_cap)
                (one_eng.ingest_additional, one_eng.ingest_dns, one_eng.ingest_pkt_drops)[kind](np.concatenate(segments))
            if rnd == 0:
                for eng in (seg_eng, one_eng):
                    eng.ingest(base[400:])
        assert seg_eng.stats()["spills"] == 0
        got, want = seg_eng.evict_ex(), one_eng.evict_ex()
        gp, op = O.sort_perm(got[0]), O.sort_perm(want[0])
        assert len(gp) == len(op) > 60
        for name, g, o in zip(("records", "dns", "additional", "pkt_drops", "rtt_min", "present"), got, want):
            assert np.array_equal(g.reshape(len(g), -1)[gp], o.reshape(len(o), -1)[op]), name
        # a second generation starts from scratch on both
        seg = make_dns(rng, keys, 90)
        _fold_segments(seg_eng, 1, [seg[:40], seg[40:]], 64)
        one_eng.ingest_dns(seg)
        got, want = seg_eng.evict_ex(), one_eng.evict_ex()
        gp, op = O.sort_perm(got[0]), O.sort_perm(want[0])
        for name, g, o in zip(("records", "dns", "additional", "pkt_drops", "rtt_min", "present"), got, want):
            assert np.array_equal(g.reshape(len(g), -1)[gp], o.reshape(len(o), -1)[op]), name


def test_counted_fold_matches_the_oracle(engine_emul):
    """The same through the oracle's FlowMap: segments of all three kinds with per-sample random values."""
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(67)
    keys = keys_of(68, 25)
    om = O.FlowMap()
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP | fa.FA_F_NO_FULL_CUT
    with fa.FlowAggEngine(1 << 10, flags=flags, max_batch=512) as eng:
        for kind, fold in ((2, om.fold_drops), (0, om.fold_additional), (1, om.fold_dns)):
            segments = [_samples(kind, rng, keys, n) for n in (300, 17, 0, 256)]
            _fold_segments(eng, kind, segments, 300)
            fold(np.concatenate(segments))
        assert compare_ex(eng, om) == 25
