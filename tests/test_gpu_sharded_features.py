"""Multi-GPU feature samples through the sharded C ABI (csrc/sharded.cu): fa_sharded_ingest_additional / _dns /
_pkt_drops and fa_sharded_evict_ex against one engine fed the same calls and against the oracle's FlowMap, bit for bit
in every block.  Shards run as [0] x k on one GPU (the route and the per-segment folds are the same code; only the
links differ), and on every visible GPU when there are several."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_lib as O
from common import gen_host
from test_gpu_features import keys_of, make_add, make_dns
from test_pktdrop import make_drops

pytestmark = pytest.mark.gpu

FEATS = 1 | 2 | 32                          # FA_F_ENABLE_RTT | FA_F_ENABLE_DNS | FA_F_ENABLE_PKT_DROP
BLOCKS = ("records", "dns", "additional", "pkt_drops", "rtt_min", "present")


class Sharded:
    """The fa_sharded_* calls this test needs, over ctypes."""

    def __init__(self, devices, max_entries, flags, max_batch):
        from netobserv_ebpf_agent_b200._lib import FA_ABI_VERSION, Config, lib
        self.L = lib()
        cfg = Config(abi_version=FA_ABI_VERSION, device=0, mode=0, flags=flags, max_entries=max_entries, max_batch=max_batch)
        self.h = C.c_void_p()
        self.check(self.L.fa_sharded_create(C.byref(cfg), (C.c_int32 * len(devices))(*devices), len(devices), C.byref(self.h)))

    def check(self, rc):
        from netobserv_ebpf_agent_b200._lib import FlowAggError
        if rc < 0:
            raise FlowAggError(rc, self.L.fa_sharded_last_error().decode(errors="replace"))
        return rc

    def ingest(self, recs):
        self.check(self.L.fa_sharded_ingest(self.h, recs.ctypes.data, len(recs)))

    def ingest_samples(self, kind, samples):
        f = (self.L.fa_sharded_ingest_additional, self.L.fa_sharded_ingest_dns, self.L.fa_sharded_ingest_pkt_drops)[kind]
        self.check(f(self.h, np.ascontiguousarray(samples).ctypes.data, len(samples)))

    def live_flows(self):
        n = C.c_size_t(0)
        self.check(self.L.fa_sharded_live_flows(self.h, C.byref(n)))
        return n.value

    def evict_ex(self, cap=None):
        from netobserv_ebpf_agent_b200._lib import EvictOut
        cap = max(self.live_flows(), 1) if cap is None else cap
        out = (np.zeros((cap, 144), np.uint8), np.zeros((cap, 64), np.uint8), np.zeros((cap, 32), np.uint8),
               np.zeros((cap, 32), np.uint8), np.zeros(cap, np.uint64), np.zeros(cap, np.uint8))
        o = EvictOut(*[a.ctypes.data for a in out])
        got = C.c_size_t(0)
        self.check(self.L.fa_sharded_evict_ex(self.h, C.byref(o), cap, C.byref(got)))
        return tuple(a[:got.value] for a in out)

    def stats(self):
        from netobserv_ebpf_agent_b200._lib import Stats
        s, nv, ov = Stats(), C.c_uint64(0), C.c_uint64(0)
        self.check(self.L.fa_sharded_get_stats(self.h, C.byref(s), C.byref(nv), C.byref(ov)))
        return s.as_dict(), nv.value, ov.value

    def close(self):
        if self.h:
            self.L.fa_sharded_destroy(self.h)
            self.h = None


def same_rows(a, b, what):
    pa, pb = O.sort_perm(a[0]), O.sort_perm(b[0])
    assert len(pa) == len(pb), (what, len(pa), len(pb))
    for name, x, y in zip(BLOCKS, a, b):
        xs, ys = x.reshape(len(x), -1)[pa], y.reshape(len(y), -1)[pb]
        if not np.array_equal(xs, ys):
            bad = np.nonzero((xs != ys).any(axis=1))[0]
            raise AssertionError(f"{what} {name}: {len(bad)} of {len(xs)} rows differ; first:\n {xs[bad[0]].tolist()}\n {ys[bad[0]].tolist()}")
    return len(pa)


def _device_sets():
    sets = [[0], [0, 0], [0, 0, 0, 0]]
    if torch.cuda.device_count() > 1:
        sets.append(list(range(torch.cuda.device_count())))
    return sets


def _calls(rng, gen, keys, hot):
    """Uneven calls of every kind; 1 in 6 samples belongs to one hot flow, so it reaches its owner from every source
    within a round and across rounds."""
    out = []
    plan = [("base", 5_000), (0, 7_001), (1, 2_500), (2, 11_000), ("base", 3_333), (1, 9_100), (0, 100), (2, 1), (1, 1),
            (0, 4_097), (2, 2_999)]
    for what, n in plan:
        if what == "base":
            out.append(("base", gen_host(seed=81, n=n, n_keys=3_000, dist=1, first=gen[0])))
            gen[0] += n
        else:
            s = (make_add, make_dns, make_drops)[what](rng, keys, n)
            s["id"][rng.random(n) < 1 / 6] = hot
            out.append((what, s))
    return out


@pytest.mark.parametrize("devices", _device_sets(), ids=lambda d: "x".join(map(str, d)))
def test_sharded_samples_equal_one_engine_and_the_oracle(devices):
    import netobserv_ebpf_agent_b200 as fa
    rng = np.random.default_rng(80 + len(devices))
    base_keys = np.unique(gen_host(seed=81, n=20_000, n_keys=3_000, dist=1)[:, :40], axis=0)
    keys = np.concatenate([base_keys, keys_of(82, 800)])                    # some flows only through samples
    hot = keys[:1]
    gen = [0]
    sh = Sharded(devices, 1 << 16, FEATS, max_batch=3_000)                  # rounds of len(devices) x 3000: calls span several
    try:
        with fa.FlowAggEngine(1 << 16, flags=FEATS, max_batch=4_096) as one:
            n_in = [0, 0, 0]
            for generation in range(2):                                     # the second one after an eviction
                om = O.FlowMap()
                calls = _calls(rng, gen, keys, hot)
                for what, x in calls if generation == 0 else calls[:5]:
                    if what == "base":
                        sh.ingest(x); one.ingest(x); om.account(x)
                    else:
                        sh.ingest_samples(what, x)
                        (one.ingest_additional, one.ingest_dns, one.ingest_pkt_drops)[what](x)
                        (om.fold_additional, om.fold_dns, om.fold_drops)[what](x)
                        n_in[what] += len(x)
                st, _, overflow = sh.stats()
                assert [st["additional_ingested"], st["dns_ingested"], st["pkt_drops_ingested"]] == n_in
                assert st["spills"] == 0 and overflow == 0
                got = sh.evict_ex()
                n = same_rows(got, one.evict_ex(), "one engine")
                assert same_rows(got, om.evict_ex(), "oracle") == n > 1_000
                assert sh.live_flows() == 0 and one.live_flows() == 0
    finally:
        sh.close()


def test_sharded_sample_errors():
    from netobserv_ebpf_agent_b200._lib import FA_E_2BIG, FA_E_INVAL, FlowAggError
    with pytest.raises(FlowAggError) as ei:
        Sharded([0, 0], 1 << 12, FEATS | 4, max_batch=1_000)                # FA_F_ENABLE_SKETCH
    assert ei.value.code == FA_E_INVAL
    sh = Sharded([0, 0], 1 << 12, 1, max_batch=1_000)                       # RTT only
    try:
        rng = np.random.default_rng(5)
        keys = keys_of(83, 50)
        for kind in (1, 2):
            with pytest.raises(FlowAggError) as ei:
                sh.ingest_samples(kind, (make_add, make_dns, make_drops)[kind](rng, keys, 10))
            assert ei.value.code == FA_E_INVAL
        sh.ingest_samples(0, make_add(rng, keys, 2_000))
        with pytest.raises(FlowAggError) as ei:
            sh.evict_ex(cap=10)
        assert ei.value.code == FA_E_2BIG
        assert sh.live_flows() == 50                                        # nothing was evicted
        got = sh.evict_ex()
        assert len(got[0]) == 50 and (got[5] == 2).all() and sh.live_flows() == 0
    finally:
        sh.close()
