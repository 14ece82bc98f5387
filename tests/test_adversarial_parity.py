"""Adversarial streams for K1 and the table probes: keys built to collide in every hash-derived filter, timestamps at
uptime scale whose high words change inside a tile, per-CPU clocks that run out of order, and pre-aggregated records
whose packet counts carry past 32 bits.

The generator's keys have well-spread hashes, its timestamps stay below 2^32 and nearly every record has one packet,
so the parity tests elsewhere never reach the far side of K1's shortcuts: the election compares 23 hash bits before
the key, the hot-flow cache matches the low 32 bits of the slot hash, the pipelined probe looks at the home slot and
the next one, tile and cache folds keep 32-bit time windows and 32-bit packet sums.  Here every shortcut is made to
fail and the result is compared bit for bit with the oracle.

Every scenario runs twice: on the engine emulation (`engine_emul`, a few thousand records, CPU suite) and on the
device (`gpu`, 10^5 to 10^6 records, several batch sizes).

The hash is invertible (DESIGN.md §4): key_premix's last round is h = (h3 ^ w4) * P1, h ^= h >> 32, and fmix64 is a
bijection, so a key with any wanted premix or slot hash is solved for directly — pick bytes 0..31, solve for
w4 = bytes 32..39, keep the key when its byte 39 (masked out of the hash) comes out 0, about 1 try in 256."""
import ctypes

import numpy as np
import pytest

import oracle_lib as O
from common import assert_same_generations, gen_host, oracle_generations

# a wedged emulation (it is thousands of OS threads) must not hang the suite: pytest-timeout, if installed
pytestmark = pytest.mark.timeout(900)

M64 = (1 << 64) - 1
P1, P2 = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F
F1, F2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
P1_INV, F1_INV, F2_INV = pow(P1, -1, 1 << 64), pow(F1, -1, 1 << 64), pow(F2, -1, 1 << 64)
SKETCH_SEED = 0x5EED0F5EED


# ---------------------------------------------------------------------------------------------------- key builders
def fmix64(x):
    x ^= x >> 33; x = (x * F1) & M64; x ^= x >> 33; x = (x * F2) & M64; x ^= x >> 33
    return x


def unfmix64(x):
    """Inverse of fmix64 (x ^= x >> 33 is an involution on 64 bits, odd multipliers are invertible mod 2^64)."""
    x ^= x >> 33; x = (x * F2_INV) & M64; x ^= x >> 33; x = (x * F1_INV) & M64; x ^= x >> 33
    return x


def premix(key40):
    w = [int.from_bytes(bytes(key40[i * 8:(i + 1) * 8]), "little") for i in range(5)]
    w[4] &= 0x00FFFFFFFFFFFFFF
    h = 0x243F6A8885A308D3
    for wi, p, s in zip(w, (P1, P2, P1, P2, P1), (32, 29, 32, 29, 32)):
        h = ((h ^ wi) * p) & M64
        h ^= h >> s
    return h


def _prefix(head32):
    """key_premix state after the first four words (bytes 0..31)."""
    h = 0x243F6A8885A308D3
    for i, (p, s) in enumerate(((P1, 32), (P2, 29), (P1, 32), (P2, 29))):
        h = ((h ^ int.from_bytes(head32[i * 8:(i + 1) * 8], "little")) * p) & M64
        h ^= h >> s
    return h


def key_with_premix(target, rng):
    """A v4-mapped key whose premix is `target`: random addresses, w4 (ports, protocol, ICMP type / code) solved."""
    t_hi = target >> 32
    u = (((t_hi << 32) | ((target & 0xFFFFFFFF) ^ t_hi)) * P1_INV) & M64      # = h3 ^ w4
    v4 = bytes(10) + b"\xff\xff"
    while True:
        head = v4 + rng.bytes(4) + v4 + rng.bytes(4)
        w4 = u ^ _prefix(head)
        if w4 >> 56 == 0:
            return np.frombuffer(head + w4.to_bytes(8, "little"), dtype=np.uint8)


def key_with_slot_hash(value, rng):
    return key_with_premix(unfmix64(value), rng)


def table_slots(max_entries):
    """fa_create's table size: load factor <= 0.75 at max_entries, at least 1024 slots."""
    want, slots = (4 * max_entries + 2) // 3, 1024
    while slots < want:
        slots <<= 1
    return slots


ELECTION_BITS = (0x7FFFFF << 16) | (511 << 40)      # (h >> 16) & 0x7FFFFF and (h >> 40) & 511: K1's tile election


def key_families(seed, slots, n_full=64, n_chain=300, n_way=32, n_elect=32):
    """The four families (dict name -> (m, 40) uint8 keys) for a table of `slots` slots:
    full: one identical 64-bit premix (so identical slot, owner, count-min and HyperLogLog hashes);
    chain_last / chain_mid: distinct premixes, one home slot (the last slot, so that probes wrap to slot 0; and one in
    the middle), longer than a tile;
    way: identical low 32 bits of the slot hash (hot-cache ways and hash tag), different high words;
    elect: identical election bits, everything else different."""
    rng = np.random.default_rng(seed)
    r64 = lambda: int(rng.integers(0, 1 << 62)) << 2 | int(rng.integers(0, 4))   # noqa: E731
    mask = slots - 1
    fam = {}
    h = r64()
    fam["full"] = [key_with_premix(h, rng) for _ in range(n_full)]
    fam["chain_last"] = [key_with_slot_hash((r64() & ~mask) | mask, rng) for _ in range(n_chain)]
    mid = (slots // 2 + 17) & mask
    fam["chain_mid"] = [key_with_slot_hash((r64() & ~mask) | mid, rng) for _ in range(n_chain // 4)]
    low = r64() & 0xFFFFFFFF
    fam["way"] = [key_with_slot_hash((r64() & ~0xFFFFFFFF) | low, rng) for _ in range(n_way)]
    e = r64() & ELECTION_BITS
    fam["elect"] = [key_with_slot_hash((r64() & ~ELECTION_BITS) | e, rng) for _ in range(n_elect)]
    return {k: np.stack(v) for k, v in fam.items()}


def all_keys(fam):
    return np.concatenate(list(fam.values()))


# ---------------------------------------------------------------------------------------------------- stream transforms
UPTIME_NS = 1_700_000_000_000_000          # ~19.7 days of uptime: every timestamp is far above 2^32


def mix_keys(recs, keys, rng, frac=0.4, varying=0):
    """Give a share of the records a colliding key.  With constant descriptors (varying=0) every colliding key keeps
    one descriptor, taken from a template record, so that its folds take the fast paths."""
    r = recs.copy()
    idx = np.nonzero(rng.random(len(r)) < frac)[0]
    which = np.minimum(rng.zipf(1.3, len(idx)) - 1, len(keys) - 1)     # a hot head and a long tail
    which = rng.permutation(len(keys))[which]
    r[idx, :40] = keys[which]
    if not varying:
        tmpl = recs[rng.integers(0, len(recs), len(keys))]
        r[idx, 68:70] = tmpl[which, 68:70]
        r[idx, 72:] = tmpl[which, 72:]
    return r


def uptime_times(recs, rng, zero_frac=0.1, per_cpu=8, chunk=24):
    """Uptime-scale timestamps that cross 2^32 boundaries (of end, and of 0 - start) inside most 256-record tiles,
    from `per_cpu` sub-streams with skewed clocks merged in chunks (non-monotone), and ~10 % zero starts / ends."""
    r = recs.copy()
    v = r.view(O.REC_DTYPE).reshape(-1)
    n = len(r)
    step = (1 << 32) // 160
    base = UPTIME_NS + np.arange(n, dtype=np.uint64) * np.uint64(step)
    skew = rng.integers(0, 1 << 34, per_cpu).astype(np.uint64)
    cpu = (np.arange(n) // chunk) % per_cpu
    start = base + skew[cpu] + rng.integers(0, 1 << 20, n).astype(np.uint64)
    end = start + rng.integers(0, 3 << 31, n).astype(np.uint64)
    start[rng.random(n) < zero_frac] = 0
    end[rng.random(n) < zero_frac] = 0
    v["start"], v["end"] = start, end
    return r


def pre_aggregate(recs, rng):
    """Records that are themselves flows: packet counts whose sums carry past 2^32, byte counts near 2^64, and
    start < end across a 2^32 boundary."""
    r = recs.copy()
    v = r.view(O.REC_DTYPE).reshape(-1)
    n = len(r)
    v["packets"] = rng.choice(np.array([1, 7, 1 << 31, 0xFFFFFFF0], dtype=np.uint32), n)
    v["bytes"] = rng.choice(np.array([60, 0xFFFFFFFF, (1 << 64) - 1, (1 << 64) - 0x1000, (1 << 63) + 5], dtype=np.uint64), n)
    s = v["start"]
    cross = (s != 0) & (rng.random(n) < 0.5)
    v["end"][cross] = (s[cross] | np.uint64(0xFFFFFFFF)) + rng.integers(1, 1 << 20, int(cross.sum())).astype(np.uint64)
    return r


def adversarial_stream(seed, n, slots, varying=0, pre_agg=False, frac=0.4, n_chain=300, bg_keys=None, dist=1):
    """(records, colliding keys): a Zipf (dist=1) or uniform background mixed with the four key families, uptime
    timestamps."""
    rng = np.random.default_rng(seed)
    fam = key_families(seed, slots, n_chain=n_chain)
    keys = all_keys(fam)
    bg = gen_host(seed=seed, n=n, n_keys=bg_keys or max(n // 16, 64), dist=dist, varying=varying)
    r = uptime_times(mix_keys(bg, keys, rng, frac, varying), rng)
    if pre_agg:
        r = pre_aggregate(r, rng)
    return r, keys


# ---------------------------------------------------------------------------------------------------- device buffers
class DevBuf:
    """Device memory for a record stream: a CUDA tensor on the GPU, fa_device_alloc memory (host memory) on the
    emulation."""

    def __init__(self, eng, nbytes, emul):
        self.emul, self.eng = emul, eng
        if emul is not None:
            self.p = ctypes.c_void_p()
            assert emul.fa_device_alloc(eng._h, max(nbytes, 16), ctypes.byref(self.p)) == 0
            self.ptr = self.p.value
        else:
            import torch
            self.t = torch.zeros(max(nbytes, 16), dtype=torch.uint8, device="cuda")
            self.ptr = self.t.data_ptr()

    def write(self, arr):
        b = O.as_bytes(arr)
        if self.emul is not None:
            ctypes.memmove(self.ptr, b.ctypes.data, b.size)
        else:
            import torch
            self.t[: b.size].copy_(torch.from_numpy(b.copy()))

    def read(self, nbytes):
        if self.emul is not None:
            out = np.zeros(nbytes, dtype=np.uint8)
            ctypes.memmove(out.ctypes.data, self.ptr, nbytes)
            return out
        return self.t[:nbytes].cpu().numpy()

    def free(self):
        if self.emul is not None and self.p:
            self.emul.fa_device_free(self.eng._h, self.p)
            self.p = ctypes.c_void_p()


# ---------------------------------------------------------------------------------------------------- scenarios
def oracle_sketch(recs, lw, depth, p):
    b = O.as_bytes(recs)
    cms = np.zeros(depth << lw, dtype=np.uint64)
    hll = np.zeros(1 << p, dtype=np.uint8)
    O.lib().oracle_cms_update(cms.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), lw, depth, SKETCH_SEED, O._p(b), b.size // O.REC)
    O.lib().oracle_hll_update(O._p(hll), p, SKETCH_SEED, O._p(b), b.size // O.REC)
    return cms, hll


def check_sketch(eng, recs, keys, lw, depth, p):
    cms, hll = eng.sketch_export(lw, depth, p)
    want_cms, want_hll = oracle_sketch(recs, lw, depth, p)
    assert int(cms.sum()) == int(want_cms.sum()), (int(cms.sum()), int(want_cms.sum()))
    assert np.array_equal(cms.reshape(-1), want_cms), "count-min counters differ"
    assert np.array_equal(hll, want_hll), "HyperLogLog registers differ"
    q = np.ascontiguousarray(keys)
    want_q = np.zeros(len(q), dtype=np.uint64)
    O.lib().oracle_cms_query(want_cms.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), lw, depth, SKETCH_SEED,
                             O._p(O.as_bytes(q)), len(q), want_q.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)))
    assert np.array_equal(eng.cms_query(q), want_q)
    assert abs(eng.hll_estimate() - O.lib().oracle_hll_estimate(O._p(want_hll), p)) < 1e-6


def run_accounter(batches, keys, max_entries, max_batch, device=False, sketch=None, emul=None):
    """fa_ingest from host or device memory, every FA_FULL cut evicted; generations (and the sketches) against the
    oracle.  sketch = (log2 width, depth, HLL precision) or None."""
    import netobserv_ebpf_agent_b200 as fa
    kw = {}
    if sketch:
        kw = dict(flags=fa.FA_F_ENABLE_SKETCH, cms_log2_width=sketch[0], cms_depth=sketch[1], hll_precision=sketch[2],
                  sketch_seed=SKETCH_SEED)
    gens = []
    with fa.FlowAggEngine(max_entries, max_batch=max_batch, **kw) as eng:
        for b in batches:
            if device:
                buf = DevBuf(eng, b.size, emul)
                buf.write(b)
                done, n = 0, len(b)
                while done < n:
                    rc, took = eng.ingest(buf.ptr + done * O.REC, n - done)
                    done += took
                    if rc == fa.FA_FULL:
                        gens.append(O.sort_records(eng.evict()))
                eng.sync()
                buf.free()
            else:
                eng.ingest_all(b, lambda r: gens.append(O.sort_records(r)))
        gens.append(O.sort_records(eng.evict()))
        if sketch:
            check_sketch(eng, np.concatenate(batches), keys, *sketch)
        st = eng.stats()
    want = oracle_generations(batches, max_entries)
    assert_same_generations(gens, want)
    assert st["full_cuts"] == len(want) - 1
    return st


def split(recs, parts):
    cuts = np.linspace(0, len(recs), parts + 1).astype(int)
    return [recs[a:b] for a, b in zip(cuts[:-1], cuts[1:])]


def run_nonblocking(recs, max_entries, max_batch, parts=3):
    """FA_F_NONBLOCKING_EVICT in ACCOUNTER mode: each generation is exact on its own."""
    import netobserv_ebpf_agent_b200 as fa
    with fa.FlowAggEngine(max_entries, flags=fa.FA_F_NONBLOCKING_EVICT, max_batch=max_batch) as eng:
        for part in split(recs, parts):
            rc, took = eng.ingest(part)
            assert rc == 0 and took == len(part)
            got = O.sort_records(eng.evict())
            acc = O.Accounter(max_entries); acc.account(part); want = O.sort_records(acc.evict()); acc.close()
            assert_same_generations([got], [want])
        assert eng.live_flows() == 0


def run_drain_refold(recs, max_entries, max_batch, parts, emul=None):
    """fa_drain_active per batch, the partials re-folded by a second engine (the multi-GPU owner's path): the flows
    equal the plain fold of the stream (descriptors are per-key constants here)."""
    import netobserv_ebpf_agent_b200 as fa
    batches = split(recs, parts)
    cap = max(len(b) for b in batches)
    with fa.FlowAggEngine(max_entries, max_batch=max_batch) as local, fa.FlowAggEngine(max_entries) as owner:
        buf = DevBuf(local, cap * O.REC, emul)
        for b in batches:
            local.ingest(b)
            k = local.drain_active(buf.ptr, cap)
            assert 0 < k <= len(np.unique(b[:, :40], axis=0))
            owner.ingest(buf.ptr, k)
        assert local.drain_active(buf.ptr, cap) == 0
        got = O.sort_records(owner.evict())
        buf.free()
    want = oracle_generations(batches, 1 << 22)[0]
    assert_same_generations([got], [want])


def run_features(base, keys, max_entries, max_batch, seed):
    """RTT / DNS / packet-drop folds on the colliding keys, some of them feature-only until a base record arrives."""
    import netobserv_ebpf_agent_b200 as fa
    from test_gpu_features import make_add, make_dns
    rng = np.random.default_rng(seed)
    n_feat = max(len(base) // 2, 500)
    add, dns = make_add(rng, keys, n_feat), make_dns(rng, keys, n_feat)
    drops = np.zeros(n_feat, dtype=O.DROPREC_DTYPE)
    drops["id"] = keys[rng.integers(0, len(keys), n_feat)]
    d = drops["drop"]
    d["start"] = np.where(rng.random(n_feat) < 0.1, 0, UPTIME_NS + rng.integers(0, 1 << 36, n_feat))
    d["end"] = np.where(rng.random(n_feat) < 0.1, 0, UPTIME_NS + rng.integers(0, 1 << 36, n_feat))
    d["bytes"] = rng.integers(0, 1 << 16, n_feat); d["packets"] = rng.integers(0, 1 << 16, n_feat)
    d["cause"] = rng.integers(0, 100, n_feat); d["flags"] = rng.integers(0, 1 << 16, n_feat)
    d["eth"] = rng.choice([0, 0x0800, 0x86DD], n_feat); d["state"] = rng.integers(0, 12, n_feat)
    drops["drop"] = d
    h = len(base) // 2
    om = O.FlowMap()
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP
    with fa.FlowAggEngine(max_entries, flags=flags, max_batch=max_batch) as eng:
        eng.ingest_additional(add); eng.ingest_pkt_drops(drops[: n_feat // 2])   # feature-only flows first
        eng.ingest(base[:h]); eng.ingest_dns(dns); eng.ingest(base[h:]); eng.ingest_pkt_drops(drops[n_feat // 2:])
        om.fold_additional(add); om.fold_drops(drops[: n_feat // 2]); om.account(base[:h]); om.fold_dns(dns)
        om.account(base[h:]); om.fold_drops(drops[n_feat // 2:])
        got = eng.evict_ex()
    want = om.evict_ex()
    gp, op = O.sort_perm(got[0]), O.sort_perm(want[0])
    assert len(gp) == len(op)
    for name, g, w in zip(("records", "dns", "additional", "pkt_drops", "rtt_min", "present"), got, want):
        g, w = np.asarray(g)[gp], np.asarray(w)[op]
        assert np.array_equal(g, w), name


def run_kernel_map(seed, n, max_entries, max_batch, ringbuf, evict_every=None):
    """KERNEL_MAP on single-packet events of colliding keys, in a map small enough to fill."""
    from test_gpu_kernel_map import check
    from test_kmap_emulation import messy_stream
    rng = np.random.default_rng(seed)
    fam = key_families(seed, table_slots(max_entries), n_chain=200)
    keys = np.concatenate([fam["full"], fam["chain_last"], fam["elect"]])
    r = messy_stream(seed, n, max(n // 8, 64), tls=False)
    idx = np.nonzero(rng.random(n) < 0.6)[0]
    r[idx, :40] = keys[rng.integers(0, len(keys), len(idx))]
    v = r.view(O.REC_DTYPE).reshape(-1)
    v["start"] = UPTIME_NS + rng.integers(0, 1 << 40, n).astype(np.uint64)
    v["end"] = v["start"]
    check(r, max_entries, max_batch, ringbuf=ringbuf, evict_every=evict_every)


def run_events(recs, max_entries, max_batch):
    """fa_ingest_events with uptime mono_ts and colliding keys (padding byte 39 set on a third of them: it is not part
    of the key), every FA_FULL cut evicted; generations against the oracle's fold of the expanded records."""
    import netobserv_ebpf_agent_b200 as fa
    from test_events import events_of, expand
    ev = events_of(recs)
    ev["id"][::3, 39] = 0x5A
    raw = ev.view(np.uint8).reshape(-1)
    gens = []
    with fa.FlowAggEngine(max_entries, max_batch=max_batch) as eng:
        done = 0
        while done < len(ev):
            rc, took = eng.ingest_events(raw[done * 64:])
            done += took
            if rc == fa.FA_FULL:
                gens.append(O.sort_records(eng.evict()))
        gens.append(O.sort_records(eng.evict()))
    assert_same_generations(gens, oracle_generations([expand(ev)], max_entries))
    return len(gens)


def run_route(recs, keys, n_shards, emul=None):
    """fa_route: every record goes to owner_hash(key) % n_shards, the order kept inside a shard; keys with one
    premix all go to one owner."""
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200.sharded import owner_of, route_host
    assert len(set(owner_of(keys[:64], n_shards).tolist())) == 1          # the "full" family: one premix
    want, want_counts = route_host(recs, n_shards)
    with fa.FlowAggEngine(1000, max_batch=max(len(recs), 1024)) as eng:
        src, dst = DevBuf(eng, recs.size, emul), DevBuf(eng, recs.size, emul)
        src.write(recs)
        counts = eng.route(src.ptr, len(recs), n_shards, dst.ptr)
        eng.sync()
        got = dst.read(recs.size).reshape(-1, O.REC)
        src.free(); dst.free()
    assert np.array_equal(counts.astype(np.int64), want_counts)
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------- CPU: the keys
@pytest.mark.parametrize("slots", [1024, 1 << 17])
def test_key_families_hash_as_built(slots):
    fam = key_families(3, slots, n_chain=40)
    f = O.lib()
    for name, keys in fam.items():
        assert len(np.unique(keys, axis=0)) == len(keys), name
        assert not keys[:, 39].any()
        assert np.array_equal(keys[:, :10], np.zeros((len(keys), 10), np.uint8)) and (keys[:, 10:12] == 0xFF).all()
        pm = [f.oracle_key_premix(O._p(np.ascontiguousarray(k))) for k in keys]
        sh = [f.oracle_slot_hash(O._p(np.ascontiguousarray(k))) for k in keys]
        assert pm == [premix(k) for k in keys] and sh == [fmix64(x) for x in pm], name
        if name == "full":
            assert len(set(pm)) == 1
        else:
            assert len(set(pm)) == len(keys), name
        if name == "chain_last":
            assert {x & (slots - 1) for x in sh} == {slots - 1}
        if name == "chain_mid":
            assert len({x & (slots - 1) for x in sh}) == 1
        if name == "way":
            assert len({x & 0xFFFFFFFF for x in sh}) == 1 and len({x >> 32 for x in sh}) == len(keys)
        if name == "elect":
            assert len({x & ELECTION_BITS for x in sh}) == 1 and len({x & 0xFFFF for x in sh}) > len(keys) // 2


def test_stream_transforms_reach_the_far_side():
    """The stream really has what the generator lacks: end and 0 - start change high word inside most tiles, the
    clock runs backwards, zero timestamps, packet sums that carry, colliding keys."""
    recs, keys = adversarial_stream(5, 4_096, 1024, pre_agg=True)
    v = recs.view(O.REC_DTYPE).reshape(-1)
    tiles = np.arange(len(v)) // 256
    end_hi = v["end"] >> np.uint64(32)
    ns_hi = (np.uint64(0) - v["start"]) >> np.uint64(32)
    nz_e, nz_s = v["end"] != 0, v["start"] != 0
    split_e = [len(np.unique(end_hi[(tiles == t) & nz_e])) > 1 for t in range(tiles.max() + 1)]
    split_s = [len(np.unique(ns_hi[(tiles == t) & nz_s])) > 1 for t in range(tiles.max() + 1)]
    assert np.mean(split_e) > 0.8 and np.mean(split_s) > 0.8
    assert (np.diff(v["start"][nz_s].astype(np.int64)) < 0).sum() > 50
    assert 0.05 < (~nz_s).mean() < 0.15 and 0.05 < (~nz_e).mean() < 0.15
    assert (v["start"][nz_s] > np.uint64(1 << 50)).all()
    acc = O.Accounter(1 << 12); acc.account(recs)
    flows = acc.evict().view(O.REC_DTYPE).reshape(-1); acc.close()
    k = np.ascontiguousarray(recs[:, :40]).view(np.dtype((np.void, 40))).reshape(-1)
    _, inv = np.unique(k, return_inverse=True)
    wide = np.bincount(inv.reshape(-1), weights=v["packets"].astype(np.float64))
    assert (wide >= 2.0 ** 32).sum() > 10                       # flows whose packet sum wraps in the table
    assert len(flows) == len(wide)
    kk = np.ascontiguousarray(keys).view(np.dtype((np.void, 40))).reshape(-1)
    assert np.isin(k, kk).mean() > 0.3


def test_k1_walks_the_chains_and_stays_exact():
    """On the K1 emulation: the chains are really walked (most representatives of a chain-only stream need the
    general loop), with the other families and uptime timestamps in the same tiles."""
    from test_k1_emulation import K1, same_flows
    rng = np.random.default_rng(17)
    fam = key_families(17, table_slots(700), n_chain=300)
    chain = np.concatenate([fam["chain_last"], fam["chain_mid"]])
    recs = uptime_times(mix_keys(gen_host(seed=17, n=2_400, n_keys=50, dist=1), chain, rng, frac=1.0), rng)
    k1 = K1(700, max_batch=4_096, grid=2)
    K1.paths()
    k1.ingest(recs[:1_200])
    K1.paths()
    k1.ingest(recs[1_200:])
    reps, slow, _ = K1.paths()
    assert slow > reps // 2, (reps, slow)
    acc = O.Accounter(1 << 12); acc.account(recs)
    same_flows(k1.evict(), acc.evict())
    others, _ = adversarial_stream(18, 2_000, table_slots(700), varying=1, pre_agg=True, n_chain=100)
    k1 = K1(700, max_batch=4_096, grid=3)
    k1.ingest(others)
    acc = O.Accounter(1 << 12); acc.account(others)
    same_flows(k1.evict(), acc.evict())


# ---------------------------------------------------------------------------------------------------- CPU: engine emulation
EMUL_N = 2_500


@pytest.mark.parametrize("device,sketch,varying", [(False, False, 1), (False, True, 0), (True, False, 0), (True, True, 1)])
def test_accounter_emul(engine_emul, device, sketch, varying):
    recs, keys = adversarial_stream(100 + varying, EMUL_N, table_slots(1 << 10), varying=varying)
    run_accounter(split(recs, 2), keys, 1 << 10, 1_024, device=device, sketch=(10, 2, 8) if sketch else None,
                  emul=engine_emul)


@pytest.mark.parametrize("device", [False, True])
def test_pre_aggregated_sketch_emul(engine_emul, device):
    """Packet sums of one flow in one tile, or in one hot-cache entry, pass 2^32: the count-min counters stay the
    64-bit sums (the flow table's packets wrap mod 2^32 by design)."""
    recs, keys = adversarial_stream(110, EMUL_N, table_slots(1 << 10), pre_agg=True)
    run_accounter([recs], keys, 1 << 10, 2_048, device=device, sketch=(10, 2, 8), emul=engine_emul)


@pytest.mark.parametrize("max_entries,n", [(16, 600), (100, 1_500), (1000, 3_000)])
def test_full_cut_emul(engine_emul, max_entries, n):
    recs, keys = adversarial_stream(120 + max_entries, n, table_slots(max_entries), pre_agg=max_entries == 100,
                                    n_chain=120, bg_keys=1_500, dist=0)
    st = run_accounter(split(recs, 2), keys, max_entries, 1_024, emul=engine_emul)
    assert st["full_cuts"] > 0


def test_nonblocking_evict_emul(engine_emul):
    recs, _ = adversarial_stream(130, EMUL_N, table_slots(1 << 11), pre_agg=True)
    run_nonblocking(recs, 1 << 11, 1_024)


def test_drain_refold_emul(engine_emul):
    recs, _ = adversarial_stream(140, EMUL_N, table_slots(1 << 11), pre_agg=True)
    run_drain_refold(recs, 1 << 11, 1_024, 3, emul=engine_emul)


def test_feature_folds_emul(engine_emul):
    recs, keys = adversarial_stream(150, 2_000, table_slots(1 << 11), varying=1, n_chain=100)
    run_features(recs, keys, 1 << 11, 1_024, 150)


@pytest.mark.parametrize("max_entries", [1 << 10, 300])
def test_events_emul(engine_emul, max_entries):
    recs, _ = adversarial_stream(155, 2_000, table_slots(max_entries), n_chain=120, bg_keys=600, dist=0)
    assert run_events(recs, max_entries, 1_024) > (max_entries < 1_000)


@pytest.mark.parametrize("impl", ["2", "1"])
@pytest.mark.parametrize("ringbuf", [True, False])
def test_kernel_map_emul(engine_emul, monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    run_kernel_map(160, 2_000, 150, 1_024, ringbuf)


def test_route_emul(engine_emul):
    recs, keys = adversarial_stream(170, 3_000, 1024)
    run_route(recs, keys, 3, emul=engine_emul)


@pytest.mark.parametrize("shape", [(4, 1, 4), (4, 8, 18), (22, 8, 4), (20, 1, 18)])
def test_sketch_shapes_emul(engine_emul, shape):
    recs, keys = adversarial_stream(180, 2_000, table_slots(1 << 10), pre_agg=True, n_chain=60)
    run_accounter([recs], keys, 1 << 10, 2_048, sketch=shape, emul=engine_emul)


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("device,sketch", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("varying,max_batch", [(0, 1 << 16), (1, 100_000), (0, 1 << 20)])
def test_accounter_gpu(device, sketch, varying, max_batch):
    recs, keys = adversarial_stream(200 + varying, 600_000, table_slots(1 << 18), varying=varying)
    run_accounter(split(recs, 2), keys, 1 << 18, max_batch, device=device, sketch=(16, 4, 14) if sketch else None)


@pytest.mark.gpu
@pytest.mark.parametrize("device,max_batch", [(False, 1 << 16), (True, 1 << 20)])
def test_pre_aggregated_sketch_gpu(device, max_batch):
    recs, keys = adversarial_stream(210, 500_000, table_slots(1 << 18), pre_agg=True)
    run_accounter([recs], keys, 1 << 18, max_batch, device=device, sketch=(12, 4, 10))


@pytest.mark.gpu
@pytest.mark.parametrize("max_entries,max_batch", [(16, 1 << 16), (100, 7_000), (1000, 50_000)])
def test_full_cut_gpu(max_entries, max_batch):
    recs, keys = adversarial_stream(220 + max_entries, 100_000, table_slots(max_entries), pre_agg=max_entries == 100,
                                    bg_keys=20_000, dist=0)
    st = run_accounter(split(recs, 2), keys, max_entries, max_batch)
    assert st["full_cuts"] > 0


@pytest.mark.gpu
def test_nonblocking_evict_gpu():
    recs, _ = adversarial_stream(230, 600_000, table_slots(1 << 18), pre_agg=True)
    run_nonblocking(recs, 1 << 18, 1 << 16)


@pytest.mark.gpu
def test_drain_refold_gpu():
    recs, _ = adversarial_stream(240, 400_000, table_slots(1 << 17), pre_agg=True)
    run_drain_refold(recs, 1 << 17, 60_000, 4)


@pytest.mark.gpu
def test_feature_folds_gpu():
    recs, keys = adversarial_stream(250, 200_000, table_slots(1 << 16), varying=1)
    run_features(recs, keys, 1 << 16, 25_000, 250)


@pytest.mark.gpu
@pytest.mark.parametrize("max_entries,max_batch", [(1 << 17, 1 << 16), (5_000, 100_000)])
def test_events_gpu(max_entries, max_batch):
    recs, _ = adversarial_stream(255, 300_000, table_slots(max_entries), bg_keys=60_000, dist=0)
    assert run_events(recs, max_entries, max_batch) > (max_entries < 10_000)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["2", "1"])
@pytest.mark.parametrize("ringbuf", [True, False])
def test_kernel_map_gpu(monkeypatch, impl, ringbuf):
    monkeypatch.setenv("FA_KMAP_IMPL", impl)
    run_kernel_map(260, 200_000, 2_000, 1 << 16, ringbuf, evict_every=100_000)


@pytest.mark.gpu
def test_route_gpu():
    recs, keys = adversarial_stream(270, 100_000, 1 << 17)
    run_route(recs, keys, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4, 1, 4), (4, 8, 18), (22, 8, 4), (20, 1, 18)])
def test_sketch_shapes_gpu(shape):
    recs, keys = adversarial_stream(280, 300_000, table_slots(1 << 17), pre_agg=True)
    run_accounter([recs], keys, 1 << 17, 1 << 16, sketch=shape)
