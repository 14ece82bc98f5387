"""K1's hot-flow cache (csrc/aggregate.cu): 12 sets of 8 ways, found through a set's 16-bit tags.

The cache only ever saves table probes, so a broken lookup would still come out exact; these tests therefore check
two things: that flows which share a set (and flows which share a set *and* a tag) are served on-chip, by the
emulation's cache-hit counter, and that everything the cache folds comes out bit for bit as the oracle has it:
timestamps outside an entry's 32-bit window, counters that wrap, descriptors that change on a cached flow (the
ordered re-fold), more hot flows in a set than it has ways, and the fused sketches."""
import ctypes

import numpy as np
import pytest

import oracle_lib as O
from common import assert_same_generations, gen_host, gpu_generations, oracle_generations
from test_k1_emulation import K1, emul, fa_slot, same_flows

pytestmark = pytest.mark.timeout(900)

SETS, WAYS = 12, 8


def cache_set(h):
    return (((h >> 16) & 0xFFFF) * SETS) >> 16


def cache_tag(h):
    return (h & 0xFFFF) | 1


_pool = None


def key_pool():
    """-> (keys (n,40), 32-bit slot hashes) of 60,000 distinct generated keys."""
    global _pool
    if _pool is None:
        keys = np.unique(gen_host(seed=41, n=60_000, n_keys=60_000, dist=0)[:, :40], axis=0)
        _pool = keys, np.array([fa_slot(k) & 0xFFFFFFFF for k in keys], dtype=np.int64)
    return _pool


def keys_sharing_bits_21_to_31(count):
    """Keys whose hashes agree in bits 21..31: one cache set, and one index under any direct-mapped use of those bits."""
    keys, h = key_pool()
    top = h >> 21
    for v in np.argsort(-np.bincount(top)):
        pick = np.nonzero(top == v)[0]
        if len(pick) >= count and len({cache_set(int(x)) for x in h[pick]}) == 1:
            return keys[pick[:count]]
    raise AssertionError("no such family in the pool")


def keys_of_one_set_with_a_shared_tag(count):
    """`count` keys of one cache set, the first two with the same 16-bit tag."""
    keys, h = key_pool()
    sets = np.array([cache_set(int(x)) for x in h])
    tags = np.array([cache_tag(int(x)) for x in h])
    seen = {}
    for i in range(len(keys)):
        j = seen.setdefault((sets[i], tags[i]), i)
        if j != i:
            rest = [k for k in np.nonzero(sets == sets[i])[0] if k not in (i, j)][: count - 2]
            return keys[[j, i] + rest]
    raise AssertionError("no tag collision in the pool")


def stream(keys, n, seed, weights=None, varying=0, pick=None):
    """n generated records whose keys are drawn from `keys`.  Timestamps, lengths and TCP flags stay as generated; the
    per-flow constants (eth_protocol and the descriptor) follow the new key unless `varying` asks for changing ones."""
    rng = np.random.default_rng(seed)
    recs = gen_host(seed=seed, n=n, n_keys=len(keys), dist=0, varying=varying).copy()
    if pick is None:
        pick = rng.choice(len(keys), n, p=weights)
    if not varying:
        _, first, inv = np.unique(recs[:, :40], axis=0, return_index=True, return_inverse=True)
        template = recs[first[inv.reshape(-1)[rng.integers(0, n, len(keys))]]]      # one generated flow per new key
        recs[:, 68:70] = template[pick, 68:70]
        recs[:, 72:] = template[pick, 72:]
    recs[:, :40] = keys[pick]
    return recs


def run_emulated(recs, launches=1, sketch=None, grid=1):
    k1 = K1(1 << 12, max_batch=1 << 15, grid=grid)
    if sketch:
        emul().k1_emul_enable_sketch(k1.h, *sketch)
    K1.paths()
    for part in np.array_split(recs, launches):
        k1.ingest(part)
    paths = K1.paths()
    acc = O.Accounter(1 << 12)
    acc.account(recs)
    fixups = k1.counter(2)
    if sketch:
        lw, depth, p, seed = sketch
        cms, hll = np.zeros(depth << lw, dtype=np.uint64), np.zeros(1 << p, dtype=np.uint8)
        emul().k1_emul_sketch_export(k1.h, cms.ctypes.data, hll.ctypes.data)
        b = O.as_bytes(recs)
        want_cms, want_hll = np.zeros_like(cms), np.zeros_like(hll)
        O.lib().oracle_cms_update(want_cms.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), lw, depth, seed, O._p(b), len(recs))
        O.lib().oracle_hll_update(O._p(want_hll), p, seed, O._p(b), len(recs))
        assert np.array_equal(cms, want_cms) and np.array_equal(hll, want_hll)
    same_flows(k1.evict(), acc.evict())
    return paths, fixups


def test_eight_hot_flows_of_one_set_are_all_served_on_chip():
    """Eight equally hot flows whose hashes agree in bits 21..31 take the eight ways of their set: after the first tiles
    nearly every record is a cache hit.  (Entries indexed directly by those bits could hold two of the eight.)"""
    recs = stream(keys_sharing_bits_21_to_31(WAYS), 8_192, seed=42)
    (reps, slow, cached), fixups = run_emulated(recs)
    assert cached > 0.8 * len(recs), (reps, slow, cached)
    assert fixups == 0


def test_two_flows_with_one_tag_in_one_set():
    """The tag is 16 bits of the hash: two hot flows of one set with the same tag must both be found (the lookup walks
    every way that carries the tag) next to five set-mates; seven flows, so each of them gets a way."""
    keys = keys_of_one_set_with_a_shared_tag(WAYS - 1)
    recs = stream(keys, 8_192, seed=43, weights=np.array([0.3, 0.3] + [0.08] * 5))
    (reps, slow, cached), _ = run_emulated(recs)
    assert cached > 0.8 * len(recs), (reps, slow, cached)     # with one of the twins left out: at most 0.7


def messy(recs, seed):
    """Timestamps in another 32-bit window or zero, packet and byte counters about to wrap."""
    rng = np.random.default_rng(seed)
    r = recs.view(O.REC_DTYPE).reshape(-1)
    r["start"][rng.random(len(r)) < 0.1] = 0
    r["end"][rng.random(len(r)) < 0.1] = 0
    r["start"][rng.random(len(r)) < 0.2] += np.uint64(1) << np.uint64(33)
    r["end"][rng.random(len(r)) < 0.2] += np.uint64(1) << np.uint64(34)
    r["packets"][rng.random(len(r)) < 0.1] = 0xFFFFFFF0
    r["bytes"][rng.random(len(r)) < 0.1] = 0xFFFFFFFFFFFFFF00
    return recs


def crowded_set_stream(n, seed, varying):
    """More hot flows in one set than it has ways (twelve, two of them tag twins), the hot subset moving every 1,024
    records, over a background of 300 other flows; `varying`: 2 % of the records differ in a descriptor field."""
    hot = keys_of_one_set_with_a_shared_tag(SETS)
    rng = np.random.default_rng(seed)
    pick = len(hot) + rng.integers(0, 300, n)
    for lo in range(0, n, 1_024):
        now = rng.choice(len(hot), 5, replace=False)
        idx = lo + np.nonzero(rng.random(min(1_024, n - lo)) < 0.7)[0]
        pick[idx] = now[rng.integers(0, len(now), len(idx))]
    recs = stream(np.concatenate([hot, key_pool()[0][-300:]]), n, seed=seed, pick=pick)
    if varying:                                  # now and then a record of a (cached) flow carries another descriptor
        r = recs.view(O.REC_DTYPE).reshape(-1)
        r["if_index"][rng.random(n) < 0.02] ^= 1
    return messy(recs, seed)


@pytest.mark.parametrize("varying", [0, 1])
def test_crowded_set_stays_exact(varying):
    """The flows that find no free way keep probing the table while their set-mates fold on-chip; a record
    whose descriptor differs from the cached one is not folded on-chip and flags the flow for the ordered re-fold."""
    recs = crowded_set_stream(16_384, seed=44 + varying, varying=varying)
    (reps, slow, cached), fixups = run_emulated(recs, launches=2)
    assert cached > len(recs) // 20, (reps, slow, cached)
    assert (fixups > 0) == bool(varying)


def test_crowded_set_with_fused_sketches():
    """The cache's 64-bit packet total (carries counted apart) reaches the count-min sketch at the flush."""
    recs = crowded_set_stream(12_288, seed=46, varying=0)
    (reps, slow, cached), _ = run_emulated(recs, sketch=(10, 4, 8, 0xC0FFEE))
    assert cached > len(recs) // 20, (reps, slow, cached)


@pytest.mark.gpu
@pytest.mark.parametrize("varying", [0, 1])
def test_gpu_crowded_set_stays_exact(varying):
    """The same streams through the C ABI on the device, tiled over every SM and over a few CTAs only."""
    recs = np.concatenate([crowded_set_stream(1 << 17, seed=47 + varying, varying=varying),
                           stream(keys_sharing_bits_21_to_31(WAYS), 1 << 16, seed=49)])
    for max_batch in (1 << 12, 1 << 18):
        got, _ = gpu_generations([recs], 1 << 12, max_batch=max_batch)
        assert_same_generations(got, oracle_generations([recs], 1 << 12))
