"""K1 at its launch boundaries: the dynamic tile schedule (each team's first tile is fixed, every later one is claimed
from a per-launch counter that the last CTA out zeroes) must fold every record exactly once, whatever the number of
tiles, CTAs and launches, and whether the record count is known on the host or only on the device.

Each case runs on the CPU emulation (tests/emul/) and, marked `gpu`, through the C ABI on the device; the evicted flows
are compared bit for bit with the oracle, and the byte and packet totals with the input's."""
import ctypes

import numpy as np
import pytest

import oracle_lib as O
from common import assert_same_generations, gen_host, gpu_generations, oracle_generations
from test_k1_emulation import K1, same_flows

pytestmark = pytest.mark.timeout(900)

TILE, TEAMS = 256, 4                 # aggregate.cu: kTile records per tile, kTeams tile pipelines per CTA


def totals(recs):
    r = np.ascontiguousarray(recs).view(O.REC_DTYPE).reshape(-1)
    return int(r["bytes"].astype(np.uint64).sum()), int(r["packets"].astype(np.uint64).sum())


def check_flows(got, recs, max_entries):
    acc = O.Accounter(max_entries)
    acc.account(recs)
    same_flows(got, acc.evict())
    assert totals(got) == totals(recs)


def ragged_sizes(grid):
    """Below one tile, one tile exactly, and one record either side of k rounds of the static first tiles."""
    first_round = TILE * TEAMS * grid
    return [100, TILE, first_round - 1, first_round + 1, 3 * first_round - 1, 3 * first_round + 1]


@pytest.mark.parametrize("grid", [1, 2, 3])
def test_ragged_tile_counts_emulated(grid):
    """Launches of every ragged size, one after the other on one table: a claim counter that is not back at zero
    would skip the next launch's tiles."""
    sizes = ragged_sizes(grid)
    recs = gen_host(seed=101 + grid, n=sum(sizes), n_keys=700, dist=1, varying=1)
    k1 = K1(1 << 12, max_batch=max(sizes), grid=grid)
    lo = 0
    for n in sizes:
        k1.ingest(recs[lo:lo + n])
        lo += n
    check_flows(k1.evict(), recs, 1 << 12)
    for n in sizes:                                      # each size on a fresh table as well
        k1 = K1(1 << 12, max_batch=max(sizes), grid=grid)
        k1.ingest(recs[:n])
        check_flows(k1.evict(), recs[:n], 1 << 12)


def test_grid_changes_between_launches_emulated():
    """The counter's base depends on the grid, which changes with the launch size."""
    recs = gen_host(seed=111, n=30_000, n_keys=2_000, dist=1)
    k1 = K1(1 << 13, max_batch=1 << 14, grid=3)
    lo = 0
    for n, grid in ((9_000, 3), (300, 3), (7_000, 1), (13_700, 2)):
        k1.grid = grid
        k1.ingest(recs[lo:lo + n])
        lo += n
    check_flows(k1.evict(), recs, 1 << 13)


# ------------------------------------------------------------------------------------------- through the C ABI
def accounter_full_cuts():
    """ACCOUNTER with a small max_entries: launches end at the FA_FULL cut, the next one starts at the cut."""
    recs = gen_host(seed=121, n=12_000, n_keys=3_000, dist=1, varying=1)
    for max_entries, max_batch in ((300, 1_024), (1_000, 4_097)):
        got, st = gpu_generations([recs[:5_000], recs[5_000:]], max_entries, max_batch=max_batch)
        want = oracle_generations([recs[:5_000], recs[5_000:]], max_entries)
        assert_same_generations(got, want)
        assert len(got) > 2 and st["records_ingested"] == len(recs)


def test_accounter_full_cuts_emulated(engine_emul):
    accounter_full_cuts()


@pytest.mark.gpu
def test_gpu_accounter_full_cuts():
    accounter_full_cuts()


def counted_launches(alloc):
    """fa_ingest_counted: the record count is on the device, so the grid is sized for max_n and most teams find no
    first tile.  `alloc(array)` returns (address, keep-alive) of a copy the engine can read."""
    import netobserv_ebpf_agent_b200 as fa
    L = fa.lib()
    recs = gen_host(seed=131, n=20_000, n_keys=1_500, dist=1, varying=1)
    max_n = 8_192
    counts = [1, 255, 257, 2_047, 4_097, 8_192, 5_000 - 1]
    with fa.FlowAggEngine(1 << 13, max_batch=max_n, flags=fa.FA_F_NO_FULL_CUT) as eng:
        lo = 0
        for c in counts:
            buf = np.zeros(max_n * O.REC, dtype=np.uint8)
            buf[:c * O.REC] = np.ascontiguousarray(recs[lo:lo + c]).view(np.uint8).reshape(-1)
            p, keep = alloc(buf)
            pn, keep_n = alloc(np.array([c], dtype=np.uint64))
            assert L.fa_ingest_counted(eng._h, ctypes.c_void_p(p), ctypes.c_void_p(pn), max_n, 0) == 0
            eng.sync()
            lo += c
            del keep, keep_n
        assert eng.live_flows() == len(O.sort_records(oracle_generations([recs[:lo]], 1 << 13)[0]))
        check_flows(O.sort_records(eng.evict()), recs[:lo], 1 << 13)


def test_device_counted_launches_emulated(engine_emul):
    def host(a):                                         # the emulated device reads host memory
        a = np.ascontiguousarray(a)
        return a.ctypes.data, a
    counted_launches(host)


@pytest.mark.gpu
def test_gpu_device_counted_launches():
    import torch

    def dev(a):
        t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()
        return t.data_ptr(), t
    counted_launches(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("max_batch", [100, 1 << 12, (1 << 15) + 1, 132 * TEAMS * TILE + 1])
def test_gpu_ragged_launch_sizes(max_batch):
    """On the device: every SM's teams claim tiles; launch sizes below one tile, just past the static first tiles of
    132 SMs, and a chunk schedule whose last launch is ragged."""
    recs = gen_host(seed=141, n=300_000, n_keys=40_000, dist=1, varying=1)
    got, st = gpu_generations([recs], 1 << 17, max_batch=max_batch)
    assert_same_generations(got, oracle_generations([recs], 1 << 17))
    assert totals(got[0]) == totals(recs)
