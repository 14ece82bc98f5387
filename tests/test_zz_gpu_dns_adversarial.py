"""K7 on the device with colliding dns_flow_ids, uptime-scale clocks and purge edges: the scenarios of
tests/test_dns_adversarial.py at 10^5 to 10^6 packets through libflowagg.so, bit for bit against the restatement.

Every walk of the table is bounded by its size; the scenarios make the walks long, never endless.  The file sorts last
and carries a thread-method timeout so that a wedged kernel here could not hold or poison the rest of the GPU suite."""
import numpy as np
import pytest

from test_dns_adversarial import (PROBE_HOME, device_ingest, dns_packets, dns_slots, latencies, one_sample_share, random_keys,
                                  run_case, scenario_hot, scenario_mixed, scenario_probe_rebuild, scenario_probe_run,
                                  scenario_purge, scenario_rebuilds, scenario_uptime, spread_transactions)
from test_dns_correlate import dns_stream

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(240, method="thread")]

DEFAULT = 1 << 20                           # dns_flows max_entries without FA_DNS_MAX_ENTRIES


def flows_for(steps):
    return max(sum(len(b) for b in steps if not isinstance(b, tuple)), 1 << 12)


@pytest.mark.parametrize("max_batch", [1 << 16, 100_000])
def test_colliding_transactions_gpu(max_batch):
    steps = scenario_mixed(110, dns_slots(DEFAULT), 20_000, 5, extra=spread_transactions(111, 200_000),
                           n_chain=600, n_mid=300, n_tuple=64)
    assert sum(map(len, steps)) > 300_000
    st = run_case(steps, flows=flows_for(steps), max_batch=max_batch)
    assert st["dns_map_full"] == 0
    assert one_sample_share(steps, DEFAULT) >= 0.8


def test_colliding_transactions_from_device_memory_gpu():
    steps = scenario_mixed(112, dns_slots(DEFAULT), 10_000, 3, extra=spread_transactions(113, 80_000), n_chain=300)
    run_case(steps, flows=flows_for(steps), max_batch=1 << 15, ingest=device_ingest(None))


@pytest.mark.parametrize("max_entries", [1024, 1 << 14])
def test_chains_across_rebuilds_gpu(monkeypatch, max_entries):
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", str(max_entries))
    steps, n_q = scenario_rebuilds(120 + max_entries, max_entries, rounds=6, n_chain=1_000, n_mid=500, n_tuple=64)
    st = run_case(steps, max_entries=max_entries, flows=flows_for(steps), max_batch=1 << 16)
    assert st["dns_map_full"] == 0
    lat = latencies(steps, max_entries)[-len(steps[-1]):]
    assert (lat["errno"] == 0).sum() == n_q
    assert one_sample_share(steps, max_entries) >= 0.8


def test_hot_colliding_keys_gpu():
    """More packets per colliding key and call than round kernels: the tail finishes them on the device."""
    steps = scenario_hot(130, dns_slots(DEFAULT), per_key=(20, 60), parts=4, n_bg=20_000)
    run_case(steps, flows=flows_for(steps), max_batch=1 << 16)


def test_probe_run_longer_than_4096_gpu(monkeypatch):
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", "4096")
    assert dns_slots(4096) - 1 == PROBE_HOME
    steps = scenario_probe_run(bg=dns_stream(140, 3_000, n_clients=20, n_ids=3))
    st = run_case(steps, max_entries=4096, flows=flows_for(steps))
    assert st["dns_map_full"] == 0
    assert (latencies(steps, 4096)[-8:]["errno"] == 0).all()


def test_probe_run_at_the_default_max_entries_gpu():
    """4,200 pending queries of one home slot in the default 2^22-slot table, around 190,000 other packets."""
    steps = scenario_probe_rebuild(4_200, spread_transactions(150, 120_000))
    st = run_case(steps, flows=flows_for(steps), max_batch=1 << 16)
    assert st["dns_map_full"] == 0
    assert (latencies(steps, DEFAULT)[-4_200:]["errno"] == 0).all()


def test_rebuild_replaces_a_run_longer_than_4096_gpu(monkeypatch):
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", "8192")
    filler = dns_packets(random_keys(np.random.default_rng(151), 12_500), True)     # orphan responses: nothing pending
    assert len(filler) + 4_200 > dns_slots(8192) // 2
    steps = scenario_probe_rebuild(4_200, filler)
    st = run_case(steps, max_entries=8192, flows=flows_for(steps))
    assert st["dns_map_full"] == 0
    assert (latencies(steps, 8192)[-4_200:]["errno"] == 0).all()


@pytest.mark.parametrize("max_entries", [1 << 14, None])
def test_uptime_clocks_gpu(monkeypatch, max_entries):
    if max_entries:
        monkeypatch.setenv("FA_DNS_MAX_ENTRIES", str(max_entries))
    me = max_entries or DEFAULT
    extra = spread_transactions(161, 25_000 if max_entries else 300_000)     # pending queries stay below max_entries
    steps = scenario_uptime(160, dns_slots(me), 10_000, 4, extra=extra, n_chain=600, n_mid=300)
    st = run_case(steps, max_entries=me, flows=flows_for(steps), max_batch=1 << 16)
    assert st["dns_map_full"] == 0
    assert one_sample_share(steps, me) >= 0.8


@pytest.mark.parametrize("device", [False, True])
def test_purge_edges_gpu(monkeypatch, device):
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", "1024")
    steps = scenario_purge(170, dns_slots(1024))
    run_case(steps, max_entries=1024, ingest=device_ingest(None) if device else None)
    assert one_sample_share(steps, 1024) >= 0.8
