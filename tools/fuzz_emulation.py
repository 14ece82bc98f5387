#!/usr/bin/env python
"""Randomised parity runs of the kernels under the host emulation (no GPU): the K1 emulation against the oracle's Accounter
(`k1`), the emulated C ABI with full cuts / chunking / re-fold (`engine`), and the feature folds + K7 through it (`features`).
Test infrastructure, like tests/emul/: usage `python tools/fuzz_emulation.py k1|engine|features SEED SECONDS`.
Round 2, shipped kernels: k1 366 iterations, engine 204, features 569 — no mismatch.  With the 12 x 8 hot-flow cache:
k1 50 iterations (seed 5, 150 s) — no mismatch."""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import oracle_lib as O  # noqa: E402
from common import gen_host  # noqa: E402


def fuzz_k1(rng, seconds):
    import test_k1_emulation as T
    t0, it = time.time(), 0
    while time.time() - t0 < seconds:
        it += 1
        n_keys = int(rng.choice([1, 3, 40, 300, 2000, 6000])); n = int(rng.integers(1, 20_000))
        dist = int(rng.integers(0, 2)); varying = int(rng.random() < 0.4)
        cap_log = int(rng.integers(max(3, int(np.ceil(np.log2(max(n_keys, 2) * 1.4)))), 15))
        max_batch = int(rng.choice([257, 1000, 4096, 16384])); grid = int(rng.integers(1, 4)); seed = int(rng.integers(1, 1 << 30))
        recs = gen_host(seed=seed, n=n, n_keys=n_keys, dist=dist, varying=varying)
        if rng.random() < 0.3:        # zero timestamps, timestamps in another 32-bit window, counters about to wrap
            r = recs.view(O.REC_DTYPE).reshape(-1)
            r["start"][rng.random(len(r)) < 0.2] = 0
            r["end"][rng.random(len(r)) < 0.1] = 0
            r["start"][rng.random(len(r)) < 0.2] += np.uint64(1) << np.uint64(33)
            r["packets"][rng.random(len(r)) < 0.05] = 0xFFFFFFF0
            r["bytes"][rng.random(len(r)) < 0.05] = 0xFFFFFFFFFFFFFF00
        params = dict(n_keys=n_keys, n=n, dist=dist, varying=varying, cap_log=cap_log, max_batch=max_batch, grid=grid, seed=seed)
        k1 = T.K1(1 << cap_log, max_batch=max_batch, var=0, grid=grid)
        acc = O.Accounter(1 << cap_log)
        cut = int(rng.integers(0, n + 1))
        try:
            k1.ingest(recs[:cut]); acc.account(recs[:cut])
            if rng.random() < 0.3:
                T.same_flows(k1.evict(), acc.evict())
            k1.ingest(recs[cut:]); acc.account(recs[cut:])
            T.same_flows(k1.evict(), acc.evict())
        except AssertionError as e:
            print("FAIL", params, cut, str(e)[:300]); sys.exit(1)
        k1.close()
    print("ok iterations", it)


def load_engine_emulation():
    import conftest
    L, lib = conftest._load_engine_emulation()
    L._lib = lib


def fuzz_engine(rng, seconds):
    load_engine_emulation()
    from common import assert_same_generations, gpu_generations, oracle_generations
    t0, it = time.time(), 0
    while time.time() - t0 < seconds:
        it += 1
        n_keys = int(rng.choice([2, 30, 200, 1500])); n = int(rng.integers(1, 6_000))
        dist = int(rng.integers(0, 2)); varying = int(rng.random() < 0.5)
        max_entries = int(rng.choice([60, 500, 5000])); max_batch = int(rng.choice([300, 1024, 4096])); seed = int(rng.integers(1, 1 << 30))
        recs = gen_host(seed=seed, n=n, n_keys=n_keys, dist=dist, varying=varying)
        cut = int(rng.integers(0, n + 1))
        try:
            got, st = gpu_generations([recs[:cut], recs[cut:]], max_entries, max_batch=max_batch)
            assert_same_generations(got, oracle_generations([recs], max_entries))
        except AssertionError as e:
            print("FAIL", dict(n_keys=n_keys, n=n, dist=dist, varying=varying, max_entries=max_entries, max_batch=max_batch, seed=seed, cut=cut), str(e)[:300]); sys.exit(1)
    print("ok iterations", it)


def fuzz_features(rng, seconds):
    load_engine_emulation()
    import netobserv_ebpf_agent_b200 as fa
    from test_dns_correlate import dns_stream, run_case
    from test_gpu_features import compare, make_add, make_dns
    t0, it = time.time(), 0
    while time.time() - t0 < seconds:
        it += 1
        seed = int(rng.integers(1, 1 << 30))
        if it % 3 == 0:                                   # K7
            n = int(rng.integers(1, 3000)); nc = int(rng.choice([1, 3, 40, 400])); ni = int(rng.integers(1, 5))
            s = dns_stream(seed, n, n_clients=nc, n_ids=ni, dup=float(rng.random() * 0.6), orphan=float(rng.random() * 0.3))
            cut = int(rng.integers(0, n + 1))
            print("k7", it, dict(seed=seed, n=n, nc=nc, ni=ni, cut=cut), flush=True)
            run_case([s[:cut], s[cut:]] if 0 < cut < n else [s])
            continue
        n_keys = int(rng.choice([3, 50, 600])); n_base = int(rng.integers(0, 4000)); n_feat = int(rng.integers(1, 4000))
        print("k6", it, dict(seed=seed, n_keys=n_keys, n_base=n_base, n_feat=n_feat), flush=True)
        r2 = np.random.default_rng(seed)
        base = gen_host(seed=seed, n=max(n_base, 1), n_keys=n_keys, dist=int(rng.integers(0, 2)), varying=int(rng.random() < 0.3))
        keys = np.unique(np.concatenate([base[:, :40], gen_host(seed=seed + 1, n=200, n_keys=max(2, n_keys // 2))[:, :40]]), axis=0)
        dns = make_dns(r2, keys, n_feat); add = make_add(r2, keys, n_feat)
        om = O.FlowMap()
        with fa.FlowAggEngine(1 << 12, flags=fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS, max_batch=int(rng.choice([500, 2048]))) as eng:
            for o in rng.permutation(3):
                if o == 0: eng.ingest(base); om.account(base)
                if o == 1: eng.ingest_dns(dns); om.fold_dns(dns)
                if o == 2: eng.ingest_additional(add); om.fold_additional(add)
            compare(eng, om)
    print("ok iterations", it)


if __name__ == "__main__":
    mode, seed, seconds = sys.argv[1], int(sys.argv[2]), float(sys.argv[3])
    {"k1": fuzz_k1, "engine": fuzz_engine, "features": fuzz_features}[mode](np.random.default_rng(seed), seconds)
