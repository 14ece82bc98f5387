"""Feature samples through the multi-GPU ABI: samples/s of fa_sharded_ingest_additional and fa_sharded_ingest_dns for
1, 2 and 4 shards on one GPU (and on distinct GPUs when the machine has several), next to one engine's
fa_ingest_additional / fa_ingest_dns on the same samples, plus the time of one round split into the stable route
(fa_route_peer_samples) and the per-segment folds (fa_ingest_samples_counted), read with CUDA events.

Shards on one GPU measure the route and fold overhead of the exchange, not NVLink: every "peer" store is local.

    python tools/sharded_features_bench.py [--samples 8388608] [--flows 1000000] [--round 1048576] [--reps 3] [--out f.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FEATS = 1 | 2                               # FA_F_ENABLE_RTT | FA_F_ENABLE_DNS
NO_FULL_CUT = 8


def samples(kind, n, n_flows, seed):
    """n random samples (uniform over n_flows keys, per-sample random values) as one flat pinned-friendly uint8 array."""
    import oracle_lib as O
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, 256, (n_flows, 40), dtype=np.uint8)
    keys[:, 39] = 0
    r = np.zeros(n, dtype=O.ADDREC_DTYPE if kind == 0 else O.DNSREC_DTYPE)
    r["id"] = keys[rng.integers(0, n_flows, n)]
    blk = r["add"] if kind == 0 else r["dns"]
    blk["start"] = rng.integers(1, 1 << 40, n)
    blk["end"] = blk["start"] + rng.integers(0, 1 << 20, n)
    if kind == 0:
        blk["rtt"] = rng.integers(0, 1 << 30, n)
    else:
        blk["latency"] = rng.integers(0, 1 << 30, n)
        blk["id"] = rng.integers(0, 1 << 16, n)
        blk["errno"] = rng.integers(0, 4, n)
    r["add" if kind == 0 else "dns"] = blk
    return r


def pinned_copy(arr):
    import torch
    t = torch.empty(arr.nbytes, dtype=torch.uint8, pin_memory=True)
    t.numpy()[:] = arr.view(np.uint8).reshape(-1)
    return t


def check_s(L, rc):
    if rc < 0:
        raise RuntimeError(L.fa_sharded_last_error().decode())


def sharded_rate(devices, kind, pin, n, n_flows, round_cap, reps):
    from netobserv_ebpf_agent_b200._lib import FA_ABI_VERSION, Config, lib
    L = lib()
    cfg = Config(abi_version=FA_ABI_VERSION, device=0, mode=0, flags=FEATS, max_entries=2 * n_flows, max_batch=round_cap)
    h = C.c_void_p()
    check_s(L, L.fa_sharded_create(C.byref(cfg), (C.c_int32 * len(devices))(*devices), len(devices), C.byref(h)))
    f = L.fa_sharded_ingest_additional if kind == 0 else L.fa_sharded_ingest_dns
    best = None
    try:
        out = np.zeros((2 * n_flows, 144), np.uint8)
        for r in range(reps + 1):                                           # the first pass warms up
            check_s(L, L.fa_sharded_sync(h))
            t0 = time.perf_counter()
            check_s(L, f(h, pin.data_ptr(), n))
            check_s(L, L.fa_sharded_sync(h))
            dt = time.perf_counter() - t0
            got = C.c_size_t(0)
            check_s(L, L.fa_sharded_evict(h, out.ctypes.data, len(out), C.byref(got)))
            if r and (best is None or dt < best):
                best = dt
    finally:
        L.fa_sharded_destroy(h)
    return n / best


def single_rate(kind, pin, n, n_flows, reps):
    import netobserv_ebpf_agent_b200 as fa
    best = None
    # fa_ingest_* refuses a call whose samples could overfill the table: room for n flows
    with fa.FlowAggEngine(max(n, 2 * n_flows), flags=FEATS) as eng:
        for r in range(reps + 1):
            eng.sync()
            t0 = time.perf_counter()
            (eng.ingest_additional if kind == 0 else eng.ingest_dns)(pin)
            eng.sync()
            dt = time.perf_counter() - t0
            eng.evict(cap=max(n, 2 * n_flows))
            if r and (best is None or dt < best):
                best = dt
    return n / best


def round_split(k, kind, dev_samples, n_flows, round_cap, reps):
    """One round of k shards on GPU 0 through the engine-level calls: k sources route a slice of round_cap samples each
    into their segments of k owners' buffers, then each owner folds its k segments; CUDA events on one stream."""
    import torch
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import check, lib
    L = lib()
    rb = 72 if kind == 0 else 104
    st = torch.cuda.Stream()
    owners = [fa.FlowAggEngine(2 * n_flows // k + 1024, flags=FEATS | NO_FULL_CUT, max_batch=k * round_cap, cuda_stream=st.cuda_stream)
              for _ in range(k)]
    recv = [torch.empty(k * round_cap * rb, dtype=torch.uint8, device="cuda") for _ in range(k)]
    seg_n = [torch.zeros(k, dtype=torch.int64, device="cuda") for _ in range(k)]
    over = torch.zeros(2, dtype=torch.int64, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    route_ms, fold_ms = [], []
    for r in range(reps + 1):
        with torch.cuda.stream(st):
            ev[0].record(st)
            for i in range(k):
                segs = (C.c_void_p * k)(*[recv[j].data_ptr() + i * round_cap * rb for j in range(k)])
                cnts = (C.c_void_p * k)(*[seg_n[j].data_ptr() + 8 * i for j in range(k)])
                src = dev_samples.data_ptr() + ((r * k + i) * round_cap % (len(dev_samples) // rb - round_cap)) * rb
                check(L.fa_route_peer_samples(owners[i]._h, kind, src, None, round_cap, k, i, segs, cnts, round_cap, over.data_ptr()))
            ev[1].record(st)
            for j in range(k):
                for i in range(k):
                    check(L.fa_ingest_samples_counted(owners[j]._h, kind, recv[j].data_ptr() + i * round_cap * rb,
                                                      seg_n[j].data_ptr() + 8 * i, round_cap, 1))
            ev[2].record(st)
        st.synchronize()
        if r:
            route_ms.append(ev[0].elapsed_time(ev[1]))
            fold_ms.append(ev[1].elapsed_time(ev[2]))
    assert int(over[0]) == 0
    for o in owners:
        o.close()
    return min(route_ms), min(fold_ms)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                                   # noqa: BLE001
        pl = f"unknown ({e})"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1 << 23)
    ap.add_argument("--flows", type=int, default=1_000_000)
    ap.add_argument("--round", type=int, default=1 << 20, help="max_batch: samples per GPU and round")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    name, pl = card()
    res = {"card": name, "power_limit": pl, "samples": a.samples, "flows": a.flows, "round_cap": a.round, "rows": []}
    sets = [[0], [0, 0], [0, 0, 0, 0]]
    if torch.cuda.device_count() > 1:
        sets += [list(range(min(k, torch.cuda.device_count()))) for k in (2, 4) if torch.cuda.device_count() >= k]
    for kind, what in ((0, "additional"), (1, "dns")):
        s = samples(kind, a.samples, a.flows, 7 + kind)
        pin = pinned_copy(s)
        dev = pin.to("cuda")
        one = single_rate(kind, pin, a.samples, a.flows, a.reps)
        res["rows"].append({"kind": what, "shards": "single engine", "samples_per_s": one})
        for devs in sets:
            rate = sharded_rate(devs, kind, pin, a.samples, a.flows, a.round, a.reps)
            row = {"kind": what, "shards": "x".join(map(str, devs)), "samples_per_s": rate}
            if len(set(devs)) == 1:
                row["round_route_ms"], row["round_fold_ms"] = round_split(len(devs), kind, dev, a.flows, a.round, a.reps)
            res["rows"].append(row)
        del dev
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
