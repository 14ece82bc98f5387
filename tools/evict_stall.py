"""How long does an eviction stall ingest?  KERNEL_MAP mode with RTT + DNS folds, blocking fa_evict vs
FA_F_NONBLOCKING_EVICT, measured in the same process and alternating.

One thread ingests device-resident records in calls of --call records (the map update of flow_monitor) while an
evictor thread calls fa_evict_ex into pinned host memory every --period seconds (records, dns, additional, rtt_min and
present blocks, as a map-path Fetcher would).  Per window and mode it prints one JSON line: the latency of every ingest
call (p50 / p99 / max, host clock around the call) and records/s (records over the window, closed by a device
synchronise).  The records come from a pre-generated pool of --pool calls over --keys uniform keys, so the map holds
about --keys x (1 - e^(-pool x call / keys)) flows once warm.  Needs a CUDA device; the first line names the card and
its power limit.

  python tools/evict_stall.py                                  # about 10 M flows in a 2^24-slot map
  python tools/evict_stall.py --keys 2000000 --slots-log2 22   # smaller
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import netobserv_ebpf_agent_b200 as fa                     # noqa: E402
from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib   # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"card": name, "power_limit": power}
    except Exception as ex:                                # the numbers are still printed; the card is then unknown
        return {"card": "unknown", "power_limit": "unknown", "error": str(ex)}


class HostBlocks:
    """Pinned host output blocks of fa_evict_ex for `cap` flows (no packet-drop block: the engine does not fold drops)."""

    WIDTHS = {"records": 144, "dns": 64, "additional": 32, "rtt_min": 8, "present": 1}

    def __init__(self, cap):
        self.cap, self.ptr = cap, {}
        for k, w in self.WIDTHS.items():
            p = C.c_void_p()
            check(lib().fa_host_alloc(cap * w, C.byref(p)))
            self.ptr[k] = p.value
        self.out = EvictOut(records=self.ptr["records"], dns=self.ptr["dns"], additional=self.ptr["additional"],
                            pkt_drops=None, rtt_min=self.ptr["rtt_min"], present=self.ptr["present"])

    def evict(self, eng):
        got = C.c_size_t(0)
        check(lib().fa_evict_ex(eng._h, C.byref(self.out), self.cap, C.byref(got)))
        return got.value

    def close(self):
        for p in self.ptr.values():
            lib().fa_host_free(C.c_void_p(p))


def window(eng, pool, call, seconds, period, blocks):
    """One timed window: ingest calls back to back, an eviction every `period` seconds on another thread."""
    lat, evictions, stop = [], [], threading.Event()

    def evictor():
        nxt = time.perf_counter() + period
        while not stop.wait(max(0.0, nxt - time.perf_counter())):
            t0 = time.perf_counter()
            n = blocks.evict(eng)
            evictions.append((n, time.perf_counter() - t0))
            nxt += period

    eng.sync()
    t = threading.Thread(target=evictor)
    t_start = time.perf_counter()
    t.start()
    calls = 0
    try:
        while time.perf_counter() - t_start < seconds:
            p = pool[calls % len(pool)]
            t0 = time.perf_counter()
            eng.ingest(p, call)
            lat.append(time.perf_counter() - t0)
            calls += 1
    finally:
        stop.set()
        t.join()
    eng.sync()
    elapsed = time.perf_counter() - t_start
    ms = np.array(lat) * 1e3
    return {"calls": calls, "p50_ms": round(float(np.percentile(ms, 50)), 3), "p99_ms": round(float(np.percentile(ms, 99)), 3),
            "max_ms": round(float(ms.max()), 3), "records_per_s": round(calls * call / elapsed, 1), "window_s": round(elapsed, 3),
            "evictions": len(evictions), "flows_per_eviction": int(np.mean([n for n, _ in evictions])) if evictions else 0,
            "eviction_s_mean": round(float(np.mean([s for _, s in evictions])), 4) if evictions else 0.0}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--slots-log2", type=int, default=24, help="map slots = 2^this (max_entries = 3/4 of them)")
    ap.add_argument("--keys", type=int, default=11_000_000, help="distinct keys of the record stream")
    ap.add_argument("--call", type=int, default=1 << 20, help="records per fa_ingest call")
    ap.add_argument("--pool", type=int, default=32, help="pre-generated device calls, cycled")
    ap.add_argument("--seconds", type=float, default=8.0, help="length of one timed window")
    ap.add_argument("--period", type=float, default=2.0, help="seconds between evictions")
    ap.add_argument("--reps", type=int, default=2, help="windows per mode, alternating the modes")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("evict_stall.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "evict_stall", **card(), "slots": 1 << a.slots_log2, "keys": a.keys, "call": a.call, "pool": a.pool,
          "seconds": a.seconds, "period": a.period})
    max_entries = 3 << (a.slots_log2 - 2)
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_RINGBUF_FALLBACK
    modes = {"blocking": flags, "nonblocking": flags | fa.FA_F_NONBLOCKING_EVICT}
    engines = {m: fa.FlowAggEngine(max_entries, mode=fa.FA_MODE_KERNEL_MAP, flags=f, max_batch=a.call) for m, f in modes.items()}
    gp = fa.GenParams(seed=17, n_keys=a.keys, dist=fa.FA_GEN_UNIFORM, zipf_s_milli=0, t0_ns=1_000_000, varying_desc=0)
    pool = [torch.empty(a.call * 144, dtype=torch.uint8, device="cuda") for _ in range(a.pool)]
    eng0 = engines["blocking"]
    for i, t in enumerate(pool):
        eng0.gen_records(gp, i * a.call, a.call, t.data_ptr())
    eng0.sync()
    ptrs = [t.data_ptr() for t in pool]
    blocks = HostBlocks(max_entries)
    try:
        for rep in range(a.reps):
            for m, eng in engines.items():
                for p in ptrs:                              # warm: the map holds its steady-state flows, untimed
                    eng.ingest(p, a.call)
                blocks.evict(eng)
                for p in ptrs:
                    eng.ingest(p, a.call)
                r = window(eng, ptrs, a.call, a.seconds, a.period, blocks)
                st = eng.stats()                            # non-zero: the map was full (--keys too large for the slots)
                emit({"mode": m, "rep": rep, **r, "ringbuf_spilled": st["ringbuf_spilled"]})
                blocks.evict(eng)
    finally:
        blocks.close()
        for eng in engines.values():
            eng.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
