"""How long does fa_lookup_flows take, and does its cost follow the number of keys rather than the table?

Shapes: zipf10m and uniform10m ACCOUNTER tables at bench.py's size (2^25 slots), and a uniform KERNEL_MAP table at
2^24 slots, each built from device-generated records.  Per shape, n keys (10^2 .. 10^7, device memory), hit ratio and
output memory (device, pinned host: the records block and `found`) it prints one JSON line with the median call time over
--reps calls (host clock around a call that returns after its outputs are complete, one untimed call first).
  hit ratio 1.0: the keys of the first n generated records (every one is live; hot flows repeat, as lookups of top
                 talkers would);
  hit ratio 0.0: keys of a disjoint generator seed (every one is absent: the probe walks the chain to an empty slot).
Yardsticks on the same table: fa_top_flows(k = n) for n <= 10^6 and fa_evict_ex, both into device memory.

The bytes of a call are a MODEL kept here, not a measurement: per key 40 B of key, 64 B per probed slot (the two sectors
that hold the key and the tag; one slot per key assumed, the tables are at load <= 0.30), 144 B of row written, 9 B of
slot and found scratch; per hit 128 + 32 B gathered (identity and hot / metric line).  No feature folds here, so no
feature blocks.  Needs a CUDA device; the first line names the card and its power limit.

  python tools/lookup_bench.py
  python tools/lookup_bench.py --shapes zipf10m --ns 100,10000 --reps 3
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import netobserv_ebpf_agent_b200 as fa                                     # noqa: E402
from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib            # noqa: E402
from evict_stall import card                                               # noqa: E402
from top_flows_bench import SHAPES, fill                                   # noqa: E402


def model_bytes(n, hits):
    """The bytes model of one call (see the module docstring)."""
    return n * (40 + 64 + 144 + 9) + hits * (128 + 32)


class Out:
    """The records block and `found` for n rows, in device memory (torch) or pinned host memory."""

    def __init__(self, n, device):
        import torch
        self.device = device
        if device:
            self.t = torch.empty(n * 145, dtype=torch.uint8, device="cuda")
            self.rec, self.found = self.t.data_ptr(), self.t.data_ptr() + n * 144
        else:
            p = C.c_void_p(); check(lib().fa_host_alloc(n * 145, C.byref(p)))
            self.p = p
            self.rec, self.found = p.value, p.value + n * 144

    def close(self):
        if not self.device:
            lib().fa_host_free(self.p)


def keys_of(eng, gp, n, buf, chunk):
    """Device tensor of the 40-byte keys of generated records [0, n)."""
    import torch
    keys = torch.empty((n, 40), dtype=torch.uint8, device="cuda")
    for first in range(0, n, chunk):
        c = min(chunk, n - first)
        eng.gen_records(gp, first, c, buf.data_ptr())
        eng.sync()
        keys[first:first + c] = buf[: c * 144].view(c, 144)[:, :40]
    torch.cuda.synchronize()
    return keys


def timed(call, reps):
    times = []
    for r in range(reps + 1):
        t0 = time.perf_counter()
        call()
        if r:
            times.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(times)), 4), round(1e3 * min(times), 4)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated: " + ", ".join(SHAPES))
    ap.add_argument("--ns", default="100,10000,1000000,10000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=1 << 24, help="records per generated and ingested chunk")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("lookup_bench.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "lookup_bench", **card(), "reps": a.reps})
    ns = [int(x) for x in a.ns.split(",")]
    buf = torch.empty(a.chunk * 144, dtype=torch.uint8, device="cuda")
    for name in a.shapes.split(","):
        mode, slots_log2, n_keys, dist, n_recs = SHAPES[name]
        max_entries = 3 << (slots_log2 - 2)
        gp = fa.GenParams(seed=7, n_keys=n_keys, dist=dist, zipf_s_milli=1100, t0_ns=1_000_000, varying_desc=0)
        absent_gp = fa.GenParams(seed=8, n_keys=1 << 32, dist=fa.FA_GEN_UNIFORM, zipf_s_milli=1100, t0_ns=1_000_000, varying_desc=0)
        with fa.FlowAggEngine(max_entries, mode=mode, max_batch=a.chunk) as eng:
            fill(eng, gp, n_recs, a.chunk, buf)
            live = eng.live_flows()
            emit({"shape": name, "slots": 1 << slots_log2, "live_flows": live})
            for ratio, kg in ((1.0, gp), (0.0, absent_gp)):
                keys_all = keys_of(eng, kg, max(ns), buf, a.chunk)
                for n in ns:
                    keys = keys_all[:n]
                    for device in (True, False):
                        o = Out(n, device)
                        eo = EvictOut(records=o.rec)
                        got = C.c_size_t(0)
                        ms, ms_min = timed(lambda: check(lib().fa_lookup_flows(eng._h, C.c_void_p(keys.data_ptr()), n, C.byref(eo),
                                                                               C.c_void_p(o.found), C.byref(got))), a.reps)
                        o.close()
                        mb = model_bytes(n, got.value)
                        emit({"shape": name, "n": n, "hit_ratio": ratio, "found": got.value, "out": "device" if device else "pinned_host",
                              "ms_median": ms, "ms_min": ms_min, "model_bytes": mb,
                              "model_GBps_at_median": round(mb / (ms * 1e-3) / 1e9, 2)})
                del keys_all
            # yardsticks on the same table, into device memory: fa_top_flows(k = n), then fa_evict_ex
            for n in [x for x in ns if x <= 1_000_000]:
                out = torch.empty(n * 144, dtype=torch.uint8, device="cuda")
                eo = EvictOut(records=out.data_ptr())
                got = C.c_size_t(0)
                ms, ms_min = timed(lambda: check(lib().fa_top_flows(eng._h, fa.FA_TOP_BYTES, n, C.byref(eo), C.byref(got))), a.reps)
                emit({"shape": name, "top_flows_k": n, "ms_median": ms, "ms_min": ms_min})
                del out
            out = torch.empty(live * 144, dtype=torch.uint8, device="cuda")
            eo = EvictOut(records=out.data_ptr())
            got = C.c_size_t(0)
            check(lib().fa_evict_ex(eng._h, C.byref(eo), live, C.byref(got)))
            fill(eng, gp, n_recs, a.chunk, buf)
            t0 = time.perf_counter()
            check(lib().fa_evict_ex(eng._h, C.byref(eo), live, C.byref(got)))
            emit({"shape": name, "evict_ex_device_ms": round(1e3 * (time.perf_counter() - t0), 3), "flows": got.value})
            del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
