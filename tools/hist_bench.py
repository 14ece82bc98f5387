"""How long does fa_histogram_flows take next to fa_group_flows on the same full-size table?

Shapes: the headline sizing (ACCOUNTER, 2^25 slots, 2^26 device-generated records, tools/top_flows_bench.py's fill)
with 10^6 Zipf-1.1 keys (about 10^6 live flows) and 10^7 Zipf-1.1 keys (about 4·10^6 live flows).  Per mask (proto + dst
port: a coarse mask, few groups; all-ones: one group per flow) fa_group_flows is timed, then fa_histogram_flows of the
flow duration (FA_HIST_DURATION: the row times, the hot line's start and end) with 10 and with 63 bounds.  Each call is
warmed up, then timed --reps times with the host clock around it (it returns when its output is complete), output into
device memory.  fa_histogram_flows runs the group scan of fa_group_flows first, so the difference of the two medians is
the cost of the index, the second scan and the emit.  Needs a CUDA device; the first line names the card and its power
limit.

  python tools/hist_bench.py
  python tools/hist_bench.py --shapes zipf10m --reps 30
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
from netobserv_ebpf_agent_b200._lib import check, lib                      # noqa: E402
from evict_stall import card                                               # noqa: E402
from top_flows_bench import fill                                           # noqa: E402

SHAPES = {"zipf1m": 1_000_000, "zipf10m": 10_000_000}                      # name: keys (Zipf 1.1)
SLOTS_LOG2, N_RECS = 25, 1 << 26
MASKS = {"proto_dport": fa.group_mask(proto=True, dst_port=True), "ones": np.full(40, 0xFF, np.uint8)}
BOUNDS = {10: np.array([10 ** i for i in range(3, 13)], np.uint64),                        # 1 us .. 1000 s in ns
          63: np.array([1 << i for i in range(63)], np.uint64)}                            # 2^0 .. 2^62


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ms.append(1e3 * (time.perf_counter() - t0))
    return np.array(ms)


def stats(ms):
    return {"median_ms": round(float(np.median(ms)), 3),
            "p10_p90_ms": [round(float(np.percentile(ms, 10)), 3), round(float(np.percentile(ms, 90)), 3)]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated: " + ", ".join(SHAPES))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=1 << 24, help="records per generated and ingested chunk")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("hist_bench.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "hist_bench", **card(), "reps": a.reps, "warmup": a.warmup})
    buf = torch.empty(a.chunk * 144, dtype=torch.uint8, device="cuda")
    max_entries = 3 << (SLOTS_LOG2 - 2)
    for name in a.shapes.split(","):
        gp = fa.GenParams(seed=7, n_keys=SHAPES[name], dist=fa.FA_GEN_ZIPF, zipf_s_milli=1100, t0_ns=1_000_000, varying_desc=0)
        with fa.FlowAggEngine(max_entries, max_batch=a.chunk) as eng:
            fill(eng, gp, N_RECS, a.chunk, buf)
            live = eng.live_flows()
            out = torch.empty(live * fa.hist_dtype(63).itemsize, dtype=torch.uint8, device="cuda")
            got = C.c_size_t(0)
            for mname, m in MASKS.items():
                ms = timed(lambda: check(lib().fa_group_flows(eng._h, m.ctypes.data, out.data_ptr(), live, C.byref(got))),
                           a.warmup, a.reps)
                emit({"shape": name, "live_flows": live, "mask": mname, "call": "fa_group_flows", "groups": got.value, **stats(ms)})
                for nb, b in BOUNDS.items():
                    def call():
                        check(lib().fa_histogram_flows(eng._h, m.ctypes.data, fa.FA_HIST_DURATION, b.ctypes.data, nb,
                                                       out.data_ptr(), live, C.byref(got)))
                    ms = timed(call, a.warmup, a.reps)
                    emit({"shape": name, "live_flows": live, "mask": mname, "call": "fa_histogram_flows", "value": "duration",
                          "n_bounds": nb, "groups": got.value, **stats(ms)})
            del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
