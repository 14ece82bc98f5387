"""How long does fa_expire_flows take against evicting the whole table, and how fast does K1 fold afterwards?

Shape: bench.py's zipf10m table (ACCOUNTER, 2^25 slots, 10^7 Zipf keys, 2^26 device-generated records; ts(i) = t0 + i, so
a flow's end is the index of its last record).  Per target fraction (default 1 %, 10 %, 50 %, 90 % of the live flows) the
table is filled again from scratch and expired once with an idle cut at that quantile of the flows' end timestamps, output
into device memory; the call is timed with the host clock around a call that returns after its outputs are complete.
Then K1 folds the next 2^26 records (indices 2^26 .. 2^27) into the survivors, timed with the host clock around the
ingest and a sync, in records per second.  Yardstick on the same table: fa_evict_ex into device memory, then K1 on the
same next records into the empty table.  Each configuration is measured --reps times (each on a fresh fill: the call is
destructive) and the median printed.  Needs a CUDA device; the first line names the card and its power limit.

  python tools/expire_bench.py
  python tools/expire_bench.py --fractions 0.1,0.5 --reps 3
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

T0 = 1_000_000


def ingest_timed(eng, gp, first, n, chunk, buf):
    """K1 over generated records [first, first + n): generation is outside the clock, ingest + sync inside."""
    secs = 0.0
    for lo in range(first, first + n, chunk):
        c = min(chunk, first + n - lo)
        eng.gen_records(gp, lo, c, buf.data_ptr())
        eng.sync()
        t0 = time.perf_counter()
        rc, took = eng.ingest(buf.data_ptr(), c)
        eng.sync()
        secs += time.perf_counter() - t0
        assert rc == fa.FA_OK and took == c, (rc, took)
    return secs


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shape", default="zipf10m", choices=list(SHAPES))
    ap.add_argument("--fractions", default="0.01,0.1,0.5,0.9")
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--chunk", type=int, default=1 << 24, help="records per generated and ingested chunk")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("expire_bench.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "expire_bench", **card(), "reps": a.reps})
    mode, slots_log2, n_keys, dist, n_recs = SHAPES[a.shape]
    max_entries = 3 << (slots_log2 - 2)
    gp = fa.GenParams(seed=7, n_keys=n_keys, dist=dist, zipf_s_milli=1100, t0_ns=T0, varying_desc=0)
    buf = torch.empty(a.chunk * 144, dtype=torch.uint8, device="cuda")
    with fa.FlowAggEngine(max_entries, mode=mode, max_batch=a.chunk) as eng:
        out = torch.empty(max_entries * 144, dtype=torch.uint8, device="cuda")
        eo = EvictOut(records=out.data_ptr())
        got = C.c_size_t(0)
        # the yardstick, and the end timestamps the idle cuts are taken from
        def clear():
            check(lib().fa_evict_ex(eng._h, C.byref(eo), max_entries, C.byref(got)))

        ev_ms, k1_empty, ends = [], [], None
        for _ in range(a.reps):
            fill(eng, gp, n_recs, a.chunk, buf)
            live = eng.live_flows()
            t0 = time.perf_counter()
            clear()
            ev_ms.append(1e3 * (time.perf_counter() - t0))
            if ends is None:
                ends = out[: got.value * 144].view(-1, 144)[:, 48:56].contiguous().view(torch.int64).cpu().numpy().astype(np.float64)
            k1_empty.append(n_recs / ingest_timed(eng, gp, n_recs, n_recs, a.chunk, buf))
            clear()
        emit({"shape": a.shape, "slots": 1 << slots_log2, "live_flows": live, "evict_ex_device_ms": round(float(np.median(ev_ms)), 3),
              "k1_after_evict_Mrec_per_s": round(float(np.median(k1_empty)) / 1e6, 1)})
        now = T0 + n_recs
        fill(eng, gp, n_recs, a.chunk, buf)                  # untimed: the first call allocates the scratch and staging
        check(lib().fa_expire_flows(eng._h, now, n_recs + 1, 0, C.byref(eo), max_entries, C.byref(got)))
        assert got.value == 0
        clear()
        for f in [float(x) for x in a.fractions.split(",")]:
            idle = now - int(np.quantile(ends, f))
            ms, k1, n_exp = [], [], 0
            for _ in range(a.reps):
                fill(eng, gp, n_recs, a.chunk, buf)
                t0 = time.perf_counter()
                check(lib().fa_expire_flows(eng._h, now, idle, 0, C.byref(eo), max_entries, C.byref(got)))
                ms.append(1e3 * (time.perf_counter() - t0))
                n_exp = got.value
                k1.append(n_recs / ingest_timed(eng, gp, n_recs, n_recs, a.chunk, buf))
                clear()
            emit({"shape": a.shape, "fraction_target": f, "expired": n_exp, "expired_fraction": round(n_exp / live, 4),
                  "expire_ms": round(float(np.median(ms)), 3), "evict_ex_ms": round(float(np.median(ev_ms)), 3),
                  "k1_after_expire_Mrec_per_s": round(float(np.median(k1)) / 1e6, 1)})
        del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
