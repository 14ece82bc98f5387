"""How long does fa_group_flows take on a full-size table, and how close does it come to HBM rate?

Shapes: the headline sizing (ACCOUNTER, 2^25 slots, 2^26 device-generated records, tools/top_flows_bench.py's fill):
10^6 and 10^7 Zipf-1.1 keys and 10^7 uniform keys, plus the 10^7 Zipf table of an engine with RTT and DNS folds where
2^20 flows carry additional and DNS samples (the row reader then reads feature lines too).  Per mask (all-zero: 1 group;
proto + dst port: few; src /120: many; all-ones: one per flow) the call is warmed up, then timed --reps times with the host
clock around it (it returns when its output is complete), output into device memory.  fa_top_flows(k = 10) is timed the
same way as the cost of one existing full-table read-side scan.

Byte model (printed with each line, and the fraction of 3.35 TB/s it implies): the occupancy bitmap (slots / 8), per live
flow two 32-byte sectors of the identity line (the key) and one of the hot line, plus 64 B per feature line the engine
keeps (its first word, and the sample times where it has samples); per group its 96-byte slot three times (the scan's
claim and updates, the emit's read, the emit's zeroing), 88 B of row and 8 B of list.  Needs a CUDA device; the first line
names the card and its power limit.

  python tools/group_bench.py
  python tools/group_bench.py --shapes zipf10m --reps 30
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
from top_flows_bench import fill                                           # noqa: E402

HBM_BPS = 3.35e12                                                          # H100 SXM 80 GB HBM3, spec sheet
SHAPES = {   # name: (keys, distribution, feature folds)
    "zipf1m": (1_000_000, fa.FA_GEN_ZIPF, False),
    "zipf10m": (10_000_000, fa.FA_GEN_ZIPF, False),
    "uniform10m": (10_000_000, fa.FA_GEN_UNIFORM, False),
    "zipf10m_rtt_dns": (10_000_000, fa.FA_GEN_ZIPF, True),
}
SLOTS_LOG2, N_RECS = 25, 1 << 26
MASKS = {"zero": fa.group_mask(), "proto_dport": fa.group_mask(proto=True, dst_port=True),
         "src120": fa.group_mask(src_prefix=120), "ones": np.full(40, 0xFF, np.uint8)}


def feature_samples(keys, rng):
    """One additional (72 B) and one DNS (104 B) sample per key: times after the base records, an RTT, a latency."""
    n = len(keys)
    add, dns = np.zeros((n, 72), np.uint8), np.zeros((n, 104), np.uint8)
    add[:, :40], dns[:, :40] = keys, keys
    t = (1 << 40) + rng.integers(0, 1 << 30, n).astype(np.uint64)
    for blk in (add, dns):
        blk[:, 40:48] = t.view(np.uint8).reshape(n, 8)                      # start
        blk[:, 48:56] = (t + np.uint64(1000)).view(np.uint8).reshape(n, 8)   # end
    add[:, 56:64] = rng.integers(1, 1 << 30, n).astype(np.uint64).view(np.uint8).reshape(n, 8)   # flow_rtt
    dns[:, 56:64] = rng.integers(1, 1 << 30, n).astype(np.uint64).view(np.uint8).reshape(n, 8)   # latency
    return add, dns


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ms.append(1e3 * (time.perf_counter() - t0))
    return np.array(ms)


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
        sys.exit("group_bench.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "group_bench", **card(), "reps": a.reps, "warmup": a.warmup})
    buf = torch.empty(a.chunk * 144, dtype=torch.uint8, device="cuda")
    slots = 1 << SLOTS_LOG2
    max_entries = 3 << (SLOTS_LOG2 - 2)
    for name in a.shapes.split(","):
        keys, dist, feats = SHAPES[name]
        flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS if feats else 0
        gp = fa.GenParams(seed=7, n_keys=keys, dist=dist, zipf_s_milli=1100, t0_ns=1_000_000, varying_desc=0)
        with fa.FlowAggEngine(max_entries, flags=flags, max_batch=a.chunk) as eng:
            fill(eng, gp, N_RECS, a.chunk, buf)
            if feats:
                eng.gen_records(gp, 0, 1 << 20, buf.data_ptr())
                eng.sync()
                k = np.unique(buf[: (1 << 20) * 144].view(-1, 144)[:, :40].cpu().numpy(), axis=0)
                add, dns = feature_samples(k, np.random.default_rng(8))
                eng.ingest_additional(add)
                eng.ingest_dns(dns)
            live = eng.live_flows()
            out = torch.empty(live * 88, dtype=torch.uint8, device="cuda")
            got = C.c_size_t(0)
            top = torch.empty(10 * 144, dtype=torch.uint8, device="cuda")
            eo = EvictOut(records=top.data_ptr())
            ms = timed(lambda: check(lib().fa_top_flows(eng._h, fa.FA_TOP_BYTES, 10, C.byref(eo), C.byref(got))), a.warmup, a.reps)
            emit({"shape": name, "slots": slots, "live_flows": live, "feature_folds": feats, "top_flows_k10_ms": round(float(np.median(ms)), 3),
                  "top_flows_k10_p10_p90_ms": [round(float(np.percentile(ms, 10)), 3), round(float(np.percentile(ms, 90)), 3)]})
            feat_lines = 2 if feats else 0
            for mname, m in MASKS.items():
                def call():
                    check(lib().fa_group_flows(eng._h, m.ctypes.data, out.data_ptr(), live, C.byref(got)))
                ms = timed(call, a.warmup, a.reps)
                groups = got.value
                model = slots / 8 + live * (64 + 32 + 64 * feat_lines) + groups * (3 * 96 + 88 + 8)
                med = float(np.median(ms))
                emit({"shape": name, "mask": mname, "groups": groups, "median_ms": round(med, 3),
                      "p10_p90_ms": [round(float(np.percentile(ms, 10)), 3), round(float(np.percentile(ms, 90)), 3)],
                      "model_bytes": int(model), "model_fraction_of_3_35_TBps": round(model / (med * 1e-3) / HBM_BPS, 3)})
            del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
