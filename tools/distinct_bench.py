"""How long does fa_distinct_flows take on a full-size table, and what does its second level cost on top of the group scan?

Shapes: those of tools/group_bench.py (ACCOUNTER, 2^25 slots, 2^26 device-generated records, tools/top_flows_bench.py's
fill): 10^6 and 10^7 Zipf-1.1 keys, 10^7 uniform keys, and the 10^7 Zipf table of an engine with RTT and DNS folds.  Per
mask pair (G, D) three calls are warmed up, then timed --reps times each, interleaved, with the host clock around them
(each returns when its output is complete), output into device memory:
  fa_distinct_flows(G, D), fa_group_flows(G | D) (level 1 alone: the same scan over the same table) and fa_group_flows(G).
distinct_ms - group_union_ms is what the second level, the selection and its wait add.  Needs a CUDA device; the first
line names the card and its power limit.

  python tools/distinct_bench.py
  python tools/distinct_bench.py --shapes zipf10m --reps 30
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
from group_bench import N_RECS, SHAPES, SLOTS_LOG2, feature_samples        # noqa: E402
from top_flows_bench import fill                                           # noqa: E402


def mask_pairs():
    """name -> (G, D): port scan, fan-out, clients per service, per dst /120, the window's destinations, distinct ==
    flows, distinct == 1 (twice), byte 39 set in both, three seeded random pairs."""
    gm = fa.group_mask
    ones = np.full(40, 0xFF, np.uint8)
    p = {"scan": (gm(src_prefix=128), gm(dst_port=True)), "fanout": (gm(src_prefix=128), gm(dst_prefix=128)),
         "clients": (gm(proto=True, dst_port=True), gm(src_prefix=128)), "dst120_src": (gm(dst_prefix=120), gm(src_prefix=128)),
         "zero_dst": (gm(), gm(dst_prefix=128)), "ones_ones": (ones, ones.copy()), "src120_zero": (gm(src_prefix=120), gm()),
         "src120_subset": (gm(src_prefix=120), gm(src_prefix=100))}
    g39, d39 = gm(src_prefix=124, proto=True), gm(dst_prefix=128, icmp=True)
    g39[39] = d39[39] = 0xFF
    p["byte39"] = (g39, d39)
    rng = np.random.default_rng(5151)
    for i in range(3):
        g, d = ((rng.random((40, 8)) < 0.12).astype(np.uint8) for _ in range(2))
        p[f"random{i}"] = (np.packbits(g, axis=1).reshape(40), np.packbits(d, axis=1).reshape(40))
    return p


def stats(ms):
    return round(float(np.median(ms)), 3), [round(float(np.percentile(ms, 10)), 3), round(float(np.percentile(ms, 90)), 3)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated: " + ", ".join(SHAPES))
    ap.add_argument("--pairs", default=",".join(mask_pairs()), help="comma-separated mask pairs")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=1 << 24, help="records per generated and ingested chunk")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("distinct_bench.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "distinct_bench", **card(), "reps": a.reps, "warmup": a.warmup})
    buf = torch.empty(a.chunk * 144, dtype=torch.uint8, device="cuda")
    max_entries = 3 << (SLOTS_LOG2 - 2)
    pairs = mask_pairs()
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
            emit({"shape": name, "slots": 1 << SLOTS_LOG2, "live_flows": live, "feature_folds": feats})
            out = torch.empty(live * 88, dtype=torch.uint8, device="cuda")
            for pname in a.pairs.split(","):
                g, d = pairs[pname]
                u = g | d
                n = {}

                def distinct():
                    got = C.c_size_t(0)
                    check(lib().fa_distinct_flows(eng._h, g.ctypes.data, d.ctypes.data, 0, out.data_ptr(), live, C.byref(got)))
                    n["groups"] = got.value

                def group_union():
                    got = C.c_size_t(0)
                    check(lib().fa_group_flows(eng._h, u.ctypes.data, out.data_ptr(), live, C.byref(got)))
                    n["pairs"] = got.value

                def group():
                    got = C.c_size_t(0)
                    check(lib().fa_group_flows(eng._h, g.ctypes.data, out.data_ptr(), live, C.byref(got)))

                calls = {"distinct": distinct, "group_union": group_union, "group": group}
                for fn in calls.values():
                    for _ in range(a.warmup):
                        fn()
                ms = {k: [] for k in calls}
                for _ in range(a.reps):                              # interleaved: drift hits the three alike
                    for k, fn in calls.items():
                        t0 = time.perf_counter()
                        fn()
                        ms[k].append(1e3 * (time.perf_counter() - t0))
                line = {"shape": name, "pair": pname, "groups": n["groups"], "pairs": n["pairs"]}
                for k in calls:
                    line[k + "_ms"], line[k + "_p10_p90_ms"] = stats(np.array(ms[k]))
                line["second_level_ms"] = round(line["distinct_ms"] - line["group_union_ms"], 3)
                emit(line)
            del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
