"""How long does fa_pb_encode (K8) take for one large eviction?

Two batches of 2^20 flows (--n), tiled on the device from 1,024 template rows each:
  typical: an IPv4 flow with one interface and at most one feature block (about 230 bytes of protobuf on average);
  max:     the largest record the engine writes: IPv6, seven interfaces with 16-byte names and 64-byte UDNs, every
           feature block at its widest (about 930 bytes; every CTA of the write kernel is then past its 64 KB stage).
Inputs, output bytes, offsets and keys are all in device memory.  Per batch it prints one JSON line with the median call
time over --reps calls after --warmup untimed ones (host clock around the call, which returns after a stream
synchronise), the output bytes and the GB/s of output written.  The first line names the card and its power limit.
FA_LIB_NAME=<other build>.so times another build of the same library (A/B in separate processes).

  python tools/pb_bench.py
  python tools/pb_bench.py --n 65536 --reps 5
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
sys.path.insert(0, HERE)
import netobserv_ebpf_agent_b200 as fa                                     # noqa: E402
from netobserv_ebpf_agent_b200._lib import lib                             # noqa: E402
from evict_stall import card                                               # noqa: E402
from test_pbflow_edges import AGENT6, MAX_TABLE, MONO, NOW, iface_rows, max_rows, pb_params, rows   # noqa: E402


def batch(kind, n):
    """kind's rows, repeated to n on the device -> [records, dns, additional, pkt_drops, present] tensors."""
    import torch
    t = 1024
    if kind == "max":
        r, d, a, p, pr = max_rows(t)
    else:
        r, d, a, p, pr = rows(t)
        rng = np.random.default_rng(1)
        r["nb_obs"], pr[:] = 0, rng.choice(np.array([0, 1, 2, 4], np.uint8), t)
        r["bytes"] = rng.integers(1, 1 << 40, t)
    r["src_port"] = np.arange(t)
    r["start"] = MONO - np.arange(t) * 1_000_003
    idx = torch.arange(n, device="cuda") % t
    return [torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(t, -1).copy()).cuda()[idx].contiguous()
            for x in (r, d, a, p, pr)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kinds", default="typical,max")
    args = ap.parse_args()
    import torch
    print(json.dumps({**card(), "lib": os.environ.get("FA_LIB_NAME", "libflowagg.so")}), flush=True)
    table, _ = iface_rows(MAX_TABLE)
    prm = pb_params(NOW, MONO, AGENT6, 0, table, len(MAX_TABLE), False)
    with fa.FlowAggEngine(64) as eng:
        for kind in args.kinds.split(","):
            blocks = batch(kind, args.n)                     # kept alive: the calls read them
            ins = [C.c_void_p(x.data_ptr()) for x in blocks]
            need = C.c_size_t(0)
            lib().fa_pb_encode(eng._h, *ins, args.n, C.byref(prm), None, 0, None, None, C.byref(need))
            out = torch.empty(need.value, dtype=torch.uint8, device="cuda")
            offs = torch.empty(args.n + 1, dtype=torch.int64, device="cuda")
            keys = torch.empty((args.n, 32), dtype=torch.uint8, device="cuda")
            dst = [C.c_void_p(out.data_ptr()), need.value, C.c_void_p(offs.data_ptr()), C.c_void_p(keys.data_ptr())]
            times = []
            for i in range(args.warmup + args.reps):
                got = C.c_size_t(0)
                t0 = time.perf_counter()
                rc = lib().fa_pb_encode(eng._h, *ins, args.n, C.byref(prm), *dst, C.byref(got))
                dt = time.perf_counter() - t0
                assert rc == 0 and got.value == need.value, rc
                if i >= args.warmup:
                    times.append(dt)
            ms = float(np.median(times)) * 1e3
            print(json.dumps({"kind": kind, "n": args.n, "bytes_out": need.value, "median_ms": round(ms, 3),
                              "min_ms": round(min(times) * 1e3, 3), "out_GBps": round(need.value / ms / 1e6, 1),
                              "digest": int(out.to(torch.int64).sum().item())}), flush=True)


if __name__ == "__main__":
    main()
