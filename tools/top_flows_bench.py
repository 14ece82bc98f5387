"""How long does fa_top_flows take on a full-size table, next to fa_evict_ex of the same table?

Shapes: zipf10m and uniform10m ACCOUNTER tables at bench.py's size (2^25 slots), and a uniform KERNEL_MAP table at
2^24 slots, each built from device-generated records.  Per shape, metric (bytes, packets), k (100, 10^4, 10^6) and
output memory (device, pinned host) it prints one JSON line with the median call time over --reps calls (host clock
around a call that returns after its outputs are complete, one untimed call first).  Then fa_evict_ex of the same table
into device memory (the yardstick; the table is re-filled and evicted once untimed first).

The select's passes are recomputed on the host from the evicted flows (numpy restatement of the radix select in
csrc/evict.cu): for each pass, the flows whose hash had to be computed, and the bytes it reads by the model
slots / 8 (bitmap) + 32 B per live flow (the sector of its metric word) + 64 B per hashed flow (two key sectors).
Needs a CUDA device; the first line names the card and its power limit.

  python tools/top_flows_bench.py
  python tools/top_flows_bench.py --shapes zipf10m --reps 3
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

SHAPES = {   # name: (mode, slots_log2, keys, distribution, records)
    "zipf10m": (fa.FA_MODE_ACCOUNTER, 25, 10_000_000, fa.FA_GEN_ZIPF, 1 << 26),
    "uniform10m": (fa.FA_MODE_ACCOUNTER, 25, 10_000_000, fa.FA_GEN_UNIFORM, 1 << 26),
    "kmap_uniform": (fa.FA_MODE_KERNEL_MAP, 24, 10_000_000, fa.FA_GEN_UNIFORM, 1 << 26),
}
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def slot_hash(keys):
    """fmix64(key_premix(key)) of (n, 40) uint8 keys (DESIGN.md §4), vectorised."""
    with np.errstate(over="ignore"):
        w = np.ascontiguousarray(keys).view("<u8").reshape(-1, 5).copy()
        w[:, 4] &= np.uint64(0x00FFFFFFFFFFFFFF)
        h = np.full(len(w), 0x243F6A8885A308D3, np.uint64)
        for i, (p, s) in enumerate(((0x9E3779B97F4A7C15, 32), (0xC2B2AE3D27D4EB4F, 29), (0x9E3779B97F4A7C15, 32),
                                    (0xC2B2AE3D27D4EB4F, 29), (0x9E3779B97F4A7C15, 32))):
            h = (h ^ w[:, i]) * np.uint64(p)
            h ^= h >> np.uint64(s)
        h ^= h >> np.uint64(33); h *= np.uint64(0xFF51AFD7ED558CCD)
        h ^= h >> np.uint64(33); h *= np.uint64(0xC4CEB9FE1A85EC53)
        h ^= h >> np.uint64(33)
    return h


def select_passes(m, lo, k, slots):
    """The digit passes of the radix select for the top k of composites (m, lo = ~hash) -> list of per-pass dicts."""
    n = min(k, len(m))
    cap = 1024
    while cap < n + 4096:
        cap <<= 1
    bits = int(m.max()).bit_length() if len(m) else 0
    pos = 64 + 8 * ((bits + 7) // 8)
    pm = plo = 0
    above, k_rem, n_cand = 0, n, len(m)
    out = []
    cand = np.ones(len(m), bool)
    while above + n_cand > cap and pos > 0:
        p = pos - 8
        hashed = int(cand.sum()) if p < 64 else 0
        d = ((m[cand] >> np.uint64(p - 64)) if p >= 64 else (lo[cand] >> np.uint64(p))) & np.uint64(255)
        hist = np.bincount(d.astype(np.int64), minlength=256)
        cum, b = 0, 255
        while b > 0 and cum + hist[b] < k_rem:
            cum += int(hist[b]); b -= 1
        above += cum; k_rem -= cum; n_cand = int(hist[b])
        if p >= 64:
            pm |= b << (p - 64)
        else:
            plo |= b << p
        pos = p
        sel = np.zeros(len(m), bool)
        sel[np.nonzero(cand)[0][d == np.uint64(b)]] = True
        cand = sel
        out.append({"digit_low_bit": p, "candidates_after": n_cand, "hashed_flows": hashed,
                    "bytes_model": slots // 8 + 32 * len(m) + 64 * hashed})
    return out


class Blocks:
    """A records block for k rows, in device memory (torch) or pinned host memory."""

    def __init__(self, k, device):
        import torch
        self.device = device
        if device:
            self.t = torch.empty(k * 144, dtype=torch.uint8, device="cuda"); self.ptr = self.t.data_ptr()
        else:
            p = C.c_void_p(); check(lib().fa_host_alloc(k * 144, C.byref(p))); self.ptr = p.value

    def close(self):
        if not self.device:
            lib().fa_host_free(C.c_void_p(self.ptr))


def fill(eng, gp, n, chunk, buf):
    for first in range(0, n, chunk):
        eng.gen_records(gp, first, chunk, buf.data_ptr())
        check_rc = eng.ingest(buf.data_ptr(), chunk)
        assert check_rc[0] == fa.FA_OK, check_rc
    eng.sync()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated: " + ", ".join(SHAPES))
    ap.add_argument("--ks", default="100,10000,1000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=1 << 24, help="records per generated and ingested chunk")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("top_flows_bench.py: no CUDA device (this measurement has no CPU path)")
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit({"tool": "top_flows_bench", **card(), "reps": a.reps})
    ks = [int(x) for x in a.ks.split(",")]
    buf = torch.empty(a.chunk * 144, dtype=torch.uint8, device="cuda")
    for name in a.shapes.split(","):
        mode, slots_log2, keys, dist, n_recs = SHAPES[name]
        max_entries = 3 << (slots_log2 - 2)
        gp = fa.GenParams(seed=7, n_keys=keys, dist=dist, zipf_s_milli=1100, t0_ns=1_000_000, varying_desc=0)
        with fa.FlowAggEngine(max_entries, mode=mode, max_batch=a.chunk) as eng:
            fill(eng, gp, n_recs, a.chunk, buf)
            live = eng.live_flows()
            emit({"shape": name, "slots": 1 << slots_log2, "live_flows": live})
            for by in ("bytes", "packets"):
                metric = fa.FA_TOP_BYTES if by == "bytes" else fa.FA_TOP_PACKETS
                for k in ks:
                    for device in (True, False):
                        blk = Blocks(k, device)
                        o = EvictOut(records=blk.ptr)
                        got = C.c_size_t(0)
                        times = []
                        for r in range(a.reps + 1):
                            t0 = time.perf_counter()
                            check(lib().fa_top_flows(eng._h, metric, k, C.byref(o), C.byref(got)))
                            if r:
                                times.append(time.perf_counter() - t0)
                        blk.close()
                        emit({"shape": name, "by": by, "k": k, "out": "device" if device else "pinned_host", "rows": got.value,
                              "ms_median": round(1e3 * float(np.median(times)), 3), "ms_min": round(1e3 * min(times), 3)})
            # yardstick: fa_evict_ex of the same table into device memory (one untimed eviction + refill first)
            out = torch.empty(live * 144, dtype=torch.uint8, device="cuda")
            o = EvictOut(records=out.data_ptr())
            got = C.c_size_t(0)
            check(lib().fa_evict_ex(eng._h, C.byref(o), live, C.byref(got)))
            fill(eng, gp, n_recs, a.chunk, buf)
            t0 = time.perf_counter()
            check(lib().fa_evict_ex(eng._h, C.byref(o), live, C.byref(got)))
            ev_ms = 1e3 * (time.perf_counter() - t0)
            emit({"shape": name, "evict_ex_device_ms": round(ev_ms, 3), "flows": got.value})
            recs = out[: got.value * 144].cpu().numpy().reshape(-1, 144)
            del out
            m_all = {"bytes": recs[:, 56:64].copy().view("<u8").reshape(-1), "packets": recs[:, 64:68].copy().view("<u4").reshape(-1).astype(np.uint64)}
            lo = ~slot_hash(recs[:, :40]) & M64
            for by, m in m_all.items():
                for k in ks:
                    emit({"shape": name, "by": by, "k": k, "passes": select_passes(m, lo, k, 1 << slots_log2)})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
