#!/usr/bin/env python
"""What share of a Zipf stream does K1's hot-flow cache absorb, per lookup / replacement policy?  (No GPU.)

Replays the zipf10m stream (oracle generator, seed 2) through a model of one CTA of `aggregate_kernel`: 4 teams, each
with its own sequence of 256-record tiles (tile = blockIdx * 4 + team + it * 4 * grid), processed round-robin, 62 tiles
per team and launch (2^23-record launches on 132 SMs), the cache empty at the start of every launch.  Per tile: every
record looks the cache up (state as the previous tiles left it); the records that miss elect one representative per
key; then the representatives with enough duplicates try to install.  Printed per policy: the share of records that
hit the cache, and the share that become representatives (= probe the flow table).

Policies
  none     cache off (`opt & 2`): the representative share of the tile election alone
  ideal    the 96 most frequent keys, resident from the first record on
  direct   64 direct-mapped entries (hash >> 26) + 32 second-chance ((hash >> 21) & 31), never replaced
  SxW      S sets of W ways, free ways filled first come first served, never replaced
  SxW/N    the same + a decision point every N tiles per team: a queued candidate (at most 32 between two decision
           points, its records summed over the tiles it was a candidate in) displaces the way of its set with the
           fewest hits since the last decision point if its own record count beats that
The model leaves out what does not move these shares: timestamp windows, the overlap of the teams inside a tile time,
and the descriptor compare.

  python tools/hot_cache_sim.py [--ctas 4] [--launches 2] [--mindups 1 2 3]
"""
import argparse
import os
import sys
from collections import Counter

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as O  # noqa: E402

TILE, TEAMS, GRID, LAUNCH = 256, 4, 132, 1 << 23
ENTRIES, QUEUE = 96, 32


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


def cta_tiles(gen, cta, launch):
    """The 32-bit slot hashes of the tiles one CTA folds in one launch, in the model's order (round-robin over teams)."""
    per_team = LAUNCH // TILE // (GRID * TEAMS)
    out = []
    for it in range(per_team):
        for team in range(TEAMS):
            tile = cta * TEAMS + team + it * GRID * TEAMS
            r = gen.records(launch * LAUNCH + tile * TILE, TILE)
            out.append((slot_hash(r[:, :40]) & np.uint64(0xFFFFFFFF)).astype(np.int64).tolist())
    return out


class Direct:
    def __init__(self):
        self.e = [None] * ENTRIES

    def _second(self, h):
        return 64 + ((h >> 21) & 31)

    def hit(self, h):
        return self.e[h >> 26] == h or self.e[self._second(h)] == h

    def install(self, h, n):
        i = h >> 26
        if self.e[i] is not None and self.e[i] != h:
            i = self._second(h)
        if self.e[i] is None:
            self.e[i] = h

    def decide(self):
        pass


class SetAssoc:
    def __init__(self, sets, ways, replace):
        self.sets, self.ways, self.replace = sets, ways, replace
        self.e = [[None] * ways for _ in range(sets)]
        self.hits = {}                                   # resident hash -> hits since the last decision point
        self.queue = {}                                  # candidate hash -> records seen while a candidate
        self.replaced = 0

    def _set(self, h):
        return self.e[((h >> 16) * self.sets) >> 16]

    def hit(self, h):
        if h in self.hits:
            self.hits[h] += 1
            return True
        return False

    def install(self, h, n):
        if h in self.hits:
            return
        s = self._set(h)
        for w in range(self.ways):
            if s[w] is None:
                s[w] = h; self.hits[h] = 0
                return
        if self.replace and (h in self.queue or len(self.queue) < QUEUE):
            self.queue[h] = self.queue.get(h, 0) + n

    def decide(self):
        for h, n in sorted(self.queue.items(), key=lambda kv: -kv[1]):
            s = self._set(h)
            w = min(range(self.ways), key=lambda i: self.hits[s[i]])
            if n > self.hits[s[w]]:
                del self.hits[s[w]]
                s[w] = h; self.hits[h] = n               # the newcomer defends its way with what got it in
                self.replaced += 1
        self.queue.clear()
        for h in self.hits:
            self.hits[h] = 0


class Ideal:
    def __init__(self, top):
        self.top = top

    def hit(self, h):
        return h in self.top

    def install(self, h, n):
        pass

    def decide(self):
        pass


def replay(tiles, cache, mindups, every):
    hits = reps = 0
    for k, tile in enumerate(tiles):
        miss = [h for h in tile if not (cache and cache.hit(h))]
        hits += len(tile) - len(miss)
        c = Counter(miss)
        reps += len(c)
        if cache:
            for h, n in c.items():
                if n - 1 >= mindups:
                    cache.install(h, n)
            if every and (k + 1) % (every * TEAMS) == 0:
                cache.decide()
    return hits, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, default=4)
    ap.add_argument("--launches", type=int, default=2)
    ap.add_argument("--mindups", type=int, nargs="+", default=[1, 2, 3])
    ap.add_argument("--n-keys", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=2)
    args = ap.parse_args()
    gen = O.Gen(args.seed, args.n_keys, dist=1, zipf_s_milli=1100)
    top = set((slot_hash(np.stack([gen.key(r) for r in range(ENTRIES)])) & np.uint64(0xFFFFFFFF)).astype(np.int64).tolist())
    runs = [cta_tiles(gen, c * (GRID // args.ctas), l) for c in range(args.ctas) for l in range(args.launches)]
    total = sum(len(t) for tiles in runs for t in tiles)
    policies = [("none", lambda: None, 0), ("ideal", lambda: Ideal(top), 0), ("direct", Direct, 0)]
    for sets, ways in ((48, 2), (24, 4), (12, 8), (1, 96)):
        policies.append((f"{sets}x{ways}", lambda s=sets, w=ways: SetAssoc(s, w, False), 0))
        for every in (4, 8, 16):
            policies.append((f"{sets}x{ways}/{every}", lambda s=sets, w=ways: SetAssoc(s, w, True), every))
    print(f"{total} records: {args.ctas} CTAs x {args.launches} launches x {len(runs[0])} tiles of {TILE}")
    print(f"{'policy':12s} {'mindups':>7s} {'cache hits':>10s} {'representatives':>15s} {'replacements / launch':>21s}")
    for name, make, every in policies:
        for md in (args.mindups if name not in ("none", "ideal") else [0]):
            hits = reps = repl = 0
            for tiles in runs:
                cache = make()
                h, r = replay(tiles, cache, md, every)
                hits += h; reps += r; repl += getattr(cache, "replaced", 0)
            print(f"{name:12s} {md:7d} {hits / total:10.4f} {reps / total:15.4f} {repl / len(runs):21.1f}")


if __name__ == "__main__":
    main()
