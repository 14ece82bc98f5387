"""K7 (fa_ingest_dns_packets / fa_purge_stale_dns, csrc/dnscorr.cu) with colliding dns_flow_ids, uptime-scale clocks
and purge edges, bit for bit against the sequential restatement (O.DnsCorrelator + O.FlowMap).

tests/test_dns_correlate.py streams well-spread keys with small, increasing timestamps.  Here the device's dns_flows
table is attacked the way tests/test_adversarial_parity.py attacks the flow table: its 40-byte dns_flow_id image
(src 16 | dst 16 | sport 2 | dport 2 | id 2 | protocol 1 | 0, the device's DnsPkt.key) is hashed by key_premix and
fmix64 exactly like a flow key, so the same solver builds keys with a chosen premix or home slot.  Families:
  full        one identical 64-bit premix (one home slot in any table);
  chain_last  one home slot at the last slot, so that probes wrap to slot 0;
  chain_mid   one home slot in the middle of the table;
  same_tuple  one address pair and port pair with many DNS ids and both protocols, homes in a narrow window, so that
              walks cross entries that differ only in the key's last word.
Every packet creates an entry (orphan responses and answered queries too) and entries leave only at a rebuild, so one
home slot can carry a run far longer than the pending queries: the probe-limit scenario walks more than 4,096 occupied
slots from one home with the map far from full.

Colliding keys get distinct addresses, so most flows carry exactly one DNS sample and the comparison of the folded
flows is a comparison of the samples themselves (asserted per scenario).  tests/test_zz_gpu_dns_adversarial.py runs the
same scenarios on an H100."""
import ctypes
import functools

import numpy as np
import pytest

import oracle_lib as O
from test_adversarial_parity import UPTIME_NS, DevBuf, fmix64, key_with_premix, key_with_slot_hash, premix
from test_dns_correlate import QR, compare_dns, dns_stream, pkt

pytestmark = pytest.mark.timeout(900)

DNS_ROUNDS = 6                  # kDnsRounds: round kernels per chunk, the single-thread tail takes the rest
PROBE_RUN = 4_096               # the walk length the table once gave up at
PROBE_HOME = (1 << 14) - 1      # the probe-limit pool's home: the last slot of a 16,384-slot table, mid-table in larger ones


# ---------------------------------------------------------------------------------------------------- keys and packets
def dns_slots(max_entries):
    """fa_ingest_dns_packets' table size: a power of two, at least 64 and at least 4 x max_entries."""
    slots = 64
    while slots < 4 * max_entries:
        slots <<= 1
    return slots


def dns_id(key):
    return int(key[36]) | int(key[37]) << 8


def dns_key(make):
    """A key from `make()` (a premix or slot-hash solver) whose DNS id is not 0."""
    while True:
        k = make()
        if dns_id(k):
            return k


def same_tuple_keys(rng, slots, n, home):
    """n keys of one address pair and port pair, DNS ids and protocols (17 and 6, both present) chosen so that the
    homes fall in a window of slots starting at `home`; the window grows with the table to keep the search short."""
    mask, window = slots - 1, max(64, slots >> 8)
    head = bytes(10) + b"\xff\xff" + rng.bytes(4) + bytes(10) + b"\xff\xff" + rng.bytes(4) + rng.bytes(4)
    out, seen = [], set()
    while len(out) < n:
        i, proto = int(rng.integers(1, 1 << 16)), (17, 6)[len(out) % 2]
        k = np.frombuffer(head + i.to_bytes(2, "little") + bytes([proto, 0]), dtype=np.uint8)
        if (fmix64(premix(k)) - home) & mask < window and (i, proto) not in seen:
            seen.add((i, proto))
            out.append(k)
    return out


def dns_families(seed, slots, n_full=24, n_chain=160, n_mid=80, n_tuple=32):
    """The four families (name -> (m, 40) uint8 dns_flow_id images) for a table of `slots` slots."""
    rng = np.random.default_rng(seed)
    r64 = lambda: int(rng.integers(0, 1 << 62)) << 2 | int(rng.integers(0, 4))   # noqa: E731
    mask, mid = slots - 1, (slots // 2 + 17) & (slots - 1)
    h = r64()
    fam = {"full": [dns_key(lambda: key_with_premix(h, rng)) for _ in range(n_full)]}
    fam["chain_last"] = [dns_key(lambda: key_with_slot_hash((r64() & ~mask) | mask, rng)) for _ in range(n_chain)]
    fam["chain_mid"] = [dns_key(lambda: key_with_slot_hash((r64() & ~mask) | mid, rng)) for _ in range(n_mid)]
    fam["same_tuple"] = same_tuple_keys(rng, slots, n_tuple, mid)
    return {k: np.stack(v) for k, v in fam.items()}


@functools.lru_cache(maxsize=None)
def probe_pool(n=4_400):
    """n keys whose slot hash is PROBE_HOME modulo 2^22, so one home slot in every table up to the default one (2^22
    slots).  About 7 ms per key: built once per session."""
    rng = np.random.default_rng(4096)
    keys = np.stack([dns_key(lambda: key_with_slot_hash((int(rng.integers(0, 1 << 42)) << 22) | PROBE_HOME, rng))
                     for _ in range(n)])
    keys.setflags(write=False)
    return keys


def random_keys(rng, n):
    """Well-spread keys (no hash targeting) for a large background: v4-mapped addresses, DNS ids 1..65535, UDP or TCP."""
    k = np.zeros((n, 40), dtype=np.uint8)
    k[:, 10:12] = k[:, 26:28] = 0xFF
    k[:, 12:16] = rng.integers(0, 256, (n, 4)); k[:, 28:32] = rng.integers(0, 256, (n, 4))
    k[:, 32:34] = rng.integers(0, 256, (n, 2)); k[:, 34:36] = rng.integers(0, 256, (n, 2))
    ids = rng.integers(1, 1 << 16, n).astype("<u2")
    k[:, 36:38] = ids.view(np.uint8).reshape(n, 2)
    k[:, 38] = rng.choice(np.array([17, 6], np.uint8), n)
    return k


def dns_packets(keys, resp, ts=0, tag=None):
    """The packets of dns_flow_ids `keys`: the query (src -> dst) or, where `resp`, the response with the tuple reversed,
    as pkt() of test_dns_correlate builds them.  `tag` (one int per packet, default the row) varies the QNAME and the
    response's RCODE bits so that samples of different packets differ."""
    keys = np.asarray(keys, dtype=np.uint8).reshape(-1, 40)
    m = len(keys)
    resp = np.broadcast_to(np.asarray(resp, bool), m)
    tag = np.arange(m) if tag is None else np.asarray(tag)
    rv = resp[:, None]
    ident = np.zeros((m, 40), dtype=np.uint8)
    ident[:, 0:16] = np.where(rv, keys[:, 16:32], keys[:, 0:16])
    ident[:, 16:32] = np.where(rv, keys[:, 0:16], keys[:, 16:32])
    ident[:, 32:34] = np.where(rv, keys[:, 34:36], keys[:, 32:34])
    ident[:, 34:36] = np.where(rv, keys[:, 32:34], keys[:, 34:36])
    ident[:, 36] = keys[:, 38]
    r = np.zeros(m, dtype=O.DNSREC_DTYPE)
    r["id"] = ident
    d = r["dns"]
    d["start"] = 7; d["latency"] = 12345; d["errno"] = 99              # ignored on input
    d["end"] = ts
    d["id"] = np.ascontiguousarray(keys[:, 36:38]).view("<u2").reshape(-1)
    d["flags"] = np.where(resp, QR | 0x0180 | (tag & 0xF), 0x0100)
    d["eth"] = 0x0800
    name = np.zeros((m, 32), dtype=np.uint8)
    name[:, 0] = 4
    for j in range(4):
        name[:, 1 + j] = 97 + (tag // 26 ** j) % 26
    d["name"] = name
    d["pad"] = 0xEE
    r["dns"] = d
    return r


def set_times(pkts, ts):
    d = pkts["dns"]
    d["end"] = ts
    pkts["dns"] = d


# ---------------------------------------------------------------------------------------------------- streams
def scripts(rng, n, answered=0.6, orphan=0.2, dup=0.08):
    """One transaction per key as a string of 'q' (query) and 'r' (response): answered (qr), now and then with a
    repeated query (qqr) or a duplicate response (qrr); a response nobody asked for (r); a query nobody answers (q)."""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < answered:
            out.append("q" + "q" * (rng.random() < dup) + "r" + "r" * (rng.random() < dup))
        else:
            out.append("r" if u < answered + orphan else "q")
    return out


def interleave(rng, keys, script, background=None):
    """A uniformly random merge of the keys' scripts and of a background packet array, each kept in its own order."""
    lens = np.array([len(s) for s in script])
    ev_key = np.repeat(np.arange(len(script)), lens)
    ev_resp = np.array([c == "r" for s in script for c in s], dtype=bool)
    n_bg = 0 if background is None else len(background)
    pos = rng.permutation(len(ev_key) + n_bg)
    p = pos[: len(ev_key)]
    p = p[np.lexsort((p, ev_key))]                 # the positions of one key's events in script order
    out = np.zeros(len(pos), dtype=O.DNSREC_DTYPE)
    out[p] = dns_packets(keys[ev_key], ev_resp, tag=ev_key)
    if n_bg:
        out[np.sort(pos[len(ev_key):])] = background
    return out


def monotone_clock(rng, n, t0=1_000):
    return (t0 + np.cumsum(rng.integers(1, 50, n))).astype(np.uint64)


def uptime_clock(rng, n, per_cpu=8, chunk=24, zero_frac=0.03):
    """Uptime-scale packet times (~1.7e15 ns) from `per_cpu` CPUs whose clocks are skewed by up to 2^34 ns, merged in
    chunks (the order of uptime_times in test_adversarial_parity): a response stamped on another CPU than its query can
    come before it, and its latency wraps mod 2^64.  A few times are 0."""
    step = (1 << 32) // 160
    base = UPTIME_NS + np.arange(n, dtype=np.uint64) * np.uint64(step)
    skew = rng.integers(0, 1 << 34, per_cpu).astype(np.uint64)
    ts = base + skew[(np.arange(n) // chunk) % per_cpu] + rng.integers(0, 1 << 20, n).astype(np.uint64)
    ts[rng.random(n) < zero_frac] = 0
    return ts


def batches(rng, pkts, parts):
    cuts = np.sort(rng.choice(np.arange(1, len(pkts)), parts - 1, replace=False))
    return np.split(pkts, cuts)


def colliding_stream(seed, fam, n_bg, clock=monotone_clock, bg_clients=4, extra=None):
    """Every family's keys as random transactions merged into a dns_stream background (and `extra` packets, e.g. a
    large well-spread background), stamped by `clock`."""
    rng = np.random.default_rng(seed)
    keys = np.concatenate(list(fam.values()))
    bg = [dns_stream(seed, n_bg, n_clients=bg_clients, n_ids=3)] if n_bg else []
    bg = np.concatenate(bg + ([] if extra is None else [extra]))
    s = interleave(rng, keys, scripts(rng, len(keys)), bg)
    set_times(s, clock(rng, len(s)))
    return s


def spread_transactions(seed, n_keys):
    """Transactions of n_keys well-spread keys (a large background; times are set by the stream's clock)."""
    rng = np.random.default_rng(seed)
    return interleave(rng, random_keys(rng, n_keys), scripts(rng, n_keys))


def one_sample_share(steps, max_entries):
    """Of the flows that get DNS samples, the share that gets exactly one (per the restatement)."""
    corr = O.DnsCorrelator(max_entries)
    ids = []
    for b in steps:
        if isinstance(b, tuple):
            corr.purge(*b[1:])
        else:
            ids.append(corr.packets(b)[:, :40])
    ids = np.concatenate(ids)
    _, counts = np.unique(np.ascontiguousarray(ids).view(np.dtype((np.void, 40))).reshape(-1), return_counts=True)
    return float((counts == 1).mean())


def latencies(steps, max_entries):
    """(latency, errno) of every sample the restatement makes of a response."""
    corr = O.DnsCorrelator(max_entries)
    out = []
    for b in steps:
        if isinstance(b, tuple):
            corr.purge(*b[1:])
        else:
            s = corr.packets(b).view(O.DNSREC_DTYPE).reshape(-1)
            out.append(s[(s["dns"]["flags"] & QR) != 0]["dns"][["latency", "errno"]])
    return np.concatenate(out)


def run_case(steps, max_entries=None, flows=1 << 12, max_batch=4_096, ingest=None):
    """The engine and the restatement side by side, as run_case of test_dns_correlate, with purges as steps.  Each
    step is a packet array (one fa_ingest_dns_packets call, made by `ingest(eng, batch)` when given) or
    ("purge", now, timeout).  The pending, map-full and purged counters must match after every call, the evicted flows
    at the end."""
    import netobserv_ebpf_agent_b200 as fa
    corr = O.DnsCorrelator(max_entries or (1 << 20))
    om = O.FlowMap()
    full = purged = 0
    with fa.FlowAggEngine(flows, flags=fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_RTT, max_batch=max_batch) as eng:
        for k, b in enumerate(steps):
            if isinstance(b, tuple):
                eng.purge_stale_dns(b[1], b[2])
                purged += corr.purge(b[1], b[2])
            else:
                (ingest or fa.FlowAggEngine.ingest_dns_packets)(eng, b)
                s = corr.packets(b)
                om.fold_dns(s)
                full += int((s.view(O.DNSREC_DTYPE).reshape(-1)["dns"]["errno"] == 249).sum())
            st = eng.stats()
            got, want = (st["dns_queries_pending"], st["dns_map_full"], st["dns_queries_purged"]), (corr.pending(), full, purged)
            assert got == want, f"after call {k}: (pending, map full, purged) engine {got}, restatement {want}"
        compare_dns(eng, om)
    return st


def device_ingest(emul):
    """fa_ingest_dns_packets from device memory: a CUDA tensor on the GPU, fa_device_alloc memory on the emulation."""
    from netobserv_ebpf_agent_b200._lib import check, lib

    def ingest(eng, b):
        buf = DevBuf(eng, b.nbytes, emul)
        buf.write(b)
        check(lib().fa_ingest_dns_packets(eng._h, ctypes.c_void_p(buf.ptr), len(b)))
        eng.sync()
        buf.free()
    return ingest


# ---------------------------------------------------------------------------------------------------- scenarios
def scenario_mixed(seed, slots, n_bg, parts, extra=None, **fam_kw):
    """1: colliding transactions of every family in a background, in `parts` calls."""
    fam = dns_families(seed, slots, **fam_kw)
    s = colliding_stream(seed, fam, n_bg, extra=extra)
    return batches(np.random.default_rng(seed + 1), s, parts)


def scenario_rebuilds(seed, max_entries, rounds=4, **fam_kw):
    """2: chain queries first, then traffic that forces rebuilds, then their responses.  The keys that ever see a query
    stay well below max_entries, so that no query meets a full map."""
    rng = np.random.default_rng(seed)
    slots = dns_slots(max_entries)
    fam = dns_families(seed, slots, **fam_kw)
    chain = np.concatenate([fam["chain_last"], fam["chain_mid"], fam["full"]])
    n_q = min(len(chain) // 2, max_entries // 3)
    asked, rest = chain[:n_q], np.array_split(chain[n_q:], rounds)
    bg_clients = max(2, min(8, max_entries // 24))
    steps = [dns_packets(asked, False)]
    for r in range(rounds):                                     # each round is at least half a table of packets
        orphans = dns_packets(rest[r], True)                    # absent entries on the chains, dropped by every rebuild
        bg = dns_stream(seed + r, max(slots // 2, 200), n_clients=bg_clients, n_ids=3)
        s = interleave(rng, fam["same_tuple"], scripts(rng, len(fam["same_tuple"])), np.concatenate([bg, orphans]))
        steps += batches(rng, s, 2)
    resp = dns_packets(asked, True)
    steps.append(np.concatenate([resp, dns_packets(asked[: n_q // 8], True)]))     # the second response of a few: ENOENT
    for i, b in enumerate(steps):
        set_times(b, monotone_clock(rng, len(b), t0=1_000 + i * 10_000_000))
    return steps, n_q


def scenario_hot(seed, slots, per_key=(8, 20), parts=3, n_bg=300):
    """3: a few colliding keys with more packets each per call than there are round kernels."""
    assert per_key[0] > DNS_ROUNDS
    rng = np.random.default_rng(seed)
    fam = dns_families(seed, slots, n_full=6, n_chain=4, n_mid=4, n_tuple=4)
    keys = np.concatenate([fam["full"], fam["chain_last"], fam["chain_mid"], fam["same_tuple"]])
    steps = []
    for p in range(parts):
        sc = ["".join(rng.choice(["q", "r"], int(rng.integers(*per_key)))) for _ in keys]
        bg = dns_stream(seed + p, n_bg, n_clients=6, n_ids=2)
        s = interleave(rng, keys, sc, bg)
        set_times(s, monotone_clock(rng, len(s), t0=1_000 + p * 1_000_000))
        steps.append(s)
    return steps


def scenario_probe_run(n_orphans=PROBE_RUN, n_queries=8, bg=None):
    """4: n_orphans responses nobody asked for, all of one home slot (PROBE_HOME), then queries of the same home: their
    walk passes every orphan's entry.  Then the responses (and a background, if given)."""
    pool = probe_pool()
    rng = np.random.default_rng(44)
    orphans = dns_packets(pool[:n_orphans], True)
    qk = pool[n_orphans:n_orphans + n_queries]
    q = dns_packets(qk, False)
    r = dns_packets(qk, True)
    steps = [orphans, q if bg is None else np.concatenate([q, bg]), r]
    for i, b in enumerate(steps):
        set_times(b, monotone_clock(rng, len(b), t0=1_000 + i * 1_000_000))
    return steps


def scenario_probe_rebuild(n_queries, filler):
    """4b: n_queries pending queries of one home slot (a run longer than PROBE_RUN), then the `filler` packets (at
    least half a table of them forces a rebuild that has to re-place the whole run), then the responses."""
    pool = probe_pool()
    rng = np.random.default_rng(45)
    qk = pool[:n_queries]
    steps = [dns_packets(qk, False), filler, dns_packets(qk, True)]
    for i, b in enumerate(steps):
        set_times(b, monotone_clock(rng, len(b), t0=1_000 + i * 1_000_000_000))
    return steps


def scenario_uptime(seed, slots, n_bg, parts, extra=None, **fam_kw):
    """5: the families on uptime-scale clocks with skewed CPUs and zero times."""
    fam = dns_families(seed, slots, **fam_kw)
    s = colliding_stream(seed, fam, n_bg, clock=uptime_clock, extra=extra)
    return batches(np.random.default_rng(seed + 1), s, parts)


T_NOW = UPTIME_NS + 10 ** 12
P63 = 1 << 63


def scenario_purge(seed, slots, per=4):
    """6: purge edges, every class `per` chain keys.  Responses to one key of a class after each purge show which
    entries went; pending / purged counters are checked after every call.
      A  now - ts == timeout exactly       purged by (now, 5000)
      B  now - ts == timeout - 1           kept by (now, 5000), purged by timeout 0
      C  ts in the future (1 s)            kept by (now, 5000) and by timeout 0
      D  ts == now                         kept by (now, 5000), purged by timeout 0
      E  ts == 0                           purged by (now, 5000)
      F  now below ts by more than 2^63    now - ts = 2^63 - 100 as a signed number: purged by (now, 5000)
      G  ts 2^62 ahead                     now - ts negative: kept by both, gone only with a negative timeout
    A is queried again after its purge (the insert must succeed and the response must see the new timestamp); the last
    purge's timeout has bit 63 set, so it is negative and every entry goes, future ones included."""
    fam = dns_families(seed, slots, n_full=8, n_chain=40, n_mid=40, n_tuple=8)
    keys = np.concatenate([fam["chain_last"], fam["chain_mid"], fam["full"]])
    ts_of = {"A": T_NOW - 5_000, "B": T_NOW - 4_999, "C": T_NOW + 10 ** 9, "D": T_NOW, "E": 0,
             "F": (T_NOW + P63 + 100) % (1 << 64), "G": T_NOW + (1 << 62)}
    cls = {c: keys[i * per:(i + 1) * per] for i, c in enumerate(ts_of)}

    def q(c, ts=None):
        return dns_packets(cls[c], False, ts=ts_of[c] if ts is None else ts)

    def r(c, i, ts):
        return dns_packets(cls[c][i:i + 1], True, ts=ts)

    orphans = dns_packets(keys[len(ts_of) * per:], True, ts=T_NOW - 10 ** 6)       # absent entries on the same chains
    tuples = dns_packets(fam["same_tuple"], False, ts=T_NOW - 1)
    steps = [("purge", T_NOW, 5_000),                                             # nothing correlated yet: a no-op
             np.concatenate([orphans[: len(orphans) // 2]] + [q(c) for c in ts_of] + [tuples, orphans[len(orphans) // 2:]]),
             ("purge", T_NOW, 5_000),
             np.concatenate([r(c, 0, T_NOW + 7) for c in ts_of]),
             ("purge", T_NOW, 0),
             np.concatenate([r(c, 1, T_NOW + 9) for c in ts_of] + [q("A", T_NOW + 11)]),  # A, purged, inserts again
             np.concatenate([r("A", 2, T_NOW + 13), q("A", T_NOW + 15)]),     # A[2]: latency 2, then new; the rest: EEXIST
             ("purge", T_NOW + 20, P63 | 7),
             np.concatenate([r(c, 2, T_NOW + 30) for c in ts_of] + [q("B", T_NOW + 31), r("B", 3, T_NOW + 40)]),
             ("purge", 0, 0),
             np.concatenate([r(c, 3, T_NOW + 50) for c in ts_of])]
    return steps


# ---------------------------------------------------------------------------------------------------- CPU: the builders
@pytest.mark.parametrize("slots", [256, 4_096, 1 << 22])
def test_dns_families_hash_as_built(slots):
    """Each family is what its name says, by the oracle's own premix and slot hash of the 40-byte image."""
    fam = dns_families(3, slots, n_chain=30, n_mid=20, n_tuple=24)
    f = O.lib()
    mask = slots - 1
    for name, keys in fam.items():
        assert len(np.unique(keys, axis=0)) == len(keys), name
        assert not keys[:, 39].any() and all(dns_id(k) for k in keys), name
        pm = [f.oracle_key_premix(O._p(np.ascontiguousarray(k))) for k in keys]
        sh = [f.oracle_slot_hash(O._p(np.ascontiguousarray(k))) for k in keys]
        assert pm == [premix(k) for k in keys] and sh == [fmix64(x) for x in pm], name
        homes = {x & mask for x in sh}
        if name == "full":
            assert len(set(pm)) == 1
        else:
            assert len(set(pm)) == len(keys), name
        if name == "chain_last":
            assert homes == {mask}
        if name == "chain_mid":
            assert homes == {(slots // 2 + 17) & mask}
        if name == "same_tuple":
            assert len({bytes(k[:36]) for k in keys}) == 1 and set(keys[:, 38].tolist()) == {6, 17}
            mid = (slots // 2 + 17) & mask
            assert all((h - mid) & mask < max(64, slots >> 8) for h in homes)
        else:                                                   # distinct addresses: one flow per packet direction
            assert len({bytes(k[:32]) for k in keys}) == len(keys), name


def test_probe_pool_is_one_home_in_every_table():
    pool = probe_pool()
    f = O.lib()
    sh = {f.oracle_slot_hash(O._p(np.ascontiguousarray(k))) & ((1 << 22) - 1) for k in pool}
    assert sh == {PROBE_HOME} and len(np.unique(pool, axis=0)) == len(pool) > PROBE_RUN + 100
    assert all(dns_id(k) for k in pool) and not pool[:, 39].any()


def test_packets_are_what_pkt_builds():
    """The vectorised builder against test_dns_correlate's pkt(), both directions; and the device's key of the
    response (the reversed tuple) is the key itself."""
    fam = dns_families(5, 1024, n_full=2, n_chain=2, n_mid=2, n_tuple=2)
    keys = np.concatenate(list(fam.values()))
    for i, k in enumerate(keys):
        src, dst, sp, dp = bytes(k[:16]), bytes(k[16:32]), int(k[32]) | int(k[33]) << 8, int(k[34]) | int(k[35]) << 8
        name = bytes([4] + [97 + (i // 26 ** j) % 26 for j in range(4)])
        want_q = pkt(src, dst, sp, dp, 1_000 + i, dns_id(k), 0x0100, proto=int(k[38]), name=name)
        want_r = pkt(dst, src, dp, sp, 2_000 + i, dns_id(k), QR | 0x0180 | (i & 0xF), proto=int(k[38]), name=name)
        assert dns_packets(k, False, 1_000 + i, tag=[i]).tobytes() == want_q.tobytes()
        assert dns_packets(k, True, 2_000 + i, tag=[i]).tobytes() == want_r.tobytes()
    # the restatement pairs each response with its query: every latency is the time difference
    s = O.DnsCorrelator().packets(np.concatenate([dns_packets(keys, False, 100), dns_packets(keys, True, 350)]))
    d = s.view(O.DNSREC_DTYPE).reshape(-1)["dns"]
    assert len(d) == len(keys) and (d["latency"] == 250).all() and (d["errno"] == 0).all()


def test_streams_reach_the_far_side():
    """The uptime stream has wrapped latencies and zero times, the rebuild scenario forces rebuilds, the purge
    scenario's edges purge what they say."""
    steps = scenario_uptime(60, 4_096, 1_500, 3)
    lat = latencies(steps, 1 << 20)
    ok = lat[lat["errno"] == 0]["latency"]
    assert (ok >= np.uint64(P63)).sum() > 20 and (ok < np.uint64(1 << 40)).sum() > 20
    assert (np.concatenate(steps)["dns"]["end"] == 0).sum() > 20
    steps, n_q = scenario_rebuilds(61, 64, rounds=4)
    assert min(len(steps[1 + 2 * r]) + len(steps[2 + 2 * r]) for r in range(4)) >= dns_slots(64) // 2   # a rebuild per round
    corr = O.DnsCorrelator(1 << 20)
    gone = []
    for b in scenario_purge(62, 4_096):
        if isinstance(b, tuple):
            gone.append(corr.purge(*b[1:]))
        else:
            corr.packets(b)
    # nothing yet; A E F; B D and the 8 same_tuple queries; everything (C G, the re-queried A); B's new queries are future
    assert gone == [0, 12, 14, 8, 0] and corr.pending() == 3


# ---------------------------------------------------------------------------------------------------- CPU: engine emulation
def test_colliding_transactions_emul(engine_emul):
    """1: every family in a dns_stream background, calls split into 512-packet chunks."""
    steps = scenario_mixed(10, dns_slots(1 << 20), 1_500, 4)
    st = run_case(steps, flows=1 << 13, max_batch=512)
    assert st["dns_map_full"] == 0 and st["dns_ingested"] > 0
    assert one_sample_share(steps, 1 << 20) >= 0.8


@pytest.mark.parametrize("max_entries", [64, 1024])
def test_chains_across_rebuilds_emul(engine_emul, monkeypatch, max_entries):
    """2: pending chain queries survive every rebuild (their responses get latencies), answered and orphan entries do
    not (a second response is ENOENT; orphans keep being re-created)."""
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", str(max_entries))
    kw = dict(n_full=8, n_chain=60, n_mid=30, n_tuple=12) if max_entries == 64 else dict(n_chain=400, n_mid=200, n_tuple=48)
    steps, n_q = scenario_rebuilds(20 + max_entries, max_entries, **kw)
    st = run_case(steps, max_entries=max_entries, flows=1 << 14)
    assert st["dns_map_full"] == 0
    lat = latencies(steps, max_entries)[-len(steps[-1]):]
    assert (lat["errno"] == 0).sum() == n_q and (lat["errno"] == 2).sum() == n_q // 8
    assert one_sample_share(steps, max_entries) >= 0.8


@pytest.mark.parametrize("rounds", [None, "0"])
def test_hot_colliding_keys_emul(engine_emul, monkeypatch, rounds):
    """3: 8..20 packets per colliding key and call: the round kernels and the tail on neighbouring entries of one chain
    (FA_EMUL_DNS_ROUNDS=0: the tail alone)."""
    if rounds is not None:
        monkeypatch.setenv("FA_EMUL_DNS_ROUNDS", rounds)
    steps = scenario_hot(30, dns_slots(1 << 20))
    run_case(steps, flows=1 << 12)


def test_probe_run_longer_than_4096_emul(engine_emul, monkeypatch):
    """4: 4,096 orphan responses of one home slot (the last: the run wraps to slot 0) in a 16,384-slot table, then
    queries of that home with 8 of 4,096 entries pending: every query is inserted and its response gets a latency."""
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", "4096")
    assert dns_slots(4096) - 1 == PROBE_HOME
    steps = scenario_probe_run()
    st = run_case(steps, max_entries=4096, flows=1 << 13)
    assert st["dns_map_full"] == 0 and st["dns_queries_pending"] == 0
    lat = latencies(steps, 4096)
    assert (lat["errno"] == 0).sum() == 8
    assert one_sample_share(steps, 4096) >= 0.8


def test_rebuild_replaces_a_run_longer_than_4096_emul(engine_emul, monkeypatch):
    """4b: 4,200 pending queries of one home (a 32,768-slot table, mid-table), then enough packets to force a rebuild:
    the rebuild re-places the whole run and every response gets its latency."""
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", "8192")
    n_filler = dns_slots(8192) // 2 - 4_200 + 512
    steps = scenario_probe_rebuild(4_200, dns_stream(46, n_filler, n_clients=20, n_ids=3))
    assert sum(map(len, steps[:2])) > dns_slots(8192) // 2                # the responses come after a rebuild
    st = run_case(steps, max_entries=8192, flows=1 << 14)
    assert st["dns_map_full"] == 0
    lat = latencies(steps, 8192)[-4_200:]
    assert (lat["errno"] == 0).all()
    assert one_sample_share(steps, 8192) >= 0.8


@pytest.mark.parametrize("max_entries", [1024, None])
def test_uptime_clocks_emul(engine_emul, monkeypatch, max_entries):
    """5: uptime-scale, skewed, sometimes zero packet times: latencies that wrap mod 2^64, bit for bit."""
    if max_entries:
        monkeypatch.setenv("FA_DNS_MAX_ENTRIES", str(max_entries))
    me = max_entries or 1 << 20
    steps = scenario_uptime(50, dns_slots(me), 800, 3, n_chain=120, n_mid=60)
    st = run_case(steps, max_entries=me, flows=1 << 13, max_batch=1_024)
    assert st["dns_map_full"] == 0
    assert one_sample_share(steps, me) >= 0.8


@pytest.mark.parametrize("device", [False, True])
def test_purge_edges_emul(engine_emul, monkeypatch, device):
    """6: the signed compare of lookupAndDeleteDNSMap at its edges, on the engine, with chains in the table."""
    monkeypatch.setenv("FA_DNS_MAX_ENTRIES", "1024")
    steps = scenario_purge(70, dns_slots(1024))
    run_case(steps, max_entries=1024, flows=1 << 12, ingest=device_ingest(engine_emul) if device else None)
    assert one_sample_share(steps, 1024) >= 0.8
