"""K8 (fa_pb_encode) at its edges, byte for byte against the Python protobuf library (tests/pbflow_ref.py).

Every group runs on the engine emulation and, marked `gpu`, on the device:
  1. field and varint edges, one field varied per record (every varint at 0, 1, 2^7k - 1, 2^7k and its type's maximum;
     negative int32 and durations; open-enum directions; the `eth == 0x86DD` address rule; wrap prefixes of 1 and 2 bytes);
  2. clock edges (mono at, behind and ahead of mono_now, pre-1970 wall clocks, results past the int64 nanosecond range,
     a monotonic delta of exactly -2^63, whose Go negation wraps to itself);
  3. DNS names (no terminator, overrunning labels, compression pointers, reserved length bytes, empty names, UTF-8);
  4. the interface table (lookup rules, length clamps, observed-interface clamp, tables that grow and shrink);
  5. launch shape (CTAs past the 64 KB stage next to staged ones and one exactly at it, misaligned device output, NULL
     offsets / keys, host and device inputs mixed, FA_E_2BIG, n = 0);
  6. batches past 2^20 flows (more than 1024 scan blocks; on the emulation the scan kernels are driven directly);
  7. fa_evict_ex into device buffers straight into fa_pb_encode.

Rules asserted as they stand today:
  * a record whose dns_name, interface name or UDN is not valid UTF-8 is emitted as zero bytes (offsets[i] ==
    offsets[i + 1]) and gets no pbflow.Records entry with FA_PB_WRAP_ENTRIES; its Kafka key is still written;
  * a feature block is used only where both its pointer and its `present` bit are set: `present` NULL means no block,
    and a present bit whose block pointer is NULL means that block is absent;
  * name_len > 16 and udn_len > 64 are clamped to the field's size, nb_obs > 6 to 6;
  * now_unix_ns is unsigned; with it the wall clock cannot fall below -2^63 ns, and its lowest value (now 0, delta
    -2^63) is tested."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
import pbflow_ref as PB
from common import gen_host

NOW, MONO = 1_700_000_000_123_456_789, 5_000_000_000_000
AGENT4 = bytes(10) + b"\xff\xff" + bytes([10, 1, 2, 3])
AGENT6 = bytes(range(0x20, 0x30))
U64 = (1 << 64) - 1
E2BIG = -7


# ------------------------------------------------------------------------------------------------------ harness
class Backend:
    """One engine and its device memory: torch on the GPU, the emulation's own allocations on the CPU."""

    def __init__(self, gpu):
        import netobserv_ebpf_agent_b200 as fa
        from netobserv_ebpf_agent_b200._lib import lib
        self.gpu, self.lib = gpu, lib()
        self.eng = fa.FlowAggEngine(64)                      # fa_pb_encode uses none of its table
        self.h = self.eng._h
        self.bufs = []                                       # (base pointer, size, owner)

    def alloc(self, nbytes, fill=0):
        if self.gpu:
            import torch
            t = torch.full((max(nbytes, 1),), fill, dtype=torch.uint8, device="cuda")
            self.bufs.append((t.data_ptr(), nbytes, t))
            return t.data_ptr()
        p = C.c_void_p()
        assert self.lib.fa_device_alloc(self.h, max(nbytes, 1), C.byref(p)) == 0
        C.memset(p.value, fill, max(nbytes, 1))
        self.bufs.append((p.value, nbytes, None))
        return p.value

    def put(self, a):
        a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        p = self.alloc(a.size)
        if self.gpu:
            import torch
            self.bufs[-1][2].copy_(torch.from_numpy(a.copy()))
        else:
            C.memmove(p, a.ctypes.data, a.size)
        return p

    def get(self, p, nbytes):
        for base, size, t in self.bufs:
            if base <= p and p + nbytes <= base + max(size, 1):
                if t is None:
                    return np.frombuffer(C.string_at(p, nbytes), np.uint8).copy()
                return t[p - base:p - base + nbytes].cpu().numpy()
        raise AssertionError("not a buffer of this backend")

    def close(self):
        if not self.gpu:
            for base, _, _ in self.bufs:
                self.lib.fa_device_free(self.h, C.c_void_p(base))
        self.bufs.clear()
        self.eng.close()


@pytest.fixture(params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emul":
        request.getfixturevalue("engine_emul")
    b = Backend(request.param == "gpu")
    try:
        yield b
    finally:
        b.close()


def iface_rows(ifaces):
    """ifaces: (if_index, mac, name bytes, udn bytes[, name_len, udn_len]) -> fa_iface_name array (None: NULL table),
    and the rows as the checker sees them (lengths clamped to 16 / 64 like the kernel does)."""
    from netobserv_ebpf_agent_b200._lib import IfaceName
    if ifaces is None:
        return None, []
    rows = (IfaceName * max(len(ifaces), 1))()
    ref = []
    for i, t in enumerate(ifaces):
        idx, mac, name, udn = t[:4]
        nl, ul = (t[4], t[5]) if len(t) > 4 else (len(name), len(udn))
        rows[i].if_index = idx
        for b in range(6):
            rows[i].mac[b] = mac[b]
        rows[i].name_len, rows[i].udn_len = nl, ul
        C.memmove(C.addressof(rows[i]) + IfaceName.name.offset, name, min(len(name), 16))
        C.memmove(C.addressof(rows[i]) + IfaceName.udn.offset, udn, min(len(udn), 64))
        ref.append((idx, bytes(mac), bytes(name[:min(nl, 16)]), bytes(udn[:min(ul, 64)])))
    return rows, ref


def pb_params(now, mono, agent, agent_v4, rows, n_ifaces, wrap):
    from netobserv_ebpf_agent_b200._lib import IfaceName, PbParams
    p = PbParams(now_unix_ns=now, mono_now_ns=mono, agent_ip_is_v4=agent_v4, flags=1 if wrap else 0,
                 ifaces=C.cast(rows, C.POINTER(IfaceName)) if rows is not None else None, n_ifaces=n_ifaces)
    for i in range(16):
        p.agent_ip[i] = agent[i]
    return p


def as_u8(a, width):
    return None if a is None else np.ascontiguousarray(a).view(np.uint8).reshape(-1, width)


def encode(be, recs, dns=None, add=None, drops=None, present=None, *, now=NOW, mono=MONO, agent=AGENT4, agent_v4=1,
           ifaces=None, wrap=False, on_device=(), out_offset=None, offsets=True, keys=True, total=None):
    """fa_pb_encode into exactly `total` bytes (None: sized first through FA_E_2BIG).  on_device: names of the inputs
    ("recs", "dns", "add", "drops", "present") handed over in device memory; out_offset: write into device memory at
    that byte offset (else a host buffer).  -> (bytes, offsets or None, keys or None)."""
    recs, dns, add, drops = as_u8(recs, 144), as_u8(dns, 64), as_u8(add, 32), as_u8(drops, 32)
    n = len(recs)
    rows, _ = iface_rows(ifaces)
    p = pb_params(now, mono, agent, agent_v4, rows, len(ifaces or ()), wrap)
    ins = {"recs": recs, "dns": dns, "add": add, "drops": drops, "present": present}
    ptr = {k: (None if v is None else C.c_void_p(be.put(v)) if k in on_device else C.c_void_p(v.ctypes.data))
           for k, v in ins.items()}
    args = (be.h, ptr["recs"], ptr["dns"], ptr["add"], ptr["drops"], ptr["present"], n, C.byref(p))
    if total is None:
        need = C.c_size_t(0)
        rc = be.lib.fa_pb_encode(*args, None, 0, None, None, C.byref(need))
        assert rc == (E2BIG if need.value else 0), rc
        total = need.value
    offs = np.full(n + 1, 0xEE, np.uint64) if offsets else None
    kout = np.full((n, 32), 0xEE, np.uint8) if keys else None
    if out_offset is None:
        out = np.full(max(total, 1), 0xA5, np.uint8)
        dst = C.c_void_p(out.ctypes.data)
    else:
        base = be.alloc(total + out_offset + 16, 0xA5)
        dst = C.c_void_p(base + out_offset)
    got = C.c_size_t(0)
    rc = be.lib.fa_pb_encode(*args, dst, total, C.c_void_p(offs.ctypes.data) if offsets else None,
                             C.c_void_p(kout.ctypes.data) if keys else None, C.byref(got))
    assert rc == 0 and got.value == total, (rc, got.value, total, be.lib.fa_last_error())
    if out_offset is None:
        assert not total or (out[total:] == 0xA5).all()
        raw = out[:total].tobytes()
    else:
        whole = be.get(base, total + out_offset + 16)
        assert (whole[:out_offset] == 0xA5).all() and (whole[out_offset + total:] == 0xA5).all()   # nothing outside
        raw = whole[out_offset:out_offset + total].tobytes()
    return raw, offs, kout


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


def _i64(v):
    v &= U64
    return v - (1 << 64) if v >= 1 << 63 else v


def go_record(rec144, dns64, add32, now, mono, agent, agent_v4, ifaces, drop32):
    """pbflow_ref.flow_to_pb completed with what protobuf-go and time.Time do at the edges tested here -> the message,
    or None where proto.Marshal fails and the Kafka exporter drops the record:
      * dns_name, DupMapEntry.interface and .udn are `string` fields: a value that is not valid UTF-8 (utf8.ValidString,
        which Python's strict decoder agrees with) fails the marshal; valid names are their UTF-8 bytes as they are;
      * currentTime.Add(-Duration(monoNow - mono)) is exact (time.Time keeps seconds and nanoseconds apart) and Go's
        negation wraps (-Duration(MinInt64) == MinInt64), so the added duration is Duration(mono - monoNow).
    ifaces: (if_index, mac, name bytes, udn bytes) rows."""
    r = np.frombuffer(rec144, O.REC_DTYPE)[0]
    name = PB.dns_dotted(np.frombuffer(dns64, O.DNS_DTYPE)[0]["name"]) if dns64 is not None else b""
    lmac = r["dst_mac"] if int(r["direction"]) == 0 else r["src_mac"]
    used = [int(r["if_index"])] + [int(x) for x in r["obs_intf"][:min(int(r["nb_obs"]), 6)]]
    strings = [name] + [x for i in used for x in PB.iface_lookup(ifaces, i, lmac)]
    try:
        for x in strings:
            if isinstance(x, bytes):
                x.decode("utf-8")
    except UnicodeDecodeError:
        return None
    text = [(i, m, nm.decode("utf-8", "replace"), u.decode("utf-8", "replace")) for i, m, nm, u in ifaces]   # bad rows unused here
    pb = PB.flow_to_pb(rec144, dns64, add32, now, mono, agent, agent_v4, text, drop32)
    if name:
        pb.dns_name = name.decode("utf-8")
    for field, t in (("time_flow_start", r["start"]), ("time_flow_end", r["end"])):
        wall = int(now) + _i64(int(t) - int(mono))
        getattr(pb, field).seconds, getattr(pb, field).nanos = wall // 10**9, wall % 10**9
    return pb


def expected(recs, dns=None, add=None, drops=None, present=None, *, now=NOW, mono=MONO, agent=AGENT4, agent_v4=1,
             ifaces=None, wrap=False):
    """What fa_pb_encode must write for each flow: the protobuf library's bytes, b"" for a dropped record."""
    recs, dns, add, drops = as_u8(recs, 144), as_u8(dns, 64), as_u8(add, 32), as_u8(drops, 32)
    _, ref_ifaces = iface_rows(ifaces)
    out = []
    for i in range(len(recs)):
        pr = 0 if present is None else int(present[i])
        blk = lambda a, bit: a[i].tobytes() if a is not None and pr & bit else None   # noqa: E731
        m = go_record(recs[i].tobytes(), blk(dns, 1), blk(add, 2), now, mono, agent, bool(agent_v4), ref_ifaces,
                      blk(drops, 4))
        body = b"" if m is None else m.SerializeToString()
        out.append(b"\x0a" + varint(len(body)) + body if wrap and body else body)
    return out


def check(be, recs, dns=None, add=None, drops=None, present=None, **kw):
    """Encode on the backend, compare with the checker; -> the per-flow expected bytes."""
    enc_kw = {k: kw.pop(k) for k in ("on_device", "out_offset", "offsets", "keys") if k in kw}
    want = expected(recs, dns, add, drops, present, **kw)
    raw, offs, keys = encode(be, recs, dns, add, drops, present, **kw, **enc_kw, total=sum(len(w) for w in want))
    if raw != b"".join(want):
        starts = np.concatenate([[0], np.cumsum([len(w) for w in want])])
        for i, w in enumerate(want):                         # name the first flow that differs
            got = raw[starts[i]:starts[i] + len(w)]
            assert got == w, (i, got.hex(), w.hex())
        assert raw == b"".join(want)
    if offs is not None:
        assert np.array_equal(offs, np.concatenate([[0], np.cumsum([len(w) for w in want])]).astype(np.uint64))
    if keys is not None:
        r = as_u8(recs, 144)
        for i in range(len(r)):
            assert keys[i].tobytes() == PB.flow_key(r[i].tobytes()), i
    for i, w in enumerate(want):                              # every emitted record parses on its own
        if w:
            m = PB.Records() if kw.get("wrap") else PB.Record()
            m.ParseFromString(w)
    if kw.get("wrap"):
        allm = PB.Records(); allm.ParseFromString(raw)
        assert len(allm.entries) == sum(1 for w in want if w)
    return want


# ------------------------------------------------------------------------------------------------------ rows
def rows(n):
    """n typical flows with every block present: (records, dns, additional, drops, present) as structured arrays."""
    r = np.zeros(n, O.REC_DTYPE)
    r["src_ip"] = list(bytes(10) + b"\xff\xff" + bytes([192, 1, 2, 3]))
    r["dst_ip"] = list(bytes(10) + b"\xff\xff" + bytes([127, 3, 2, 1]))
    r["src_port"], r["dst_port"], r["proto"], r["eth"], r["direction"] = 4321, 443, 6, 0x0800, 1
    r["src_mac"] = [0xaa, 0xbb, 0xcc, 0xdd, 0xee, 0xff]; r["dst_mac"] = [0x11, 0x22, 0x33, 0x44, 0x55, 0x66]
    r["bytes"], r["packets"], r["flags"], r["sampling"], r["dscp"] = 789, 987, 0x10, 50, 10
    r["if_index"], r["nb_obs"] = 7, 1
    r["obs_intf"][:, 0], r["obs_dir"][:, 0] = 9, 0
    r["start"], r["end"] = MONO - 5_000_000_000, MONO - 1
    r["ssl_version"], r["cipher"], r["key_share"], r["tls_types"] = 0x0303, 0x1301, 0x001d, 3
    d = np.zeros(n, O.DNS_DTYPE)
    d["id"], d["flags"], d["latency"] = 7, 0x8180, 12_345
    d["name"] = list(b"\x03www\x07example\x03com".ljust(32, b"\x00"))
    a = np.zeros(n, O.ADD_DTYPE)
    a["rtt"], a["ipsec_enc"] = 1_500, 1
    p = np.zeros(n, O.DROP_DTYPE)
    p["bytes"], p["packets"], p["cause"], p["flags"], p["state"] = 60, 1, 2, 0x10, 7
    return r, d, a, p, np.full(n, 7, np.uint8)


IFACES = [(7, bytes(6), b"veth0", b""), (9, bytes(6), b"eth0", b"blue")]


def edges(bits):
    """0, 1, 2^7k - 1 and 2^7k up to the type's maximum, and the maximum."""
    top = (1 << bits) - 1
    v = {0, 1, top}
    for k in range(1, 10):
        v |= {x for x in ((1 << 7 * k) - 1, 1 << 7 * k) if x <= top}
    return sorted(v)


# (block, field, values): every varint of the record at its edges
VARINT_FIELDS = [
    ("rec", "bytes", edges(64)), ("rec", "packets", edges(32)), ("rec", "src_port", edges(16)), ("rec", "dst_port", edges(16)),
    ("rec", "sampling", edges(32)), ("rec", "flags", edges(16)), ("rec", "dscp", edges(8)), ("rec", "proto", edges(8)),
    ("rec", "icmp_type", edges(8)), ("rec", "icmp_code", edges(8)), ("rec", "ssl_version", edges(16)),
    ("rec", "cipher", edges(16)), ("rec", "key_share", edges(16)), ("rec", "tls_types", edges(8)), ("rec", "misc", [0, 1, 2, 3, 255]),
    ("rec", "if_index", edges(32)), ("rec", "direction", [0, 1, 2, 255]),
    ("drop", "bytes", edges(16)), ("drop", "packets", edges(16)), ("drop", "flags", edges(16)), ("drop", "state", edges(8)),
    ("drop", "cause", edges(32)),
    ("dns", "id", edges(16)), ("dns", "flags", edges(16)), ("dns", "errno", edges(8)),
    ("dns", "latency", [0, 1, 999_999_999, 10**9, 10**9 + 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, U64]),
    ("add", "rtt", [0, 1, 999_999_999, 10**9, 10**9 + 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, U64]),
    ("add", "ipsec_ret", [-(1 << 31), -1, 0, 1, (1 << 31) - 1]), ("add", "ipsec_enc", [0, 1, 2, 255]),
]


def varied(cases):
    """One flow per (block, field, value): the typical flow with that one field changed."""
    r, d, a, p, pr = rows(len(cases))
    blocks = {"rec": r, "dns": d, "add": a, "drop": p}
    for i, (blk, field, v) in enumerate(cases):
        blocks[blk][field][i] = v
    return r, d, a, p, pr


# ------------------------------------------------------------------------------------------------------ 1. fields
def test_every_varint_at_its_edges(be):
    cases = [(b, f, v) for b, f, vals in VARINT_FIELDS for v in vals]
    r, d, a, p, pr = varied(cases)
    check(be, r, d, a, p, pr, ifaces=IFACES)
    pr[::3] = 0                                              # and without the blocks
    check(be, r, d, a, p, pr, ifaces=IFACES, wrap=True, agent=AGENT6, agent_v4=0)


def test_eth_decides_the_address_family(be):
    mapped = list(bytes(10) + b"\xff\xff" + bytes([10, 0, 0, 1])), list(bytes(10) + b"\xff\xff" + bytes([10, 0, 0, 2]))
    native = list(bytes.fromhex("20010db8000000000000000000000001")), list(bytes.fromhex("fe800000000000000000000000000002"))
    cases = [(eth, addrs) for eth in (0, 0x0800, 0x86DD, 0x8100, 0xFFFF) for addrs in (mapped, native)]
    r, d, a, p, pr = rows(len(cases))
    for i, (eth, (s, t)) in enumerate(cases):
        r["eth"][i], r["src_ip"][i], r["dst_ip"][i] = eth, s, t
    check(be, r, d, a, p, pr, ifaces=IFACES)


def test_wrap_prefix_of_one_and_two_bytes(be):
    """Bodies from well under to well over 128 bytes: the Records entry's length takes 1 byte, then 2."""
    cases = [(b, sp) for b in [0] + [1 << 7 * k for k in range(10)] for sp in (0, 1, 128, 16384)]
    r, d, a, p, pr = rows(len(cases))
    pr[:], r["nb_obs"] = 0, 0                                # no blocks, one interface: bodies of 118 to 133 bytes
    for i, (b, sp) in enumerate(cases):
        r["bytes"][i], r["src_port"][i] = b, sp
    want = [len(w) for w in check(be, r, d, a, p, pr, ifaces=IFACES)]
    assert min(want) < 127 and {127, 128} <= set(want) and max(want) > 130, want
    check(be, r, d, a, p, pr, ifaces=IFACES, wrap=True)


# ------------------------------------------------------------------------------------------------------ 2. clocks
CLOCKS = [  # (now_unix_ns, mono_now_ns, [start / end values])
    (NOW, MONO, [MONO, MONO + 1, MONO + 10**9 + 7, MONO + (1 << 62), MONO - 1, MONO - 10**9, 0, 1, U64,
                 MONO + (1 << 63) - 1,                       # Add(+2^63 - 1 ns): past year 2262, out of the int64 ns range
                 (MONO + (1 << 63)) & U64,                   # monoNow - mono == -2^63: -Duration wraps to itself
                 (MONO - (1 << 63)) & U64, (MONO + (1 << 63) + 1) & U64]),
    (0, 0, [0, 1, 10**9, U64, 1 << 63, (1 << 63) - 1, (1 << 63) + 1]),   # now 0, mono_now 0: pre-1970 and the lowest wall clock
    (5, 0, [0, 6, 10**9 + 3, 2 * 10**9 - 1, U64 - 10**9]),   # now smaller than the delta: pre-1970, nanos in [0, 1e9)
    (NOW, U64, [0, U64, U64 - 1, 1 << 63]),
    ((1 << 63) - 1, MONO, [MONO, MONO + (1 << 62), MONO + (1 << 63) - 1, 0]),
]


@pytest.mark.parametrize("clock", range(len(CLOCKS)))
def test_wall_clock_edges(be, clock):
    now, mono, vals = CLOCKS[clock]
    pairs = [(s, e) for s in vals for e in vals[:3]]
    r, d, a, p, pr = rows(len(pairs))
    for i, (s, e) in enumerate(pairs):
        r["start"][i], r["end"][i] = s, e
    check(be, r, d, a, p, pr, now=now, mono=mono, ifaces=IFACES)


def test_clock_far_from_mono_now_is_exact(be):
    """The wall clock past 2262: Go's time.Time.Add keeps seconds and nanoseconds apart, so it does not wrap."""
    r, d, a, p, pr = rows(1)
    r["start"], r["end"] = MONO + (1 << 63) - 1, MONO
    raw, _, _ = encode(be, r, now=NOW, mono=MONO, ifaces=IFACES, total=len(expected(r, ifaces=IFACES)[0]))
    m = PB.Record(); m.ParseFromString(raw)
    assert m.time_flow_start.seconds * 10**9 + m.time_flow_start.nanos == NOW + (1 << 63) - 1
    assert m.time_flow_end.seconds * 10**9 + m.time_flow_end.nanos == NOW


# ------------------------------------------------------------------------------------------------------ 3. DNS names
VALID_NAMES = [
    b"\x03www\x07example\x03com\x00",
    b"abcdefghijklmnopqrstuvwxyz012345",                      # 32 bytes, no terminator: 'a' = 97 overruns
    b"\x1fabcdefghijklmnopqrstuvwxyz01234",                  # one 31-byte label filling all 32 bytes
    b"\x05abc",                                              # a label that overruns the name
    b"\x03abc\x09de",                                        # the second label overruns
    b"\xc0\x0c\x03www",                                      # compression pointer first
    b"\x03www\xc0\x0c\x03com",                               # compression pointer in the middle
    b"\x03abc\x40abc", b"\x03abc\x7fabc", b"\x03abc\x80abc", b"\x03abc\xbfabc",   # length bytes 0x40-0xBF
    b"\x40" + b"a" * 31, b"\x3f" + b"a" * 31,
    b"\x00\x03www", b"", b"\x00" * 32,                       # empty names: no field
    b"\x02" + "\u00e9".encode() + b"\x03" + "\u65e5".encode(),          # multi-byte UTF-8 inside labels
    b"\x04" + "\U0001f600".encode() + b"\x02" + "\u00df".encode(),
    b"\x03" + "\u20ac".encode() + b"\x03" + "\ud7ff".encode() + b"\x03" + "\ue000".encode(),   # around the surrogates
    b"\x04" + "\U0010ffff".encode(),
]
INVALID_NAMES = [
    b"\x01\x80", b"\x03ab\xbf",                              # lone continuation bytes
    b"\x02\xc0\xaf", b"\x02\xc1\xbf", b"\x03\xe0\x80\xaf", b"\x04\xf0\x80\x80\xaf",   # overlong forms
    b"\x03\xed\xa0\x80", b"\x03\xed\xbf\xbf",                # surrogates U+D800, U+DFFF
    b"\x04\xf4\x90\x80\x80", b"\x01\xf5", b"\x01\xff",       # past U+10FFFF, bytes that never occur
    b"\x02\xe2\x82", b"\x01\xc3", b"\x03\xf0\x9f\x98",       # truncated sequences
    b"\x01\xc3\x01\xa9",                                     # a valid pair split by the dot between labels
]


def name_rows(names):
    r, d, a, p, pr = rows(len(names))
    for i, nm in enumerate(names):
        d["name"][i] = list(nm[:32].ljust(32, b"\x00"))
    return r, d, a, p, pr


def test_dns_name_edges(be):
    r, d, a, p, pr = name_rows(VALID_NAMES)
    want = check(be, r, d, a, p, pr, ifaces=IFACES)
    assert all(want)
    names = [PB.dns_dotted(bytes(d["name"][i])) for i in range(len(d))]
    assert names[1] == b"" and names[3] == b"" and names[5] == b"" and names[6] == b"www" and names[13] == b""


def test_invalid_utf8_dns_name_drops_the_record(be):
    """protobuf-go refuses a `string` field that is not UTF-8 and the Kafka exporter drops the record: zero bytes,
    no Records entry, the key still written; the valid flows around it are unaffected."""
    names = [nm for bad in INVALID_NAMES for nm in (VALID_NAMES[0], bad)]
    r, d, a, p, pr = name_rows(names)
    r["src_port"] = np.arange(len(r))
    for wrap in (False, True):
        want = check(be, r, d, a, p, pr, ifaces=IFACES, wrap=wrap)
        assert [bool(w) for w in want] == [True, False] * len(INVALID_NAMES)
    pr[1::2] = 6                                             # without its DNS block the same flow is emitted
    assert all(check(be, r, d, a, p, pr, ifaces=IFACES))


# ------------------------------------------------------------------------------------------------------ 4. interfaces
MAC_S, MAC_D, MAC_X = bytes([2, 0, 0, 0, 0, 1]), bytes([2, 0, 0, 0, 0, 2]), bytes([2, 0, 0, 0, 0, 3])
TABLE = [
    (7, MAC_X, b"veth-other", b"red"),                       # three rows for ifindex 7: the MAC decides, else the first
    (7, MAC_S, b"veth-src", b"udn-src"), (7, MAC_D, b"veth-dst", b""),
    (8, MAC_X, b"only-row", b"green"),                       # one row: its name whatever the MAC
    (9, MAC_X, b"0123456789abcdef", b"u" * 64),              # 16 / 64 bytes exactly
    (10, MAC_X, b"ABCDEFGHIJKLMNOP", b"v" * 64, 200, 255),   # longer lengths: clamped to 16 / 64
    (11, MAC_X, b"", b"", 0, 0),                             # an empty name
    (0, MAC_X, b"lo-zero", b""),                             # ifindex 0
    (12, MAC_X, "\u00e9\u65e5\U0001f600".encode(), "\u00fc".encode()),   # multi-byte UTF-8
    (13, MAC_X, b"bad\xff", b""), (14, MAC_X, b"ok", b"bad\xc3"),   # not UTF-8: the flows naming them are dropped
    (15, MAC_X, b"\xe2\x82\xac\xe2\x82\xac\xe2\x82\xac\xe2\x82\xac\xe2\x82\xac\xe2", b""),   # 16 bytes end mid-sequence
    (16, MAC_X, b"\xe2\x82\xac\xe2\x82\xac\xe2\x82\xac\xe2\x82\xac\xe2\x82\xac\x21\x82\xac", b"", 18, 0),  # the clamp cuts a bad tail
]


def iface_cases():
    """Flows over the table: every ifindex in both directions, observed lists of 0 to 6 interfaces and more."""
    idx = [7, 8, 9, 10, 11, 0, 12, 13, 14, 15, 16, 99]
    cases = [(i, dirn, 0, []) for i in idx for dirn in (0, 1, 2)]
    for nb in (0, 1, 2, 3, 4, 5, 6, 7, 255):
        cases.append((7, 1, nb, [idx[(k + nb) % 7] for k in range(6)]))
    cases.append((7, 0, 3, [13, 7, 7, 0, 0, 0]))            # only the observed list names a bad interface
    cases.append((7, 0, 3, [9, 7, 12, 13, 13, 13]))          # the bad one lies past nb_obs: not looked at
    return cases


def iface_rows_of(cases):
    r, d, a, p, pr = rows(len(cases))
    r["src_mac"], r["dst_mac"] = list(MAC_S), list(MAC_D)
    for i, (ifx, dirn, nb, obs) in enumerate(cases):
        r["if_index"][i], r["direction"][i], r["nb_obs"][i] = ifx, dirn, nb
        for k, o in enumerate(obs):
            r["obs_intf"][i][k], r["obs_dir"][i][k] = o, (k + dirn) % 3
    return r, d, a, p, pr


def test_interface_table_rules(be):
    r, d, a, p, pr = iface_rows_of(iface_cases())
    want = check(be, r, d, a, p, pr, ifaces=TABLE)
    check(be, r, d, a, p, pr, ifaces=TABLE, wrap=True)
    m = PB.Record(); m.ParseFromString(want[0])                          # ifindex 7, direction 0: the dst MAC's row
    assert m.dup_list[0].interface == "veth-dst"
    m.ParseFromString(want[1])                                           # direction 1: the src MAC's row
    assert (m.dup_list[0].interface, m.dup_list[0].udn) == ("veth-src", "udn-src")
    dropped = {c[0] for c, w in zip(iface_cases(), want) if not w and not c[3]}
    assert dropped == {13, 14, 15}
    m.ParseFromString(want[3 * 3])                                       # ifindex 10: clamped to 16 / 64 bytes
    assert (m.dup_list[0].interface, m.dup_list[0].udn) == ("ABCDEFGHIJKLMNOP", "v" * 64)
    n_obs = [len(PB.Record.FromString(w).dup_list) - 1 for w, c in zip(want, iface_cases()) if c[2] and w]
    assert max(n_obs) == 6


def test_no_interface_table_names_every_interface_unknown(be):
    r, d, a, p, pr = iface_rows_of(iface_cases()[:20])
    want = check(be, r, d, a, p, pr, ifaces=None)
    assert all(e.interface == "unknown" and e.udn == "" for w in want for e in PB.Record.FromString(w).dup_list)


def test_interface_table_grows_shrinks_and_grows_again(be):
    """The engine keeps its copy of the table across calls: a shorter table must hide the rows a longer one left."""
    r, d, a, p, pr = iface_rows_of(iface_cases())
    big = TABLE + [(100 + k, MAC_X, f"extra{k}".encode(), b"") for k in range(40)]
    for table in (TABLE[:1], big, TABLE[3:5], big + [(7, MAC_D, b"late-row", b"")] * 30):
        check(be, r, d, a, p, pr, ifaces=table)


# ------------------------------------------------------------------------------------------------------ 5. launch shape
MAX_TABLE = [(k, MAC_X, ("ifname%02d-\u00e9" % k).encode().ljust(16, b"_"), ("udn-%d-" % k).encode().ljust(64, b"z"))
             for k in range(1, 8)]


def max_rows(n):
    """The largest records: IPv6, seven interfaces with 16-byte names and 64-byte UDNs, every block at its widest."""
    r, d, a, p, pr = rows(n)
    r["eth"], r["src_ip"], r["dst_ip"] = 0x86DD, list(b"\xfe" * 16), list(b"\xfd" * 16)
    for f, bits in (("src_port", 16), ("dst_port", 16), ("proto", 8), ("icmp_type", 8), ("icmp_code", 8), ("bytes", 64),
                    ("packets", 32), ("flags", 16), ("sampling", 32), ("dscp", 8), ("ssl_version", 16), ("cipher", 16),
                    ("key_share", 16), ("tls_types", 8), ("misc", 8), ("direction", 8)):
        r[f] = (1 << bits) - 1
    r["src_mac"], r["dst_mac"] = [0xff] * 6, [0xfe] * 6
    r["if_index"], r["nb_obs"] = 1, 6
    r["obs_intf"], r["obs_dir"] = list(range(2, 8)), [255] * 6
    r["start"], r["end"] = 1, 2
    d["id"], d["flags"], d["errno"], d["latency"] = 0xFFFF, 0xFFFF, 255, U64
    d["name"] = list(b"\x1f" + b"m" * 31)
    a["rtt"], a["ipsec_ret"], a["ipsec_enc"] = U64, -1, 1
    p["bytes"], p["packets"], p["flags"], p["state"], p["cause"] = 0xFFFF, 0xFFFF, 0xFFFF, 255, 0xFFFFFFFF
    return r, d, a, p, pr


def cat(*parts):
    return tuple(np.concatenate(x) for x in zip(*parts))


def mixed(n, seed):
    """n flows in CTA-sized runs that alternate between typical and maximum-size records, some dropped."""
    rng = np.random.default_rng(seed)
    r, d, a, p, pr = rows(n)
    r["nb_obs"], pr[:] = 0, rng.choice(np.array([0, 1, 2, 4], np.uint8), n)   # typical: at most one block
    r["src_port"] = rng.integers(0, 1 << 16, n)
    r["start"] = rng.integers(0, MONO * 2, n)
    d["name"][rng.random(n) < 0.02] = list(b"\x02\xc3\x28".ljust(32, b"\x00"))
    big = max_rows(n)
    for i in range(n):
        if (i // 256) % 2 == 1 or rng.random() < 0.02:
            for x, y in zip((r, d, a, p, pr), big):
                x[i] = y[i]
    return r, d, a, p, pr


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1023, 1024, 1025])
def test_launch_shapes(be, n):
    r, d, a, p, pr = mixed(n, seed=n)
    want = check(be, r, d, a, p, pr, ifaces=MAX_TABLE, agent=AGENT6, agent_v4=0)
    per_cta = [sum(len(w) for w in want[k:k + 256]) for k in range(0, n, 256)]
    if n >= 512:
        assert max(per_cta) > 65536 and min(per_cta) < 65536     # non-staged CTAs next to staged ones
    if be.gpu or n in (257, 1025):
        check(be, r, d, a, p, pr, ifaces=MAX_TABLE, agent=AGENT6, agent_v4=0, wrap=True, out_offset=n % 16 or 3)


STAGE_TARGETS = (65536, 65537, 65535, 65536)              # a CTA's bytes plus its 16-byte skew


def stage_edge_flows(off):
    """256 typical flows, then CTAs of 256 flows whose bytes plus skew (the output pointer's phase, off + the bytes
    before the CTA, mod 16) come to exactly STAGE_TARGETS, then 10 more flows."""
    pool = []                                                # typical flows whose one-label DNS name sets the size
    for ln in range(1, 32):
        f = rows(1); f[1]["name"][0] = list((bytes([ln]) + b"q" * ln).ljust(32, b"\x00"))
        pool.append((len(expected(*f, ifaces=MAX_TABLE)[0]), f))
    sizes = [sz for sz, _ in pool]
    lo, hi = sizes[0], sizes[-1]
    assert sizes == list(range(lo, hi + 1))                  # contiguous
    big = max_rows(1)
    m = len(expected(*big, ifaces=MAX_TABLE)[0])
    parts = [rows(256)]
    done = sum(len(w) for w in expected(*parts[0], ifaces=MAX_TABLE))
    for target in STAGE_TARGETS:
        need = target - ((off + done) & 15)
        k = next(k for k in range(256) if (256 - k) * lo <= need - k * m <= (256 - k) * hi)
        extra = need - k * m - (256 - k) * lo
        parts += [big] * k
        for _ in range(256 - k):
            e = min(extra, hi - lo); extra -= e
            parts.append(pool[e][1])
        done += need
    parts.append(rows(10))
    return cat(*parts)


@pytest.mark.parametrize("out_offset", [None, 0, 7, 15])
def test_ctas_at_the_stage_limit(be, out_offset):
    """The staged / direct choice at its boundary: CTAs of 65535, 65536 (staged) and 65537 (direct) bytes with skew."""
    off = out_offset or 0
    flows = stage_edge_flows(off)
    want = check(be, *flows, ifaces=MAX_TABLE, out_offset=out_offset)
    starts = np.concatenate([[0], np.cumsum([len(w) for w in want])])
    for c, target in enumerate(STAGE_TARGETS, start=1):
        assert starts[256 * (c + 1)] - starts[256 * c] + ((off + starts[256 * c]) & 15) == target


def test_misaligned_device_output_and_null_offsets_or_keys(be):
    r, d, a, p, pr = mixed(300, seed=3)
    for off in range(1, 16) if be.gpu else (1, 9, 15):
        check(be, r, d, a, p, pr, ifaces=MAX_TABLE, out_offset=off, offsets=off % 2 == 0, keys=off % 3 == 0)


def test_host_and_device_inputs_mixed(be):
    r, d, a, p, pr = mixed(300, seed=4)
    names = ("recs", "dns", "add", "drops", "present")
    for mask in (0b11111, 0b00001, 0b10110, 0b01001):
        check(be, r, d, a, p, pr, ifaces=MAX_TABLE, on_device={k for b, k in enumerate(names) if mask >> b & 1},
              out_offset=None if mask & 1 else 5)


def test_present_and_block_pointers_disagree(be):
    """A block is used only where its pointer and its present bit are both set."""
    r, d, a, p, pr = rows(8)
    pr[:] = np.arange(8)
    bare = b"".join(expected(r, ifaces=IFACES))
    raw_no_present, _, _ = encode(be, r, d, a, p, None, ifaces=IFACES, total=len(bare))
    raw_no_blocks, _, _ = encode(be, r, None, None, None, pr, ifaces=IFACES, total=len(bare))
    assert raw_no_present == raw_no_blocks == bare
    check(be, r, d, None, p, pr, ifaces=IFACES)
    check(be, r, None, a, None, pr, ifaces=IFACES, on_device={"recs", "add", "present"})


def test_capacity_one_short_writes_nothing(be):
    r, d, a, p, pr = mixed(300, seed=5)
    want = b"".join(expected(r, d, a, p, pr, ifaces=MAX_TABLE))
    rows_, _ = iface_rows(MAX_TABLE)
    prm = pb_params(NOW, MONO, AGENT4, 1, rows_, len(MAX_TABLE), False)
    u8 = [as_u8(x, w) for x, w in ((r, 144), (d, 64), (a, 32), (p, 32))]
    ins = [C.c_void_p(x.ctypes.data) for x in u8] + [C.c_void_p(pr.ctypes.data)]
    out = np.full(len(want) + 64, 0x5A, np.uint8)
    for dev_out in (False, True):
        offs, keys = np.full(301, 0x5A, np.uint64), np.full((300, 32), 0x5A, np.uint8)
        dst = C.c_void_p(be.alloc(len(want) + 64, 0x5A)) if dev_out else C.c_void_p(out.ctypes.data)
        got = C.c_size_t(0)
        rc = be.lib.fa_pb_encode(be.h, *ins, 300, C.byref(prm), dst, len(want) - 1,
                                 C.c_void_p(offs.ctypes.data), C.c_void_p(keys.ctypes.data), C.byref(got))
        assert rc == E2BIG and got.value == len(want)
        img = be.get(dst.value, len(want) + 64) if dev_out else out
        assert (img == 0x5A).all() and (offs == 0x5A).all() and (keys == 0x5A).all()
        rc = be.lib.fa_pb_encode(be.h, *ins, 300, C.byref(prm), dst, len(want),
                                 C.c_void_p(offs.ctypes.data), C.c_void_p(keys.ctypes.data), C.byref(got))
        assert rc == 0 and got.value == len(want)
        img = be.get(dst.value, len(want) + 64) if dev_out else out
        assert img[:len(want)].tobytes() == want and (img[len(want):] == 0x5A).all()


def test_zero_flows(be):
    r = rows(1)[0]
    got = C.c_size_t(7)
    prm = pb_params(NOW, MONO, AGENT4, 1, None, 0, True)
    assert be.lib.fa_pb_encode(be.h, C.c_void_p(r.ctypes.data), None, None, None, None, 0, C.byref(prm), None, 0, None, None,
                               C.byref(got)) == 0
    assert got.value == 0


def test_all_flows_dropped(be):
    r, d, a, p, pr = name_rows([b"\x01\xff"] * 300)
    for wrap in (False, True):
        raw, offs, keys = encode(be, r, d, a, p, pr, ifaces=IFACES, wrap=wrap, total=0)
        assert raw == b"" and not offs.any()
        assert all(keys[i].tobytes() == PB.flow_key(r[i].tobytes()) for i in range(300))


# ------------------------------------------------------------------------------------------------------ 6. past 2^20
def pb_total(body, wrap):
    body = body.astype(np.uint64)
    if not wrap:
        return body
    vl = np.ones_like(body)
    for k in range(1, 5):
        vl += body >= (1 << 7 * k)
    return np.where(body > 0, body + 1 + vl, 0)


def scan_emul():
    import os
    from emul_build import EMUL, build, csrc
    so = build("pb_scan_emul", csrc("pbflow.cu", "common.cuh", "kernels.cuh") + [os.path.join(EMUL, "simt.h")])
    lib = C.CDLL(so)
    lib.pb_scan_emul.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.pb_scan_sums_emul.argtypes = [C.c_void_p, C.c_uint32]
    return lib


def test_scan_of_the_emulation_against_cumsum():
    """pb_scan_block / pb_scan_sums / pb_scan_add over given sizes (zeros, 2- to 5-byte prefixes, u32 maxima whose sum
    passes 2^32); then pb_scan_sums alone over 3,000 block sums, where its carry loop runs three times."""
    lib = scan_emul()
    rng = np.random.default_rng(11)
    for n in (2500,):
        sizes = rng.choice(np.array([0, 1, 127, 128, 16383, 16384, (1 << 21), (1 << 32) - 8], np.uint32), n)
        for wrap in (0, 1):
            offs = np.full(n + 1, 0xEE, np.uint64)
            lib.pb_scan_emul(sizes.ctypes.data, n, wrap, offs.ctypes.data)
            want = np.concatenate([[0], np.cumsum(pb_total(sizes, wrap))]).astype(np.uint64)
            assert np.array_equal(offs, want), (n, wrap)
    for nb in (3000,):
        sums = rng.integers(0, 1 << 40, nb, dtype=np.uint64)
        got = sums.copy()
        lib.pb_scan_sums_emul(got.ctypes.data, nb)
        assert np.array_equal(got, np.concatenate([[0], np.cumsum(sums)[:-1]]).astype(np.uint64)), nb


def templates(t):
    """t distinct flows of varied sizes (about 2 % at the maximum, 1 % dropped for a bad name)."""
    from test_gpu_features import make_add, make_dns
    rng = np.random.default_rng(17)
    recs = gen_host(seed=93, n=t, n_keys=t, dist=0, varying=1).copy()
    rv = recs.view(O.REC_DTYPE).reshape(-1)
    rv["start"] = rng.integers(0, 1 << 64, t, dtype=np.uint64)
    rv["bytes"][::7] = rng.integers(1 << 40, 1 << 63, len(rv[::7]))
    dns = make_dns(rng, recs[:, :40], t)["dns"].copy()
    dns["name"][:, 0] = rng.integers(0, 32, t)               # a first label of 0 to 31 bytes: names of varied length
    dns["name"][::97] = list(b"\x02\xed\xa0".ljust(32, b"\x00"))
    add = make_add(rng, recs[:, :40], t)["add"].copy()
    drops = np.zeros(t, O.DROP_DTYPE)
    drops["bytes"], drops["cause"] = rng.integers(0, 1 << 16, t), rng.integers(0, 1 << 32, t)
    present = rng.integers(0, 8, t).astype(np.uint8)
    big = max_rows(t)
    sel = np.arange(t) % 50 == 3
    r = recs.view(O.REC_DTYPE).reshape(-1)
    for x, y in zip((r, dns, add, drops, present), big):
        x[sel] = y[sel]
    return r, dns, add, drops, present


@pytest.mark.gpu
@pytest.mark.parametrize("n,wrap", [(1 << 20, False), ((1 << 20) + 1, True), (3 * (1 << 20) + 5, False)])
def test_past_2_pow_20_flows_gpu(n, wrap):
    """More than 1024 scan blocks: the templates' own bytes, tiled, are the expected output; offsets are the running
    sum of the template sizes; wrapped, the whole output is one pbflow.Records."""
    import torch
    from netobserv_ebpf_agent_b200._lib import lib
    t = 4_099
    tpl = templates(t)
    be = Backend(gpu=True)
    try:
        eng = be.eng
        want = check(be, *tpl, ifaces=MAX_TABLE, wrap=wrap)       # the templates against the checker
        sizes = np.array([len(w) for w in want], np.uint64)
        assert sizes.max() > 600 and (sizes == 0).sum() > 10
        idx = torch.arange(n, device="cuda") % t
        dev = [torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(t, -1).copy()).cuda()[idx].contiguous()
               for x in tpl]
        rows_, _ = iface_rows(MAX_TABLE)
        prm = pb_params(NOW, MONO, AGENT4, 1, rows_, len(MAX_TABLE), wrap)
        ptrs = [C.c_void_p(x.data_ptr()) for x in dev]
        need = C.c_size_t(0)
        assert lib().fa_pb_encode(eng._h, *ptrs, n, C.byref(prm), None, 0, None, None, C.byref(need)) == E2BIG
        reps, rest = divmod(n, t)
        assert need.value == int(sizes.sum()) * reps + int(sizes[:rest].sum())
        out = torch.full((need.value,), 0xA5, dtype=torch.uint8, device="cuda")
        keys = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
        offs = np.zeros(n + 1, np.uint64)
        assert lib().fa_pb_encode(eng._h, *ptrs, n, C.byref(prm), C.c_void_p(out.data_ptr()), out.numel(),
                                  C.c_void_p(offs.ctypes.data), C.c_void_p(keys.data_ptr()), C.byref(need)) == 0
        cycle = torch.from_numpy(np.frombuffer(b"".join(want), np.uint8).copy()).cuda()
        head = int(sizes[:rest].sum())
        assert torch.equal(out, torch.cat([cycle.repeat(reps), cycle[:head]]))
        assert np.array_equal(offs, np.concatenate([[0], np.cumsum(np.tile(sizes, reps + 1)[:n])]).astype(np.uint64))
        tkeys = torch.from_numpy(np.stack([np.frombuffer(PB.flow_key(x.tobytes()), np.uint8)
                                           for x in as_u8(tpl[0], 144)])).cuda()
        assert torch.equal(keys, tkeys[idx])
        if wrap:
            allm = PB.Records(); allm.ParseFromString(out.cpu().numpy().tobytes())
            assert len(allm.entries) == int((sizes > 0).sum()) * reps + int((sizes[:rest] > 0).sum())
    finally:
        be.close()


# ------------------------------------------------------------------------------------------------------ 7. end to end
def check_end_to_end(be, mode, n, n_keys):
    """Ingest with RTT, DNS and packet drops, fa_evict_ex every block into device memory, fa_pb_encode from there:
    the protobuf library's bytes over the host copy of the same rows."""
    import netobserv_ebpf_agent_b200 as fa
    from netobserv_ebpf_agent_b200._lib import EvictOut
    from test_gpu_features import make_add, make_dns
    from test_pktdrop import make_drops
    rng = np.random.default_rng(23)
    recs = gen_host(seed=24, n=n, n_keys=n_keys, dist=1)
    keys = np.unique(recs[:, :40], axis=0)
    dns = make_dns(rng, keys, n // 3)
    dns["dns"]["name"][::41] = list(b"\x03ab\xff".ljust(32, b"\x00"))        # carried through the fold, then dropped
    dns["dns"]["name"][::2, 0] = rng.integers(0, 32, len(dns[::2]))
    add, drops = make_add(rng, keys, n // 3), make_drops(rng, keys, n // 3)
    flags = fa.FA_F_ENABLE_RTT | fa.FA_F_ENABLE_DNS | fa.FA_F_ENABLE_PKT_DROP
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=flags) as eng:
        assert eng.ingest(recs)[1] == n
        eng.ingest_dns(dns); eng.ingest_additional(add); eng.ingest_pkt_drops(drops)
        live = eng.live_flows()
        widths = (144, 64, 32, 32, 8, 1)
        bufs = [be.alloc(live * w, 0xFF) for w in widths]
        got = C.c_size_t(0)
        assert be.lib.fa_evict_ex(eng._h, C.byref(EvictOut(*bufs)), live, C.byref(got)) == 0 and got.value == live
        host = [be.get(b, live * w).reshape(live, w) for b, w in zip(bufs, widths)]
        assert (host[5] & 1).any() and (host[5] & 2).any() and (host[5] & 4).any()
        table, _ = iface_rows(MAX_TABLE)
        prm = pb_params(NOW, MONO, AGENT6, 0, table, len(MAX_TABLE), False)
        need = C.c_size_t(0)
        ins = [C.c_void_p(bufs[k]) for k in (0, 1, 2, 3, 5)]
        assert be.lib.fa_pb_encode(eng._h, *ins, live, C.byref(prm), None, 0, None, None, C.byref(need)) == E2BIG
        out = be.alloc(need.value + 16, 0xA5)
        offs = np.zeros(live + 1, np.uint64)
        assert be.lib.fa_pb_encode(eng._h, *ins, live, C.byref(prm), C.c_void_p(out + 3), need.value,
                                   C.c_void_p(offs.ctypes.data), None, C.byref(need)) == 0
        raw = be.get(out + 3, need.value).tobytes()
    want = expected(host[0], host[1], host[2], host[3], host[5].reshape(-1), agent=AGENT6, agent_v4=0, ifaces=MAX_TABLE)
    assert raw == b"".join(want)
    assert np.array_equal(offs, np.concatenate([[0], np.cumsum([len(w) for w in want])]).astype(np.uint64))
    assert 0 < sum(1 for w in want if not w) < live


@pytest.mark.parametrize("mode", ["accounter", "kmap"])
def test_evicted_blocks_from_device_memory_end_to_end(be, mode):
    import netobserv_ebpf_agent_b200 as fa
    m = fa.FA_MODE_KERNEL_MAP if mode == "kmap" else fa.FA_MODE_ACCOUNTER
    if be.gpu:
        check_end_to_end(be, m, 200_000, 20_000)
    else:
        check_end_to_end(be, m, 1_500, 300)
