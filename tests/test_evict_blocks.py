"""fa_evict_ex returns zero in every requested block the table does not produce, whatever memory each block is in: in
blocking and FA_F_NONBLOCKING_EVICT eviction, in both modes, with no feature fold and with RTT only.  Every block is
pre-filled with 0xFF and is host or device memory independently of the others.  The blocks the table does produce
equal what a blocking eviction of the same stream returns into host memory."""
import ctypes as C
import itertools

import numpy as np
import pytest

import oracle_lib as O
from common import gen_host
from test_gpu_features import keys_of, make_add

BLOCKS = ("records", "dns", "additional", "pkt_drops", "rtt_min", "present")
WIDTHS = (144, 64, 32, 32, 8, 1)
PLACEMENTS = list(itertools.product((False, True), repeat=len(BLOCKS)))     # True: the block is device memory
# (mode, non-blocking eviction, RTT fold); ACCOUNTER refuses FA_F_NONBLOCKING_EVICT with feature folds
CONFIGS = [(mode, nb, rtt) for mode in ("accounter", "kmap") for nb in (False, True) for rtt in (False, True)
           if not (mode == "accounter" and nb and rtt)]


def config_id(c):
    return f"{c[0]}-{'nonblocking' if c[1] else 'blocking'}-{'rtt' if c[2] else 'nofold'}"


def evict_ex_filled(eng, cap, device, on_gpu):
    """fa_evict_ex into blocks pre-filled with 0xFF, each in host memory or, where device[i] is set, in device memory
    (torch on the GPU, the engine's own allocations on the emulation) -> the six blocks as (n, width) uint8 arrays."""
    from netobserv_ebpf_agent_b200._lib import EvictOut, check, lib
    bufs, ptrs = [], []
    for w, dev in zip(WIDTHS, device):
        if not dev:
            b = np.full(cap * w, 0xFF, np.uint8); p = b.ctypes.data
        elif on_gpu:
            import torch
            b = torch.full((cap * w,), 0xFF, dtype=torch.uint8, device="cuda"); p = b.data_ptr()
        else:
            b = C.c_void_p(); check(lib().fa_device_alloc(eng._h, cap * w, C.byref(b))); p = b.value
            C.memset(p, 0xFF, cap * w)
        bufs.append(b); ptrs.append(p)
    got = C.c_size_t(0)
    check(lib().fa_evict_ex(eng._h, C.byref(EvictOut(*ptrs)), cap, C.byref(got)))
    out = []
    for b, w in zip(bufs, WIDTHS):
        if isinstance(b, C.c_void_p):
            a = np.frombuffer(C.string_at(b.value, cap * w), np.uint8).copy()
            check(lib().fa_device_free(eng._h, b))
        elif isinstance(b, np.ndarray):
            a = b
        else:
            a = b.cpu().numpy()
        out.append(a[: got.value * w].reshape(got.value, w))
    return out


def check_blocks(config, n, n_keys, placements, on_gpu):
    import netobserv_ebpf_agent_b200 as fa
    mode, nonblocking, rtt = config
    mode = fa.FA_MODE_KERNEL_MAP if mode == "kmap" else fa.FA_MODE_ACCOUNTER
    folds = fa.FA_F_ENABLE_RTT if rtt else 0
    recs = gen_host(seed=5, n=n, n_keys=n_keys, dist=1)
    keys = np.concatenate([np.unique(recs[:, :40], axis=0), keys_of(6, 8)])          # a few flows of samples only
    add = make_add(np.random.default_rng(7), keys, n // 4)
    produced = {"records", "additional", "rtt_min", "present"} if rtt else {"records"}
    flags = folds | (fa.FA_F_NONBLOCKING_EVICT if nonblocking else 0)
    with fa.FlowAggEngine(4 * n_keys, mode=mode, flags=flags) as eng, fa.FlowAggEngine(4 * n_keys, mode=mode, flags=folds) as ref:
        for device in placements:
            for e in (eng, ref):
                assert e.ingest(recs) == (fa.FA_OK, n)
                if rtt:
                    e.ingest_additional(add)
            want = [np.ascontiguousarray(b).view(np.uint8).reshape(len(b), -1) for b in ref.evict_ex()]
            got = evict_ex_filled(eng, len(want[0]), device, on_gpu)
            gp, wp = O.sort_perm(got[0]), O.sort_perm(want[0])
            assert len(gp) == len(wp) > 0
            for name, g, w in zip(BLOCKS, got, want):
                what = (config_id(config), dict(zip(BLOCKS, device)), name)
                if name not in produced:
                    assert not g.any(), what
                assert np.array_equal(g[gp], w[wp]), what


# all blocks in host memory, all in device memory, and each block alone in device memory
FEW_PLACEMENTS = [PLACEMENTS[0], PLACEMENTS[-1]] + [tuple(i == j for j in range(len(BLOCKS))) for i in range(len(BLOCKS))]


@pytest.mark.parametrize("config", CONFIGS, ids=config_id)
def test_unproduced_blocks_are_zero_on_the_emulation(engine_emul, config):
    check_blocks(config, n=1_000, n_keys=150, placements=FEW_PLACEMENTS, on_gpu=False)


@pytest.mark.gpu
@pytest.mark.parametrize("config", CONFIGS, ids=config_id)
def test_unproduced_blocks_are_zero_gpu(config):
    check_blocks(config, n=200_000, n_keys=20_000, placements=PLACEMENTS, on_gpu=True)
