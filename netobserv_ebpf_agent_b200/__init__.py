"""netobserv_ebpf_agent_b200 — H100-native flow-aggregation engine.

Host-side Python mirror of the C ABI in include/flowagg.h.  The compute path is
libflowagg.so (hand-written sm_90a CUDA); there is NO CPU fallback: importing
works anywhere (so the build can be checked without a GPU), but creating an
engine without a CUDA device raises FlowAggError(FA_E_NODEV).
"""
from ._lib import (FA_FULL, FA_OK, FlowAggError, GenParams, Stats, lib, lib_path,  # noqa: F401
                   FA_F_ENABLE_DNS, FA_F_ENABLE_RTT, FA_F_ENABLE_SKETCH, FA_F_NO_FULL_CUT, FA_F_RINGBUF_FALLBACK, FA_F_ENABLE_PKT_DROP, FA_F_NONBLOCKING_EVICT,
                   FA_GEN_UNIFORM, FA_GEN_ZIPF, FA_TOP_BYTES, FA_TOP_PACKETS, FA_TOP_MAX_K,
                   FA_HIST_BYTES, FA_HIST_PACKETS, FA_HIST_DURATION, FA_HIST_RTT, FA_HIST_DNS_LATENCY, FA_HIST_MAX_BOUNDS,
                   FA_MODE_ACCOUNTER, FA_MODE_KERNEL_MAP, DISTINCT_DTYPE, GROUP_DTYPE, REC_BYTES, hist_dtype)
from .engine import FILTER_CIDR_DTYPE, FILTER_RULE_DTYPE, FlowAggEngine, gen_records_host, gen_key, group_mask  # noqa: F401
from .accounter import Accounter, MapTracer, new_record_times  # noqa: F401

__all__ = ["FlowAggEngine", "Accounter", "MapTracer", "FlowAggError", "GenParams", "Stats", "lib", "lib_path",
           "gen_records_host", "gen_key", "group_mask", "hist_dtype", "new_record_times"]
