// pb_scan_emul.cpp — K8's exclusive scan (pb_scan_block / pb_scan_sums / pb_scan_add of csrc/pbflow.cu) on the host
// over simt.h, one OS thread per CUDA thread (test infrastructure, never part of libflowagg.so).  A batch past 1024 scan
// blocks (2^20 flows) is too large for fa_pb_encode on the engine emulation, so tests/test_pbflow_edges.py drives the
// scan kernels directly over given record sizes.
#define FA_HOST_EMUL 1
#include "simt.h"

#include <vector>

#undef __shared__
#define __shared__ static          // static shared arrays: one CTA at a time
#include "../../netobserv_ebpf_agent_b200/csrc/pbflow.cu"
#undef __shared__

using namespace fa;

namespace {
void launch_serial(unsigned grid, unsigned block, const std::function<void()>& body) {
    for (unsigned b = 0; b < grid; b++) {
        std::vector<std::thread> th;
        simt::Cta cta; cta.sync_all = std::make_unique<simt::Barrier>(block);
        for (unsigned w = 0; w < block / 32; w++) cta.warps.push_back(std::make_unique<simt::Warp>());
        for (unsigned t = 0; t < block; t++)
            th.emplace_back([&, t] {
                simt::Ctx c; c.tid = {t, 0, 0}; c.bid = {b, 0, 0}; c.bdim = {block, 1, 1}; c.gdim = {grid, 1, 1};
                c.lane = (int)(t & 31); c.cta = &cta; c.warp = cta.warps[t >> 5].get();
                simt::g_ctx = &c; body(); simt::g_ctx = nullptr;
            });
        for (auto& x : th) x.join();
    }
}
}  // namespace

// the three scan kernels over n record sizes -> offsets (n + 1 entries), as launch_pb_sizes runs them
extern "C" void pb_scan_emul(const uint32_t* sizes, uint32_t n, uint32_t wrap, unsigned long long* offsets) {
    const uint32_t nb = (n + kScanBlock - 1) / kScanBlock;
    std::vector<unsigned long long> sums(nb);
    unsigned long long* bs = sums.data();
    launch_serial(nb, kScanBlock, [=] { pb_scan_block_kernel(sizes, n, wrap, offsets, bs); });
    launch_serial(1, kScanBlock, [=] { pb_scan_sums_kernel(bs, nb); });
    launch_serial(nb, kScanBlock, [=] { pb_scan_add_kernel(offsets, n, bs, sizes, wrap); });
}
// pb_scan_sums_kernel alone over n_blocks block sums, in place (its carry loop runs once per 1024 of them)
extern "C" void pb_scan_sums_emul(unsigned long long* block_sums, uint32_t n_blocks) {
    launch_serial(1, kScanBlock, [=] { pb_scan_sums_kernel(block_sums, n_blocks); });
}
