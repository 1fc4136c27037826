// emul_bgzf.cpp -- TEST INFRASTRUCTURE ONLY.  The BGZF compressor (bgzf_deflate.cuh, k_bgzf_deflate) and the member cut of `view -f bam`
// (kernels.cuh, k_bam_next .. k_bam_members) compiled for the host against the CUDA-on-CPU emulation (cuda_shim.hpp), so that
// tests/test_emul_bam.py can inflate the members with zlib and compare the cut with the CPU restatement (tools/view_count_oracle.c).
// Never part of libbdepth.so.
#include "../../sambamba_b200/csrc/launch.cuh"
#include "../../sambamba_b200/csrc/kernels.cuh"
#include <vector>

using namespace bdk;

extern "C" {

// Members i < n: len[i] bytes at in + off[i], compressed at `level` into out + i * 65536 (out_len[i] bytes).  grid: CTAs to launch.
void emul_bgzf_compress(const uint8_t* in, const uint64_t* off, const uint32_t* len, uint32_t n, int level, uint32_t grid, uint8_t* out, uint32_t* out_len) {
    std::vector<uint32_t> tok((size_t)grid * DF_THREADS * 256);
    std::vector<unsigned long long> o(off, off + n);
    if (n) BD_LAUNCH(grid, DF_THREADS, DF_SMEM, nullptr, k_bgzf_deflate)(in, o.data(), len, n, level, out, out_len, tok.data());
}

// One sub-batch of the member cut: R records of size[r] bytes (0: not selected) behind *P carried bytes with BamWriter._current_size *cur.
// Writes the closed members' stage offsets and lengths (m_off, m_len: room for 3 * (P + total) / 0xFF00 + 4) and returns their number;
// *P and *cur become the carried state after the sub-batch.
uint32_t emul_bam_cut(const uint32_t* size, uint32_t R, uint32_t* P, unsigned long long* cur, unsigned long long* m_off, uint32_t* m_len) {
    std::vector<unsigned long long> off(R + 1), base(R + 2), ctl(16, 0);
    std::vector<uint32_t> sz(size, size + R), cnt(R + 1), tsum(R / SAM_SCAN_TILE + 2);
    std::vector<unsigned long long> toff(R / SAM_SCAN_TILE + 2);
    const uint32_t n_tiles = (R + SAM_SCAN_TILE - 1) / SAM_SCAN_TILE;
    BD_LAUNCH(n_tiles, 256, 0, nullptr, k_sam_tile_sum)(sz.data(), R, tsum.data());
    BD_LAUNCH(1, 1024, 0, nullptr, k_text_scan)(tsum.data(), n_tiles, toff.data(), &ctl[0]);
    BD_LAUNCH(n_tiles, 256, 0, nullptr, k_sam_scan_apply)(sz.data(), R, toff.data(), off.data());
    const unsigned long long total = ctl[0];
    const unsigned long long groups = std::min<unsigned long long>(R, 2 * (*P + total) / BGZF_BLOCK + 3);
    uint32_t K = 1; while ((1ull << K) < groups + 1) K++;
    std::vector<uint32_t> J((size_t)(R + 1) * K); std::vector<uint8_t> mark(R + 1, 0); uint32_t s0 = 0;
    const unsigned g = (R + 256) / 256;
    BD_LAUNCH(g, 256, 0, nullptr, k_bam_next)(off.data(), R, total, J.data());
    for (uint32_t k = 1; k < K; k++) BD_LAUNCH(g, 256, 0, nullptr, k_bam_jump)(J.data() + (size_t)(k - 1) * (R + 1), J.data() + (size_t)k * (R + 1), R);
    BD_LAUNCH(1, 1, 0, nullptr, k_bam_start)(off.data(), R, total, *cur, mark.data(), &s0);
    for (uint32_t k = K; k-- > 0;) BD_LAUNCH(g, 256, 0, nullptr, k_bam_mark)(J.data() + (size_t)k * (R + 1), mark.data(), R);
    BD_LAUNCH(g, 256, 0, nullptr, k_bam_members<false>)(off.data(), R, total, J.data(), mark.data(), &s0, *P, *cur, cnt.data(), nullptr, nullptr, nullptr, nullptr);
    const uint32_t n2 = (R + 1 + SAM_SCAN_TILE - 1) / SAM_SCAN_TILE;
    std::vector<uint32_t> ts2(n2 + 1); std::vector<unsigned long long> to2(n2 + 1);
    BD_LAUNCH(n2, 256, 0, nullptr, k_sam_tile_sum)(cnt.data(), R + 1, ts2.data());
    BD_LAUNCH(1, 1024, 0, nullptr, k_text_scan)(ts2.data(), n2, to2.data(), &ctl[5]);
    BD_LAUNCH(n2, 256, 0, nullptr, k_sam_scan_apply)(cnt.data(), R + 1, to2.data(), base.data());
    BD_LAUNCH(g, 256, 0, nullptr, k_bam_members<true>)(off.data(), R, total, J.data(), mark.data(), &s0, *P, *cur, cnt.data(), base.data(), m_off, m_len, &ctl[3]);
    *P = (uint32_t)ctl[3]; *cur = ctl[4];
    return (uint32_t)ctl[5];
}

}
