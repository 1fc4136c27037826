// emul_sam.cpp -- TEST INFRASTRUCTURE ONLY.  The SAM formatter of kernels.cuh (sam_line, k_sam_len, the offset scan, k_sam_write and the %g
// routine sam_fmt_g) compiled for the host against the CUDA-on-CPU emulation (cuda_shim.hpp), so that tests/test_emul_sam.py can compare it with
// the CPU restatement (tools/view_count_oracle.c) on many random records, and sam_fmt_g with the C library's snprintf("%g").  Never part of
// libbdepth.so.
#include "../../sambamba_b200/csrc/launch.cuh"
#include "../../sambamba_b200/csrc/kernels.cuh"
#include <stdio.h>
#include <vector>

using namespace bdk;

extern "C" {

// The lines of every record of u (records at rec_off[i], the offset of the refID field), as k_sam_len + scan + k_sam_write make them.
// Returns 0, or the SAM_ERR_* code the kernels met; -1 when out_cap is too small.
int emul_sam_format(const uint8_t* u_in, size_t u_len, const int64_t* rec_off, uint32_t R, const char* names, const uint32_t* name_off, int n_ref,
                    char* out, size_t out_cap, size_t* out_len) {
    std::vector<uint8_t> u(u_len + 512, 0);
    memcpy(u.data(), u_in, u_len);
    std::vector<int64_t> off(rec_off, rec_off + R);
    std::vector<uint32_t> meta(R), ncl(R), len(R + 1), tsum(R / SAM_SCAN_TILE + 2);
    std::vector<unsigned long long> offs(R + 1), toff(R / SAM_SCAN_TILE + 2), ctl(4, 0);
    for (uint32_t r = 0; r < R; r++) {
        const uint8_t* p = u.data() + off[r];
        meta[r] = (ldu32(p + 12) >> 16) << 16;
        ncl[r] = (ldu32(p + 8) & 0xFFu) | ((ldu32(p + 12) & 0xFFFFu) << 8);
    }
    RecordSoA soa{nullptr, nullptr, meta.data(), off.data(), ncl.data(), nullptr};
    ViewSel vs{}; vs.region_mode = VIEW_ALL;
    SamTab t{names, name_off, n_ref, ctl.data()};
    const uint32_t n_tiles = (R + SAM_SCAN_TILE - 1) / SAM_SCAN_TILE;
    BD_LAUNCH((R + 7) / 8 ? (R + 7) / 8 : 1, 256, 0, nullptr, k_sam_len)(soa, u.data(), R, INT64_MIN, vs, t, len.data());
    if (ctl[2]) return (int)ctl[2];
    if (n_tiles) {
        BD_LAUNCH(n_tiles, 256, 0, nullptr, k_sam_tile_sum)(len.data(), R, tsum.data());
        BD_LAUNCH(1, 1024, 0, nullptr, k_text_scan)(tsum.data(), n_tiles, toff.data(), ctl.data());
        BD_LAUNCH(n_tiles, 256, 0, nullptr, k_sam_scan_apply)(len.data(), R, toff.data(), offs.data());
    }
    *out_len = ctl[0];
    if (ctl[0] > out_cap) return -1;
    if (R) BD_LAUNCH((R + 7) / 8, 256, 0, nullptr, k_sam_write)(off.data(), u.data(), 0u, R, len.data(), offs.data(), t, out);
    return 0;
}

uint32_t emul_fmt_g(uint32_t bits, char* out) { return sam_fmt_g(bits, out); }

// sam_fmt_g against snprintf("%g", (double)f) on the patterns first + i * step (mod 2^32), i < count: the number of differences, the first in *bad
uint64_t emul_check_g(uint32_t first, uint32_t step, uint64_t count, uint32_t* bad) {
    uint64_t n_bad = 0;
    for (uint64_t i = 0; i < count; i++) {
        const uint32_t bits = first + (uint32_t)i * step;
        float f; memcpy(&f, &bits, 4);
        char a[32], b[64];
        const uint32_t na = sam_fmt_g(bits, a);
        const int nb = snprintf(b, sizeof b, "%g", (double)f);
        if ((int)na != nb || memcmp(a, b, na)) { if (!n_bad) *bad = bits; n_bad++; }
    }
    return n_bad;
}

}
