// emul_json.cpp -- TEST INFRASTRUCTURE ONLY.  The JSON formatter of kernels.cuh (json_line, k_json_len, the offset scan, k_json_write) compiled
// for the host against the CUDA-on-CPU emulation (cuda_shim.hpp), so that tests/test_emul_json.py can compare it with the CPU restatement of
// toJson (tools/view_count_oracle.c) on many random records.  Never part of libbdepth.so.
#include "../../sambamba_b200/csrc/launch.cuh"
#include "../../sambamba_b200/csrc/kernels.cuh"
#include <vector>

using namespace bdk;

extern "C" {

// The JSON records of every record of u (records at rec_off[i], the offset of the refID field), as k_json_len + scan + k_json_write make
// them; names / name_off are the reference names as the library uploads them, quoted and escaped.  Returns 0, or the SAM_ERR_* code the
// kernels met; -1 when out_cap is too small.
int emul_json_format(const uint8_t* u_in, size_t u_len, const int64_t* rec_off, uint32_t R, const char* names, const uint32_t* name_off, int n_ref,
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
    BD_LAUNCH((R + 7) / 8 ? (R + 7) / 8 : 1, 256, 0, nullptr, k_json_len)(soa, u.data(), R, INT64_MIN, vs, t, len.data());
    if (ctl[2]) return (int)ctl[2];
    if (n_tiles) {
        BD_LAUNCH(n_tiles, 256, 0, nullptr, k_sam_tile_sum)(len.data(), R, tsum.data());
        BD_LAUNCH(1, 1024, 0, nullptr, k_text_scan)(tsum.data(), n_tiles, toff.data(), ctl.data());
        BD_LAUNCH(n_tiles, 256, 0, nullptr, k_sam_scan_apply)(len.data(), R, toff.data(), offs.data());
    }
    *out_len = ctl[0];
    if (ctl[0] > out_cap) return -1;
    if (R) BD_LAUNCH((R + 7) / 8, 256, 0, nullptr, k_json_write)(off.data(), u.data(), 0u, R, len.data(), offs.data(), t, out);
    return 0;
}

}
