// emul_valid.cpp -- TEST INFRASTRUCTURE ONLY.  The validator of `view -v` in kernels.cuh (k_view_valid) compiled for the host against the
// CUDA-on-CPU emulation (cuda_shim.hpp), so that tests/test_emul_valid.py can compare it with the CPU restatement of isValid
// (tools/view_count_oracle.c) on many random records.  Never part of libbdepth.so.
#include "../../sambamba_b200/csrc/launch.cuh"
#include "../../sambamba_b200/csrc/kernels.cuh"
#include <vector>

using namespace bdk;

extern "C" {

// st[i] = the VV_* status k_view_valid gives the record at rec_off[i] of u (the offset of its refID field): 0 valid, 255 invalid, otherwise the
// SAM_ERR_* code of the refusal.
void emul_view_valid(const uint8_t* u_in, size_t u_len, const int64_t* rec_off, uint32_t R, uint8_t* st) {
    std::vector<uint8_t> u(u_len + 512, 0);
    memcpy(u.data(), u_in, u_len);
    std::vector<int64_t> off(rec_off, rec_off + R);
    RecordSoA soa{nullptr, nullptr, nullptr, off.data(), nullptr, nullptr};
    if (R) BD_LAUNCH((R + VV_WARPS - 1) / VV_WARPS, VV_WARPS * 32, 0, nullptr, k_view_valid)(soa, u.data(), R, INT64_MIN, st);
}

}
