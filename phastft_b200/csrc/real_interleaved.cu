// real_interleaved.cu -- instantiates the interleaved-spectrum ends of the real transforms (phastft_{r2c,c2r}_interleaved_any_*):
// R2C-UNTANGLE-IL / C2R-PRE-IL (power of two), CHIRP-POST-R2C-IL / CHIRP-PRE-C2R-IL (Bluestein), SMOOTH-PRE-C2R-IL, the last
// pass's ODD-R2C-IL store and SMOOTH-POST-R2C-IL (mixed radix).  The MODE_C2R_IN_IL pass tiles come from reg_strided.cu.
// Compiled per precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

template <>
cudaError_t real_il_init<PHAST_T>() {
    return cudaFuncSetAttribute((const void*)odd_tile_kernel<PHAST_T, CHIRP_R2C_DIRECT_IL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                ODD_MAX_ROWS * 128);
}

template <>
void launch_real_il<PHAST_T>(bool untangle, const RealParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    if (untangle) r2c_untangle_kernel<PHAST_T, true><<<grid, 256, 0, stream>>>(p);
    else c2r_preprocess_kernel<PHAST_T, true><<<grid, 256, 0, stream>>>(p);
}

// CHIRP-POST of the r2c modes, CHIRP-PRE of the c2r ones
template <>
void launch_chirp_real_il<PHAST_T>(int mode, const ChirpParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    switch (mode) {
        case CHIRP_R2C_HALVED_IL: chirp_post_kernel<T, CHIRP_R2C_HALVED_IL><<<grid, 256, 0, stream>>>(p); break;
        case CHIRP_R2C_DIRECT_IL: chirp_post_kernel<T, CHIRP_R2C_DIRECT_IL><<<grid, 256, 0, stream>>>(p); break;
        case CHIRP_C2R_HALVED_IL: chirp_pre_kernel<T, CHIRP_C2R_HALVED_IL><<<grid, 256, 0, stream>>>(p); break;
        default: chirp_pre_kernel<T, CHIRP_C2R_DIRECT_IL><<<grid, 256, 0, stream>>>(p); break;
    }
}

template <>
void launch_smooth_pre_real_il<PHAST_T>(int mode, const SmoothParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    if (mode == CHIRP_C2R_HALVED_IL) smooth_pre_kernel<PHAST_T, CHIRP_C2R_HALVED_IL><<<grid, 256, 0, stream>>>(p);
    else smooth_pre_kernel<PHAST_T, CHIRP_C2R_DIRECT_IL><<<grid, 256, 0, stream>>>(p);
}

// the direct r2c's last pass; the halved r2c's stores Z with the complex CHIRP_C2C_IL store (any_interleaved.cu)
template <>
bool launch_odd_r2c_il<PHAST_T>(const OddParams<PHAST_T>& q, int r, size_t smem, unsigned grid, cudaStream_t stream) {
    return launch_odd_kernel<PHAST_T, CHIRP_R2C_DIRECT_IL>(q, r, smem, grid, stream);
}

template <>
void launch_smooth_post_r2c_il<PHAST_T>(const SmoothPostParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    smooth_post_r2c_kernel<PHAST_T, true><<<grid, 256, 0, stream>>>(p);
}

}  // namespace phast
