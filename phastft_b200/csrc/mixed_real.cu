// mixed_real.cu -- instantiates the real any-length plan's modes of the mixed-radix kernels (SMOOTH-PRE-R2C / -C2R, the last
// ODD pass's ODD-R2C / ODD-C2R stores, SMOOTH-POST-R2C).  Compiled per precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

template <>
cudaError_t mixed_real_init<PHAST_T>() {
    using T = PHAST_T;
    for (const void* k : {(const void*)odd_tile_kernel<T, CHIRP_R2C_DIRECT>, (const void*)odd_tile_kernel<T, CHIRP_C2R_HALVED>,
                          (const void*)odd_tile_kernel<T, CHIRP_C2R_DIRECT>})
        if (cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, ODD_MAX_ROWS * 128)) return e;
    return cudaSuccess;
}

// the halved r2c's last pass stores Z with the C2C store (launch_odd_kernel<T, CHIRP_C2C> in phastft_cuda.cu)
template <>
bool launch_odd_real<PHAST_T>(int mode, const OddParams<PHAST_T>& q, int r, size_t smem, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    switch (mode) {
        case CHIRP_R2C_DIRECT: return launch_odd_kernel<T, CHIRP_R2C_DIRECT>(q, r, smem, grid, stream);
        case CHIRP_C2R_HALVED: return launch_odd_kernel<T, CHIRP_C2R_HALVED>(q, r, smem, grid, stream);
        case CHIRP_C2R_DIRECT: return launch_odd_kernel<T, CHIRP_C2R_DIRECT>(q, r, smem, grid, stream);
        default: return false;
    }
}

template <>
void launch_smooth_pre_real<PHAST_T>(int mode, const SmoothParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    switch (mode) {
        case CHIRP_R2C_HALVED: smooth_pre_kernel<T, CHIRP_R2C_HALVED><<<grid, 256, 0, stream>>>(p); break;
        case CHIRP_R2C_DIRECT: smooth_pre_kernel<T, CHIRP_R2C_DIRECT><<<grid, 256, 0, stream>>>(p); break;
        case CHIRP_C2R_HALVED: smooth_pre_kernel<T, CHIRP_C2R_HALVED><<<grid, 256, 0, stream>>>(p); break;
        default: smooth_pre_kernel<T, CHIRP_C2R_DIRECT><<<grid, 256, 0, stream>>>(p); break;
    }
}

template <>
void launch_smooth_post_r2c<PHAST_T>(const SmoothPostParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    smooth_post_r2c_kernel<PHAST_T><<<grid, 256, 0, stream>>>(p);
}

}  // namespace phast
