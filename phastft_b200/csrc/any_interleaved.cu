// any_interleaved.cu -- instantiates the interleaved complex modes (CHIRP_C2C_IL / CHIRP_C2C_IL_SWAP) of the any-length plan's
// end kernels: CHIRP-PRE-IL / CHIRP-POST-IL (Bluestein), SMOOTH-PRE-IL and the last pass's ODD-IL store (mixed radix).
// Compiled per precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

template <>
cudaError_t any_il_init<PHAST_T>() {
    using T = PHAST_T;
    for (const void* k : {(const void*)odd_tile_kernel<T, CHIRP_C2C_IL>, (const void*)odd_tile_kernel<T, CHIRP_C2C_IL_SWAP>})
        if (cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, ODD_MAX_ROWS * 128)) return e;
    return cudaSuccess;
}

template <>
bool launch_odd_il<PHAST_T>(int mode, const OddParams<PHAST_T>& q, int r, size_t smem, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    return mode == CHIRP_C2C_IL ? launch_odd_kernel<T, CHIRP_C2C_IL>(q, r, smem, grid, stream)
                                : launch_odd_kernel<T, CHIRP_C2C_IL_SWAP>(q, r, smem, grid, stream);
}

template <>
void launch_smooth_pre_il<PHAST_T>(int mode, const SmoothParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    if (mode == CHIRP_C2C_IL) smooth_pre_kernel<T, CHIRP_C2C_IL><<<grid, 256, 0, stream>>>(p);
    else smooth_pre_kernel<T, CHIRP_C2C_IL_SWAP><<<grid, 256, 0, stream>>>(p);
}

template <>
void launch_chirp_il<PHAST_T>(int mode, bool post, const ChirpParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    if (mode == CHIRP_C2C_IL) {
        if (post) chirp_post_kernel<T, CHIRP_C2C_IL><<<grid, 256, 0, stream>>>(p);
        else chirp_pre_kernel<T, CHIRP_C2C_IL><<<grid, 256, 0, stream>>>(p);
    } else {
        if (post) chirp_post_kernel<T, CHIRP_C2C_IL_SWAP><<<grid, 256, 0, stream>>>(p);
        else chirp_pre_kernel<T, CHIRP_C2C_IL_SWAP><<<grid, 256, 0, stream>>>(p);
    }
}

}  // namespace phast
