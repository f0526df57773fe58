// conv.cu -- instantiates CONV-PRE, CONV-MUL and CONV-POST (fft_kernels.cuh), the elementwise kernels of linear convolution and
// correlation around the L-point real or complex plan.  Kept out of the main unit so that its compile time does not grow.
// Compiled per precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

template <>
void launch_conv(int stage, bool cplx, bool corr, const ConvParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    if (stage == CONV_STAGE_PRE) {
        if (cplx) {
            if (corr) conv_pre_kernel<T, true, true><<<grid, 256, 0, stream>>>(p);
            else conv_pre_kernel<T, true, false><<<grid, 256, 0, stream>>>(p);
        } else {
            if (corr) conv_pre_kernel<T, false, true><<<grid, 256, 0, stream>>>(p);
            else conv_pre_kernel<T, false, false><<<grid, 256, 0, stream>>>(p);
        }
    } else if (stage == CONV_STAGE_MUL) {
        conv_mul_kernel<T><<<grid, 256, 0, stream>>>(p);
    } else if (cplx) {
        conv_post_kernel<T, true><<<grid, 256, 0, stream>>>(p);
    } else {
        conv_post_kernel<T, false><<<grid, 256, 0, stream>>>(p);
    }
}

}  // namespace phast
