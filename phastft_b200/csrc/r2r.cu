// r2r.cu -- instantiates DCT-PRE and DCT-POST (fft_kernels.cuh), the elementwise ends of the DCT / DST types 2 and 3 around the
// real any-length plan's interleaved r2c / c2r.  Kept out of the main unit so that its compile time does not grow.  Compiled per
// precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

template <>
void launch_dct<PHAST_T>(bool post, int kind, const DctParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    switch (kind + 4 * post) {
        case DCT_KIND_DCT2: dct_pre_kernel<T, DCT_KIND_DCT2><<<grid, 256, 0, stream>>>(p); break;
        case DCT_KIND_DCT3: dct_pre_kernel<T, DCT_KIND_DCT3><<<grid, 256, 0, stream>>>(p); break;
        case DCT_KIND_DST2: dct_pre_kernel<T, DCT_KIND_DST2><<<grid, 256, 0, stream>>>(p); break;
        case DCT_KIND_DST3: dct_pre_kernel<T, DCT_KIND_DST3><<<grid, 256, 0, stream>>>(p); break;
        case 4 + DCT_KIND_DCT2: dct_post_kernel<T, DCT_KIND_DCT2><<<grid, 256, 0, stream>>>(p); break;
        case 4 + DCT_KIND_DCT3: dct_post_kernel<T, DCT_KIND_DCT3><<<grid, 256, 0, stream>>>(p); break;
        case 4 + DCT_KIND_DST2: dct_post_kernel<T, DCT_KIND_DST2><<<grid, 256, 0, stream>>>(p); break;
        default: dct_post_kernel<T, DCT_KIND_DST3><<<grid, 256, 0, stream>>>(p); break;
    }
}

}  // namespace phast
