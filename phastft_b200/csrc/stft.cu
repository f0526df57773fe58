// stft.cu -- instantiates STFT-FRAME and ISTFT-OLA (fft_kernels.cuh), the elementwise kernels of the short-time Fourier
// transform and its inverse around the n_fft-point real or complex plan.  Kept out of the main unit so that its compile time
// does not grow.  Compiled per precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

template <>
void launch_stft(bool ola, bool cplx, bool even_fix, const StftParams<PHAST_T>& p, unsigned grid, cudaStream_t stream) {
    using T = PHAST_T;
    if (!ola) {
        if (cplx) stft_frame_kernel<T, true><<<grid, 256, 0, stream>>>(p);
        else stft_frame_kernel<T, false><<<grid, 256, 0, stream>>>(p);
    } else if (cplx) {
        istft_ola_kernel<T, true, false><<<grid, 256, 0, stream>>>(p);
    } else if (even_fix) {
        istft_ola_kernel<T, false, true><<<grid, 256, 0, stream>>>(p);
    } else {
        istft_ola_kernel<T, false, false><<<grid, 256, 0, stream>>>(p);
    }
}

}  // namespace phast
