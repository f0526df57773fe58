// fft_device.cuh -- register-level building blocks for the sm_90a FFT pass kernels.
//
// Replaces, on the GPU, the reference's SIMD butterflies:
//   src/kernels/dit.rs:13-1115   (radix-2 stage kernels, one HBM/L1 sweep per stage)
//   src/kernels/codelets.rs:34-498 (fused FFT-16 / FFT-32 register codelets)
// Here every thread owns a radix-2/4/8/16 DFT entirely in registers (the codelet idea,
// one level up), so a 512-point sub-transform is 3 register stages instead of 9 sweeps.
//
// The "fma(2, lo, -out0)" butterfly form is the reference's own trick
// (kernels/dit.rs:181-183): out0 = lo + w*hi costs 2 FMAs per component and
// out1 = 2*lo - out0 one more, i.e. 6 FMA-pipe ops per butterfly instead of 8.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace phast {

template <typename T> struct Vec2T;
template <> struct Vec2T<double> { using type = double2; };
template <> struct Vec2T<float> { using type = float2; };
template <typename T> using cx = typename Vec2T<T>::type;  // .x = re, .y = im

template <typename T> __device__ __forceinline__ cx<T> make_cx(T re, T im) { cx<T> v; v.x = re; v.y = im; return v; }

__device__ __forceinline__ double fma_t(double a, double b, double c) { return fma(a, b, c); }
__device__ __forceinline__ float fma_t(float a, float b, float c) { return fmaf(a, b, c); }

// a * b (complex)
template <typename T>
__device__ __forceinline__ cx<T> cmul(const cx<T>& a, const cx<T>& b) {
    cx<T> r;
    r.x = fma_t(-a.y, b.y, a.x * b.x);
    r.y = fma_t(a.y, b.x, a.x * b.y);
    return r;
}
__device__ __forceinline__ double2 cmul_d(const double2& a, const double2& b) {
    return make_double2(fma(-a.y, b.y, a.x * b.x), fma(a.y, b.x, a.x * b.y));
}

// ---------------------------------------------------------------------------------------------
// Butterfly primitives on split re/im register arrays.
// bf_w : (lo, hi) -> (lo + w*hi, lo - w*hi) with a generic twiddle, 6 FMA-pipe ops.
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void bf_w(T& lr, T& li, T& hr, T& hi, T wr, T wi) {
    T o0r = fma_t(-wi, hi, fma_t(wr, hr, lr));
    T o0i = fma_t(wi, hr, fma_t(wr, hi, li));
    hr = fma_t(T(2), lr, -o0r);
    hi = fma_t(T(2), li, -o0i);
    lr = o0r;
    li = o0i;
}
// w = 1
template <typename T>
__device__ __forceinline__ void bf_1(T& lr, T& li, T& hr, T& hi) {
    T a = lr + hr, b = li + hi;
    hr = lr - hr; hi = li - hi;
    lr = a; li = b;
}
// w = -j : w*hi = (hi.im, -hi.re)
template <typename T>
__device__ __forceinline__ void bf_mj(T& lr, T& li, T& hr, T& hi) {
    T a = lr + hi, b = li - hr;
    T c = lr - hi, d = li + hr;
    lr = a; li = b; hr = c; hi = d;
}
// w = (1 - j)/sqrt2 : w*hi = s*(hr + hi, hi - hr)
template <typename T>
__device__ __forceinline__ void bf_w8_1(T& lr, T& li, T& hr, T& hi) {
    const T s = T(0.70710678118654752440084436210484903928);
    T p = hr + hi, q = hi - hr;
    T o0r = fma_t(s, p, lr), o0i = fma_t(s, q, li);
    hr = fma_t(T(2), lr, -o0r);
    hi = fma_t(T(2), li, -o0i);
    lr = o0r; li = o0i;
}
// w = (-1 - j)/sqrt2 : w*hi = s*(hi - hr, -(hr + hi))
template <typename T>
__device__ __forceinline__ void bf_w8_3(T& lr, T& li, T& hr, T& hi) {
    const T s = T(0.70710678118654752440084436210484903928);
    T p = hi - hr, q = hr + hi;
    T o0r = fma_t(s, p, lr), o0i = fma_t(-s, q, li);
    hr = fma_t(T(2), lr, -o0r);
    hi = fma_t(T(2), li, -o0i);
    lr = o0r; li = o0i;
}

// ---------------------------------------------------------------------------------------------
// Forward DFTs of length 2/4/8/16 on register arrays, natural order in and out.
// ---------------------------------------------------------------------------------------------
template <typename T, int RAD> struct Dft;

template <typename T> struct Dft<T, 1> {
    static __device__ __forceinline__ void run(T (&)[1], T (&)[1]) {}
};

template <typename T> struct Dft<T, 2> {
    static __device__ __forceinline__ void run(T (&r)[2], T (&i)[2]) { bf_1(r[0], i[0], r[1], i[1]); }
};

template <typename T> struct Dft<T, 4> {
    static __device__ __forceinline__ void run(T (&r)[4], T (&i)[4]) {
        // E = DFT2(x0, x2), O = DFT2(x1, x3)
        bf_1(r[0], i[0], r[2], i[2]);  // r0 = E0, r2 = E1
        bf_1(r[1], i[1], r[3], i[3]);  // r1 = O0, r3 = O1
        // X0 = E0 + O0, X2 = E0 - O0 ; X1 = E1 - j O1, X3 = E1 + j O1
        bf_1(r[0], i[0], r[1], i[1]);   // r0 = X0, r1 = X2
        bf_mj(r[2], i[2], r[3], i[3]);  // r2 = X1, r3 = X3
        T t;
        t = r[1]; r[1] = r[2]; r[2] = t;
        t = i[1]; i[1] = i[2]; i[2] = t;
    }
};

template <typename T> struct Dft<T, 8> {
    static __device__ __forceinline__ void run(T (&r)[8], T (&i)[8]) {
        T er[4] = {r[0], r[2], r[4], r[6]}, ei[4] = {i[0], i[2], i[4], i[6]};
        T orr[4] = {r[1], r[3], r[5], r[7]}, oi[4] = {i[1], i[3], i[5], i[7]};
        Dft<T, 4>::run(er, ei);
        Dft<T, 4>::run(orr, oi);
        bf_1(er[0], ei[0], orr[0], oi[0]);
        bf_w8_1(er[1], ei[1], orr[1], oi[1]);
        bf_mj(er[2], ei[2], orr[2], oi[2]);
        bf_w8_3(er[3], ei[3], orr[3], oi[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k) { r[k] = er[k]; i[k] = ei[k]; r[k + 4] = orr[k]; i[k + 4] = oi[k]; }
    }
};

template <typename T> struct Dft<T, 16> {
    static __device__ __forceinline__ void run(T (&r)[16], T (&i)[16]) {
        T er[8], ei[8], orr[8], oi[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { er[k] = r[2 * k]; ei[k] = i[2 * k]; orr[k] = r[2 * k + 1]; oi[k] = i[2 * k + 1]; }
        Dft<T, 8>::run(er, ei);
        Dft<T, 8>::run(orr, oi);
        const T c1 = T(0.92387953251128675612818318939678828682);  // cos(pi/8)
        const T s1 = T(0.38268343236508977172845998403039886676);  // sin(pi/8)
        bf_1(er[0], ei[0], orr[0], oi[0]);
        bf_w(er[1], ei[1], orr[1], oi[1], c1, -s1);
        bf_w8_1(er[2], ei[2], orr[2], oi[2]);
        bf_w(er[3], ei[3], orr[3], oi[3], s1, -c1);
        bf_mj(er[4], ei[4], orr[4], oi[4]);
        bf_w(er[5], ei[5], orr[5], oi[5], -s1, -c1);
        bf_w8_3(er[6], ei[6], orr[6], oi[6]);
        bf_w(er[7], ei[7], orr[7], oi[7], -c1, -s1);
#pragma unroll
        for (int k = 0; k < 8; ++k) { r[k] = er[k]; i[k] = ei[k]; r[k + 8] = orr[k]; i[k + 8] = oi[k]; }
    }
};

// Radix 32: two radix-16 halves + one level of W_32^k butterflies. 64 live scalars per thread: only
// worth it where it removes a whole shared-memory exchange (1024 = 32*32 in two stages).
template <typename T> struct Dft<T, 32> {
    static __device__ __forceinline__ void run(T (&r)[32], T (&i)[32]) {
        T er[16], ei[16], orr[16], oi[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) { er[k] = r[2 * k]; ei[k] = i[2 * k]; orr[k] = r[2 * k + 1]; oi[k] = i[2 * k + 1]; }
        Dft<T, 16>::run(er, ei);
        Dft<T, 16>::run(orr, oi);
        const T c1 = T(0.980785280403230449126182236134239036973934);  // cos(pi/16)
        const T s1 = T(0.195090322016128267848284868477022240927692);  // sin(pi/16)
        const T c2 = T(0.923879532511286756128183189396788286822417);  // cos(2pi/16)
        const T s2 = T(0.382683432365089771728459984030398866761345);  // sin(2pi/16)
        const T c3 = T(0.831469612302545237078788377617905756738561);  // cos(3pi/16)
        const T s3 = T(0.555570233019602224742830813948532874374937);  // sin(3pi/16)
        bf_1(er[0], ei[0], orr[0], oi[0]);
        bf_w(er[1], ei[1], orr[1], oi[1], c1, -s1);
        bf_w(er[2], ei[2], orr[2], oi[2], c2, -s2);
        bf_w(er[3], ei[3], orr[3], oi[3], c3, -s3);
        bf_w8_1(er[4], ei[4], orr[4], oi[4]);
        bf_w(er[5], ei[5], orr[5], oi[5], s3, -c3);
        bf_w(er[6], ei[6], orr[6], oi[6], s2, -c2);
        bf_w(er[7], ei[7], orr[7], oi[7], s1, -c1);
        bf_mj(er[8], ei[8], orr[8], oi[8]);
        bf_w(er[9], ei[9], orr[9], oi[9], -s1, -c1);
        bf_w(er[10], ei[10], orr[10], oi[10], -s2, -c2);
        bf_w(er[11], ei[11], orr[11], oi[11], -s3, -c3);
        bf_w8_3(er[12], ei[12], orr[12], oi[12]);
        bf_w(er[13], ei[13], orr[13], oi[13], -c3, -s3);
        bf_w(er[14], ei[14], orr[14], oi[14], -c2, -s2);
        bf_w(er[15], ei[15], orr[15], oi[15], -c1, -s1);
#pragma unroll
        for (int k = 0; k < 16; ++k) { r[k] = er[k]; i[k] = ei[k]; r[k + 16] = orr[k]; i[k + 16] = oi[k]; }
    }
};

// ---------------------------------------------------------------------------------------------
// Forward DFTs of length 3/5/7 (the odd passes of the mixed-radix path), natural order in and out.  With a_j = x_j + x_(p-j)
// and b_j = x_j - x_(p-j):  X_k = A_k - i B_k and X_(p-k) = A_k + i B_k,  A_k = x_0 + sum_j cos(2 pi jk/p) a_j,
// B_k = sum_j sin(2 pi jk/p) b_j: real constants times complex values, all in FMA form.
// ---------------------------------------------------------------------------------------------
// (X_k, X_(p-k)) from A and B
template <typename T>
__device__ __forceinline__ void odd_pair(T ar, T ai, T br, T bi, T& kr, T& ki, T& mr, T& mi) {
    kr = ar + bi; ki = ai - br;
    mr = ar - bi; mi = ai + br;
}

template <typename T> struct Dft<T, 3> {
    static __device__ __forceinline__ void run(T (&r)[3], T (&i)[3]) {
        const T s = T(0.8660254037844386467637231707529361834714);  // sin(2pi/3)
        const T ar = r[1] + r[2], ai = i[1] + i[2];
        const T br = s * (r[1] - r[2]), bi = s * (i[1] - i[2]);
        const T mr = fma_t(T(-0.5), ar, r[0]), mi = fma_t(T(-0.5), ai, i[0]);
        r[0] += ar; i[0] += ai;
        odd_pair(mr, mi, br, bi, r[1], i[1], r[2], i[2]);
    }
};

template <typename T> struct Dft<T, 5> {
    static __device__ __forceinline__ void run(T (&r)[5], T (&i)[5]) {
        const T c1 = T(0.3090169943749474241022934171828190588602);   // cos(2pi/5)
        const T c2 = T(-0.8090169943749474241022934171828190588602);  // cos(4pi/5)
        const T s1 = T(0.9510565162951535721164393333793821434057);   // sin(2pi/5)
        const T s2 = T(0.5877852522924731291687059546390727685977);   // sin(4pi/5)
        const T a1r = r[1] + r[4], a1i = i[1] + i[4], b1r = r[1] - r[4], b1i = i[1] - i[4];
        const T a2r = r[2] + r[3], a2i = i[2] + i[3], b2r = r[2] - r[3], b2i = i[2] - i[3];
        const T A1r = fma_t(c2, a2r, fma_t(c1, a1r, r[0])), A1i = fma_t(c2, a2i, fma_t(c1, a1i, i[0]));
        const T A2r = fma_t(c1, a2r, fma_t(c2, a1r, r[0])), A2i = fma_t(c1, a2i, fma_t(c2, a1i, i[0]));
        const T B1r = fma_t(s2, b2r, s1 * b1r), B1i = fma_t(s2, b2i, s1 * b1i);
        const T B2r = fma_t(-s1, b2r, s2 * b1r), B2i = fma_t(-s1, b2i, s2 * b1i);
        r[0] += a1r + a2r; i[0] += a1i + a2i;
        odd_pair(A1r, A1i, B1r, B1i, r[1], i[1], r[4], i[4]);
        odd_pair(A2r, A2i, B2r, B2i, r[2], i[2], r[3], i[3]);
    }
};

template <typename T> struct Dft<T, 7> {
    static __device__ __forceinline__ void run(T (&r)[7], T (&i)[7]) {
        const T c1 = T(0.6234898018587335305250048840042398106323);   // cos(2pi/7)
        const T c2 = T(-0.2225209339563144042889025644967947594664);  // cos(4pi/7)
        const T c3 = T(-0.9009688679024191262361023195074450511659);  // cos(6pi/7)
        const T s1 = T(0.7818314824680298087084445266740577502323);   // sin(2pi/7)
        const T s2 = T(0.9749279121818236070181316829939312172328);   // sin(4pi/7)
        const T s3 = T(0.4338837391175581204757683328483587546100);   // sin(6pi/7)
        const T a1r = r[1] + r[6], a1i = i[1] + i[6], b1r = r[1] - r[6], b1i = i[1] - i[6];
        const T a2r = r[2] + r[5], a2i = i[2] + i[5], b2r = r[2] - r[5], b2i = i[2] - i[5];
        const T a3r = r[3] + r[4], a3i = i[3] + i[4], b3r = r[3] - r[4], b3i = i[3] - i[4];
        const T A1r = fma_t(c3, a3r, fma_t(c2, a2r, fma_t(c1, a1r, r[0]))), A1i = fma_t(c3, a3i, fma_t(c2, a2i, fma_t(c1, a1i, i[0])));
        const T A2r = fma_t(c1, a3r, fma_t(c3, a2r, fma_t(c2, a1r, r[0]))), A2i = fma_t(c1, a3i, fma_t(c3, a2i, fma_t(c2, a1i, i[0])));
        const T A3r = fma_t(c2, a3r, fma_t(c1, a2r, fma_t(c3, a1r, r[0]))), A3i = fma_t(c2, a3i, fma_t(c1, a2i, fma_t(c3, a1i, i[0])));
        const T B1r = fma_t(s3, b3r, fma_t(s2, b2r, s1 * b1r)), B1i = fma_t(s3, b3i, fma_t(s2, b2i, s1 * b1i));
        const T B2r = fma_t(-s1, b3r, fma_t(-s3, b2r, s2 * b1r)), B2i = fma_t(-s1, b3i, fma_t(-s3, b2i, s2 * b1i));
        const T B3r = fma_t(s2, b3r, fma_t(-s1, b2r, s3 * b1r)), B3i = fma_t(s2, b3i, fma_t(-s1, b2i, s3 * b1i));
        r[0] += a1r + a2r + a3r; i[0] += a1i + a2i + a3i;
        odd_pair(A1r, A1i, B1r, B1i, r[1], i[1], r[6], i[6]);
        odd_pair(A2r, A2i, B2r, B2i, r[2], i[2], r[5], i[5]);
        odd_pair(A3r, A3i, B3r, B3i, r[3], i[3], r[4], i[4]);
    }
};

// ---------------------------------------------------------------------------------------------
// Complex-array interface of the DFTs: DftC<T, RAD>::run(x[RAD]) and ctwid(a, w) = a * w.
// Both precisions unpack into the split re/im arrays above (the reference's fma(2, lo, -out0) butterfly,
// kernels/dit.rs:181-183).  The float twiddle product rounds a.y*w.x (not a.x*w.y) before its imaginary FMA; the
// f32 results of the library are defined with that order.
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ cx<T> ctwid(const cx<T>& a, const cx<T>& w) { return cmul<T>(a, w); }
template <> __device__ __forceinline__ float2 ctwid<float>(const float2& a, const float2& w) {
    return make_float2(fmaf(-a.y, w.y, a.x * w.x), fmaf(a.x, w.y, a.y * w.x));
}
template <typename T> __device__ __forceinline__ cx<T> cscale(const cx<T>& a, T s) { return make_cx<T>(a.x * s, a.y * s); }

template <typename T, int RAD> struct DftC {
    static __device__ __forceinline__ void run(cx<T> (&x)[RAD]) {
        T r[RAD], i[RAD];
#pragma unroll
        for (int k = 0; k < RAD; ++k) { r[k] = x[k].x; i[k] = x[k].y; }
        Dft<T, RAD>::run(r, i);
#pragma unroll
        for (int k = 0; k < RAD; ++k) x[k] = make_cx<T>(r[k], i[k]);
    }
};

// ---------------------------------------------------------------------------------------------
// Compile-time radix lists.
// ---------------------------------------------------------------------------------------------
__host__ __device__ constexpr int ilog2_c(int v) { return v <= 1 ? 0 : 1 + ilog2_c(v >> 1); }

template <int... Rs> struct RadixList {
    static constexpr int S = sizeof...(Rs);
    __host__ __device__ static constexpr int rad(int s) {
        constexpr int a[sizeof...(Rs)] = {Rs...};
        return a[s];
    }
    __host__ __device__ static constexpr int R() {
        int p = 1;
        for (int s = 0; s < S; ++s) p *= rad(s);
        return p;
    }
    // product of radices before stage s (Ns)
    __host__ __device__ static constexpr int Ns(int s) {
        int p = 1;
        for (int q = 0; q < s; ++q) p *= rad(q);
        return p;
    }
    __host__ __device__ static constexpr int max_rad() {
        int m = 1;
        for (int s = 0; s < S; ++s) m = rad(s) > m ? rad(s) : m;
        return m;
    }
    __host__ __device__ static constexpr int min_rad() {
        int m = 1 << 30;
        for (int s = 0; s < S; ++s) m = rad(s) < m ? rad(s) : m;
        return m;
    }
};

// Offset (in complex elements) of stage s's [i][m] twiddle table inside the concatenation used by the one-CTA kernels:
// stage q (1 <= q < S) owns L_q = Ns(q) * rad(q) entries.
template <class RL>
__host__ __device__ constexpr int tw_im_offset(int s) {
    int off = 0;
    for (int q = 1; q < s; ++q) off += RL::Ns(q) * RL::rad(q);
    return off;
}

// Digit reversal of the tail index for stage 1:  mp = n_2*(M/r_2) + n_3*(M/(r_2 r_3)) + ... + n_S
//   ->  j = n_2 + r_2*n_3 + r_2*r_3*n_4 + ...        (M = R / r_1)
template <class RL>
__device__ __forceinline__ int rev_tail(int mp) {
    if constexpr (RL::S <= 2) {
        return mp;
    } else {
        constexpr int M = RL::R() / RL::rad(0);
        int j = 0;
        int w_in = M, w_out = 1;
#pragma unroll
        for (int s = 1; s < RL::S; ++s) {
            const int rs = RL::rad(s);
            w_in /= rs;
            j += ((mp / w_in) & (rs - 1)) * w_out;
            w_out *= rs;
        }
        return j;
    }
}

// Two-level twiddle lookup: W_N^(e_n) = hi[e_n >> lo_bits] * lo[e_n & lo_mask], tables in f64.
struct Tw2 {
    const double2* __restrict__ hi;
    const double2* __restrict__ lo;
    int lo_bits;
    __device__ __forceinline__ double2 get(uint32_t e_n) const {
        double2 h = __ldg(hi + (e_n >> lo_bits));
        double2 l = __ldg(lo + (e_n & ((1u << lo_bits) - 1u)));
        return cmul_d(h, l);
    }
};

template <typename T> __device__ __forceinline__ cx<T> to_cx(const double2& v) { return make_cx<T>(T(v.x), T(v.y)); }

}  // namespace phast
