// phastft.hpp -- C++ host-side mirror of PhastFT's public API over the C ABI (include/phastft_cuda.h).
//
// The reference is compiled code (Rust) and there is no Rust toolchain in the build image, so the
// host side above the C ABI is also provided in C++: same names, argument meaning and error
// behaviour as the reference crate (src/lib.rs:143-226, src/planner.rs, src/options.rs,
// src/algorithms/r2c.rs:521-895).  Where the reference panics these throw phastft::Panic whose
// what() is the reference's panic message.  Header-only; link with -lphastft_cuda.
#pragma once

#include <complex>
#include <cstddef>
#include <stdexcept>
#include <string>
#include <vector>

#include "../include/phastft_cuda.h"

namespace phastft {

struct Panic : std::runtime_error {
    int code;
    Panic(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

inline void check(int32_t code) {
    if (code == PHASTFT_OK) return;
    std::string msg = phastft_status_message(code);
    if (code >= PHASTFT_ERR_INVALID_ARG) { msg += ": "; msg += phastft_last_error(); }
    throw Panic(code, msg);
}

/// planner.rs:10-16
enum class Direction : int { Forward = 1, Reverse = -1 };
/// planner.rs:25-32
enum class PlannerMode : int { Heuristic = 0, Tune = 1 };   // Tune is real here (times candidate plans); the reference ignores it, planner.rs:65

/// options.rs:10-43
struct Options {
    bool multithreaded_bit_reversal = false;
    std::size_t smallest_parallel_chunk_size = 16384;
    static Options guess_options(std::size_t input_size) {
        phastft_options o;
        phastft_options_guess(input_size, &o);
        Options r;
        r.multithreaded_bit_reversal = o.multithreaded_bit_reversal != 0;
        r.smallest_parallel_chunk_size = o.smallest_parallel_chunk_size;
        return r;
    }
};

namespace detail {
template <typename T> struct Api;
template <> struct Api<double> {
    using Dit = phastft_plan_dit_f64; using R2c = phastft_plan_r2c_f64;
    static int32_t dit_create(std::size_t n, int dev, int mode, Dit** o) { return phastft_plan_dit_f64_create(n, dev, mode, o); }
    static void dit_destroy(Dit* p) { phastft_plan_dit_f64_destroy(p); }
    static std::size_t dit_size(const Dit* p) { return phastft_plan_dit_f64_size(p); }
    static const char* dit_describe(const Dit* p) { return phastft_plan_dit_f64_describe(p); }
    static int32_t dit_reserve(const Dit* p, std::size_t b) { return phastft_plan_dit_f64_reserve(p, b); }
    static int32_t fft_dev(const Dit* p, double* re, double* im, int d, std::size_t b, std::size_t st, void* s) { return phastft_fft_dit_f64_dev(p, re, im, d, b, st, s); }
    static int32_t fft_batch_host(Dit* const* ps, int np, double* re, double* im, std::size_t b, std::size_t st, int d) { return phastft_fft_dit_f64_batch_sharded_host(ps, np, re, im, b, st, d); }
    static int32_t r2c_oneshot(const double* in, std::size_t li, double* ore, std::size_t lre, double* oim, std::size_t lim) { return phastft_r2c_f64_oneshot(in, li, ore, lre, oim, lim, 0); }
    static int32_t c2r_oneshot(const double* ire, std::size_t lre, const double* iim, std::size_t lim, double* out, std::size_t lo) { return phastft_c2r_f64_oneshot(ire, lre, iim, lim, out, lo, 0); }
    static int32_t fft_host(const Dit* p, double* re, std::size_t lr, double* im, std::size_t li, int d) { return phastft_fft_dit_f64_host(p, re, lr, im, li, d, nullptr); }
    static int32_t r2c_create(std::size_t n, int dev, R2c** o) { return phastft_plan_r2c_f64_create(n, dev, o); }
    static int32_t r2c_reserve(const R2c* p, std::size_t b) { return phastft_plan_r2c_f64_reserve(p, b); }
    static const char* r2c_describe(const R2c* p, std::size_t b) { return phastft_plan_r2c_f64_describe_batch(p, b); }
    static int32_t r2c_batch_dev(const R2c* p, const double* in, std::size_t is, double* ore, double* oim, std::size_t os, std::size_t b, void* s) { return phastft_r2c_f64_batch_dev(p, in, is, ore, oim, os, b, s); }
    static int32_t c2r_batch_dev(const R2c* p, const double* ire, const double* iim, std::size_t is, double* out, std::size_t os, double* sre, double* sim, std::size_t b, void* s) { return phastft_c2r_f64_batch_dev(p, ire, iim, is, out, os, sre, sim, b, s); }
    static void r2c_destroy(R2c* p) { phastft_plan_r2c_f64_destroy(p); }
    static int32_t r2c_host(const R2c* p, const double* in, std::size_t li, double* ore, std::size_t lre, double* oim, std::size_t lim) { return phastft_r2c_f64_host(p, in, li, ore, lre, oim, lim); }
    static int32_t c2r_host(const R2c* p, const double* ire, std::size_t lre, const double* iim, std::size_t lim, double* out, std::size_t lo, double* sre, std::size_t lsr, double* sim, std::size_t lsi) { return phastft_c2r_f64_host(p, ire, lre, iim, lim, out, lo, sre, lsr, sim, lsi); }
    using Any = phastft_plan_any_f64;
    static int32_t any_create(std::size_t n, int dev, int algo, Any** o) { return phastft_plan_any_f64_create_with(n, dev, algo, o); }
    static void any_destroy(Any* p) { phastft_plan_any_f64_destroy(p); }
    static std::size_t any_size(const Any* p) { return phastft_plan_any_f64_size(p); }
    static const char* any_describe(const Any* p) { return phastft_plan_any_f64_describe(p); }
    static int32_t any_reserve(const Any* p, std::size_t b) { return phastft_plan_any_f64_reserve(p, b); }
    static int32_t any_dev(const Any* p, double* re, double* im, int d, std::size_t b, std::size_t st, void* s) { return phastft_fft_any_f64_dev(p, re, im, d, b, st, s); }
    static int32_t any_host(const Any* p, double* re, std::size_t lr, double* im, std::size_t li, int d) { return phastft_fft_any_f64_host(p, re, lr, im, li, d); }
    static int32_t any_il_dev(const Any* p, double* sig, int d, std::size_t b, std::size_t st, void* s) { return phastft_fft_interleaved_any_f64_dev(p, sig, d, b, st, s); }
    static int32_t any_il_host(const Any* p, double* sig, std::size_t len, int d) { return phastft_fft_interleaved_any_f64_host(p, sig, len, d); }
    using R2cAny = phastft_plan_r2c_any_f64;
    static int32_t r2c_any_create(std::size_t n, int dev, int algo, R2cAny** o) { return phastft_plan_r2c_any_f64_create_with(n, dev, algo, o); }
    static void r2c_any_destroy(R2cAny* p) { phastft_plan_r2c_any_f64_destroy(p); }
    static std::size_t r2c_any_size(const R2cAny* p) { return phastft_plan_r2c_any_f64_size(p); }
    static const char* r2c_any_describe(const R2cAny* p) { return phastft_plan_r2c_any_f64_describe(p); }
    static int32_t r2c_any_reserve(const R2cAny* p, std::size_t b) { return phastft_plan_r2c_any_f64_reserve(p, b); }
    static int32_t r2c_any_dev(const R2cAny* p, const double* in, std::size_t is, double* ore, double* oim, std::size_t os, std::size_t b, void* s) { return phastft_r2c_any_f64_dev(p, in, is, ore, oim, os, b, s); }
    static int32_t c2r_any_dev(const R2cAny* p, const double* ire, const double* iim, std::size_t is, double* out, std::size_t os, std::size_t b, void* s) { return phastft_c2r_any_f64_dev(p, ire, iim, is, out, os, b, s); }
    static int32_t r2c_any_host(const R2cAny* p, const double* in, std::size_t li, double* ore, std::size_t lre, double* oim, std::size_t lim) { return phastft_r2c_any_f64_host(p, in, li, ore, lre, oim, lim); }
    static int32_t c2r_any_host(const R2cAny* p, const double* ire, std::size_t lre, const double* iim, std::size_t lim, double* out, std::size_t lo) { return phastft_c2r_any_f64_host(p, ire, lre, iim, lim, out, lo); }
    static int32_t r2c_il_dev(const R2cAny* p, const double* in, std::size_t is, double* out, std::size_t os, std::size_t b, void* s) { return phastft_r2c_interleaved_any_f64_dev(p, in, is, out, os, b, s); }
    static int32_t c2r_il_dev(const R2cAny* p, const double* in, std::size_t is, double* out, std::size_t os, std::size_t b, void* s) { return phastft_c2r_interleaved_any_f64_dev(p, in, is, out, os, b, s); }
    static int32_t r2c_il_host(const R2cAny* p, const double* in, std::size_t li, double* out, std::size_t lo) { return phastft_r2c_interleaved_any_f64_host(p, in, li, out, lo); }
    static int32_t c2r_il_host(const R2cAny* p, const double* in, std::size_t li, double* out, std::size_t lo) { return phastft_c2r_interleaved_any_f64_host(p, in, li, out, lo); }
    using Dct = phastft_plan_dct_f64;
    static int32_t dct_create(std::size_t n, int dev, int algo, Dct** o) { return phastft_plan_dct_f64_create_with(n, dev, algo, o); }
    static void dct_destroy(Dct* p) { phastft_plan_dct_f64_destroy(p); }
    static std::size_t dct_size(const Dct* p) { return phastft_plan_dct_f64_size(p); }
    static const char* dct_describe(const Dct* p) { return phastft_plan_dct_f64_describe(p); }
    static int32_t dct_reserve(const Dct* p, std::size_t b) { return phastft_plan_dct_f64_reserve(p, b); }
    static int32_t dct_dev(const Dct* p, int k, int nm, const double* in, std::size_t is, double* out, std::size_t os, std::size_t b, void* s) { return phastft_dct_f64_dev(p, k, nm, in, is, out, os, b, s); }
    static int32_t dct_host(const Dct* p, int k, int nm, const double* in, std::size_t li, double* out, std::size_t lo) { return phastft_dct_f64_host(p, k, nm, in, li, out, lo); }
    using Conv = phastft_plan_conv_f64;
    static int32_t conv_create(std::size_t nx, std::size_t nh, int dom, int dev, Conv** o) { return phastft_plan_conv_f64_create(nx, nh, dom, dev, o); }
    static void conv_destroy(Conv* p) { phastft_plan_conv_f64_destroy(p); }
    static std::size_t conv_fft_len(const Conv* p) { return phastft_plan_conv_f64_fft_len(p); }
    static const char* conv_describe(const Conv* p) { return phastft_plan_conv_f64_describe(p); }
    static int32_t conv_reserve(const Conv* p, std::size_t b) { return phastft_plan_conv_f64_reserve(p, b); }
    static int32_t conv_dev(const Conv* p, int op, int m, const double* x, std::size_t xs, const double* h, std::size_t hs, double* y, std::size_t ys, std::size_t b, void* s) { return phastft_conv_f64_dev(p, op, m, x, xs, h, hs, y, ys, b, s); }
    static int32_t conv_host(const Conv* p, int op, int m, const double* x, std::size_t lx, const double* h, std::size_t lh, double* y, std::size_t ly) { return phastft_conv_f64_host(p, op, m, x, lx, h, lh, y, ly); }
    using Stft = phastft_plan_stft_f64;
    static int32_t stft_create(std::size_t n, std::size_t nf, std::size_t hop, const double* w, std::size_t wl, int c, int pm, int dom, int dev, Stft** o) { return phastft_plan_stft_f64_create(n, nf, hop, w, wl, c, pm, dom, dev, o); }
    static void stft_destroy(Stft* p) { phastft_plan_stft_f64_destroy(p); }
    static std::size_t stft_frames(const Stft* p) { return phastft_plan_stft_f64_frames(p); }
    static std::size_t stft_bins(const Stft* p) { return phastft_plan_stft_f64_bins(p); }
    static const char* stft_describe(const Stft* p) { return phastft_plan_stft_f64_describe(p); }
    static int32_t stft_reserve(const Stft* p, std::size_t b) { return phastft_plan_stft_f64_reserve(p, b); }
    static int32_t stft_dev(const Stft* p, int nz, const double* x, std::size_t xs, double* s, std::size_t fs, std::size_t b, void* st) { return phastft_stft_f64_dev(p, nz, x, xs, s, fs, b, st); }
    static int32_t istft_dev(const Stft* p, int nz, const double* s, std::size_t fs, double* y, std::size_t ys, std::size_t b, void* st) { return phastft_istft_f64_dev(p, nz, s, fs, y, ys, b, st); }
    static int32_t stft_host(const Stft* p, int nz, const double* x, std::size_t lx, double* s, std::size_t ls) { return phastft_stft_f64_host(p, nz, x, lx, s, ls); }
    static int32_t istft_host(const Stft* p, int nz, const double* s, std::size_t ls, double* y, std::size_t ly) { return phastft_istft_f64_host(p, nz, s, ls, y, ly); }
};
template <> struct Api<float> {
    using Dit = phastft_plan_dit_f32; using R2c = phastft_plan_r2c_f32;
    static int32_t dit_create(std::size_t n, int dev, int mode, Dit** o) { return phastft_plan_dit_f32_create(n, dev, mode, o); }
    static void dit_destroy(Dit* p) { phastft_plan_dit_f32_destroy(p); }
    static std::size_t dit_size(const Dit* p) { return phastft_plan_dit_f32_size(p); }
    static const char* dit_describe(const Dit* p) { return phastft_plan_dit_f32_describe(p); }
    static int32_t dit_reserve(const Dit* p, std::size_t b) { return phastft_plan_dit_f32_reserve(p, b); }
    static int32_t fft_dev(const Dit* p, float* re, float* im, int d, std::size_t b, std::size_t st, void* s) { return phastft_fft_dit_f32_dev(p, re, im, d, b, st, s); }
    static int32_t fft_batch_host(Dit* const* ps, int np, float* re, float* im, std::size_t b, std::size_t st, int d) { return phastft_fft_dit_f32_batch_sharded_host(ps, np, re, im, b, st, d); }
    static int32_t r2c_oneshot(const float* in, std::size_t li, float* ore, std::size_t lre, float* oim, std::size_t lim) { return phastft_r2c_f32_oneshot(in, li, ore, lre, oim, lim, 0); }
    static int32_t c2r_oneshot(const float* ire, std::size_t lre, const float* iim, std::size_t lim, float* out, std::size_t lo) { return phastft_c2r_f32_oneshot(ire, lre, iim, lim, out, lo, 0); }
    static int32_t fft_host(const Dit* p, float* re, std::size_t lr, float* im, std::size_t li, int d) { return phastft_fft_dit_f32_host(p, re, lr, im, li, d, nullptr); }
    static int32_t r2c_create(std::size_t n, int dev, R2c** o) { return phastft_plan_r2c_f32_create(n, dev, o); }
    static int32_t r2c_reserve(const R2c* p, std::size_t b) { return phastft_plan_r2c_f32_reserve(p, b); }
    static const char* r2c_describe(const R2c* p, std::size_t b) { return phastft_plan_r2c_f32_describe_batch(p, b); }
    static int32_t r2c_batch_dev(const R2c* p, const float* in, std::size_t is, float* ore, float* oim, std::size_t os, std::size_t b, void* s) { return phastft_r2c_f32_batch_dev(p, in, is, ore, oim, os, b, s); }
    static int32_t c2r_batch_dev(const R2c* p, const float* ire, const float* iim, std::size_t is, float* out, std::size_t os, float* sre, float* sim, std::size_t b, void* s) { return phastft_c2r_f32_batch_dev(p, ire, iim, is, out, os, sre, sim, b, s); }
    static void r2c_destroy(R2c* p) { phastft_plan_r2c_f32_destroy(p); }
    static int32_t r2c_host(const R2c* p, const float* in, std::size_t li, float* ore, std::size_t lre, float* oim, std::size_t lim) { return phastft_r2c_f32_host(p, in, li, ore, lre, oim, lim); }
    static int32_t c2r_host(const R2c* p, const float* ire, std::size_t lre, const float* iim, std::size_t lim, float* out, std::size_t lo, float* sre, std::size_t lsr, float* sim, std::size_t lsi) { return phastft_c2r_f32_host(p, ire, lre, iim, lim, out, lo, sre, lsr, sim, lsi); }
    using Any = phastft_plan_any_f32;
    static int32_t any_create(std::size_t n, int dev, int algo, Any** o) { return phastft_plan_any_f32_create_with(n, dev, algo, o); }
    static void any_destroy(Any* p) { phastft_plan_any_f32_destroy(p); }
    static std::size_t any_size(const Any* p) { return phastft_plan_any_f32_size(p); }
    static const char* any_describe(const Any* p) { return phastft_plan_any_f32_describe(p); }
    static int32_t any_reserve(const Any* p, std::size_t b) { return phastft_plan_any_f32_reserve(p, b); }
    static int32_t any_dev(const Any* p, float* re, float* im, int d, std::size_t b, std::size_t st, void* s) { return phastft_fft_any_f32_dev(p, re, im, d, b, st, s); }
    static int32_t any_host(const Any* p, float* re, std::size_t lr, float* im, std::size_t li, int d) { return phastft_fft_any_f32_host(p, re, lr, im, li, d); }
    static int32_t any_il_dev(const Any* p, float* sig, int d, std::size_t b, std::size_t st, void* s) { return phastft_fft_interleaved_any_f32_dev(p, sig, d, b, st, s); }
    static int32_t any_il_host(const Any* p, float* sig, std::size_t len, int d) { return phastft_fft_interleaved_any_f32_host(p, sig, len, d); }
    using R2cAny = phastft_plan_r2c_any_f32;
    static int32_t r2c_any_create(std::size_t n, int dev, int algo, R2cAny** o) { return phastft_plan_r2c_any_f32_create_with(n, dev, algo, o); }
    static void r2c_any_destroy(R2cAny* p) { phastft_plan_r2c_any_f32_destroy(p); }
    static std::size_t r2c_any_size(const R2cAny* p) { return phastft_plan_r2c_any_f32_size(p); }
    static const char* r2c_any_describe(const R2cAny* p) { return phastft_plan_r2c_any_f32_describe(p); }
    static int32_t r2c_any_reserve(const R2cAny* p, std::size_t b) { return phastft_plan_r2c_any_f32_reserve(p, b); }
    static int32_t r2c_any_dev(const R2cAny* p, const float* in, std::size_t is, float* ore, float* oim, std::size_t os, std::size_t b, void* s) { return phastft_r2c_any_f32_dev(p, in, is, ore, oim, os, b, s); }
    static int32_t c2r_any_dev(const R2cAny* p, const float* ire, const float* iim, std::size_t is, float* out, std::size_t os, std::size_t b, void* s) { return phastft_c2r_any_f32_dev(p, ire, iim, is, out, os, b, s); }
    static int32_t r2c_any_host(const R2cAny* p, const float* in, std::size_t li, float* ore, std::size_t lre, float* oim, std::size_t lim) { return phastft_r2c_any_f32_host(p, in, li, ore, lre, oim, lim); }
    static int32_t c2r_any_host(const R2cAny* p, const float* ire, std::size_t lre, const float* iim, std::size_t lim, float* out, std::size_t lo) { return phastft_c2r_any_f32_host(p, ire, lre, iim, lim, out, lo); }
    static int32_t r2c_il_dev(const R2cAny* p, const float* in, std::size_t is, float* out, std::size_t os, std::size_t b, void* s) { return phastft_r2c_interleaved_any_f32_dev(p, in, is, out, os, b, s); }
    static int32_t c2r_il_dev(const R2cAny* p, const float* in, std::size_t is, float* out, std::size_t os, std::size_t b, void* s) { return phastft_c2r_interleaved_any_f32_dev(p, in, is, out, os, b, s); }
    static int32_t r2c_il_host(const R2cAny* p, const float* in, std::size_t li, float* out, std::size_t lo) { return phastft_r2c_interleaved_any_f32_host(p, in, li, out, lo); }
    static int32_t c2r_il_host(const R2cAny* p, const float* in, std::size_t li, float* out, std::size_t lo) { return phastft_c2r_interleaved_any_f32_host(p, in, li, out, lo); }
    using Dct = phastft_plan_dct_f32;
    static int32_t dct_create(std::size_t n, int dev, int algo, Dct** o) { return phastft_plan_dct_f32_create_with(n, dev, algo, o); }
    static void dct_destroy(Dct* p) { phastft_plan_dct_f32_destroy(p); }
    static std::size_t dct_size(const Dct* p) { return phastft_plan_dct_f32_size(p); }
    static const char* dct_describe(const Dct* p) { return phastft_plan_dct_f32_describe(p); }
    static int32_t dct_reserve(const Dct* p, std::size_t b) { return phastft_plan_dct_f32_reserve(p, b); }
    static int32_t dct_dev(const Dct* p, int k, int nm, const float* in, std::size_t is, float* out, std::size_t os, std::size_t b, void* s) { return phastft_dct_f32_dev(p, k, nm, in, is, out, os, b, s); }
    static int32_t dct_host(const Dct* p, int k, int nm, const float* in, std::size_t li, float* out, std::size_t lo) { return phastft_dct_f32_host(p, k, nm, in, li, out, lo); }
    using Conv = phastft_plan_conv_f32;
    static int32_t conv_create(std::size_t nx, std::size_t nh, int dom, int dev, Conv** o) { return phastft_plan_conv_f32_create(nx, nh, dom, dev, o); }
    static void conv_destroy(Conv* p) { phastft_plan_conv_f32_destroy(p); }
    static std::size_t conv_fft_len(const Conv* p) { return phastft_plan_conv_f32_fft_len(p); }
    static const char* conv_describe(const Conv* p) { return phastft_plan_conv_f32_describe(p); }
    static int32_t conv_reserve(const Conv* p, std::size_t b) { return phastft_plan_conv_f32_reserve(p, b); }
    static int32_t conv_dev(const Conv* p, int op, int m, const float* x, std::size_t xs, const float* h, std::size_t hs, float* y, std::size_t ys, std::size_t b, void* s) { return phastft_conv_f32_dev(p, op, m, x, xs, h, hs, y, ys, b, s); }
    static int32_t conv_host(const Conv* p, int op, int m, const float* x, std::size_t lx, const float* h, std::size_t lh, float* y, std::size_t ly) { return phastft_conv_f32_host(p, op, m, x, lx, h, lh, y, ly); }
    using Stft = phastft_plan_stft_f32;
    static int32_t stft_create(std::size_t n, std::size_t nf, std::size_t hop, const float* w, std::size_t wl, int c, int pm, int dom, int dev, Stft** o) { return phastft_plan_stft_f32_create(n, nf, hop, w, wl, c, pm, dom, dev, o); }
    static void stft_destroy(Stft* p) { phastft_plan_stft_f32_destroy(p); }
    static std::size_t stft_frames(const Stft* p) { return phastft_plan_stft_f32_frames(p); }
    static std::size_t stft_bins(const Stft* p) { return phastft_plan_stft_f32_bins(p); }
    static const char* stft_describe(const Stft* p) { return phastft_plan_stft_f32_describe(p); }
    static int32_t stft_reserve(const Stft* p, std::size_t b) { return phastft_plan_stft_f32_reserve(p, b); }
    static int32_t stft_dev(const Stft* p, int nz, const float* x, std::size_t xs, float* s, std::size_t fs, std::size_t b, void* st) { return phastft_stft_f32_dev(p, nz, x, xs, s, fs, b, st); }
    static int32_t istft_dev(const Stft* p, int nz, const float* s, std::size_t fs, float* y, std::size_t ys, std::size_t b, void* st) { return phastft_istft_f32_dev(p, nz, s, fs, y, ys, b, st); }
    static int32_t stft_host(const Stft* p, int nz, const float* x, std::size_t lx, float* s, std::size_t ls) { return phastft_stft_f32_host(p, nz, x, lx, s, ls); }
    static int32_t istft_host(const Stft* p, int nz, const float* s, std::size_t ls, float* y, std::size_t ly) { return phastft_istft_f32_host(p, nz, s, ls, y, ly); }
};

/// planner.rs:34-114
template <typename T>
class PlannerDit {
  public:
    explicit PlannerDit(std::size_t num_points, int device = 0) : PlannerDit(num_points, PlannerMode::Heuristic, device) {}
    PlannerDit(std::size_t num_points, PlannerMode mode, int device = 0) { check(Api<T>::dit_create(num_points, device, (int)mode, &raw_)); }
    static PlannerDit with_mode(std::size_t num_points, PlannerMode mode) { return PlannerDit(num_points, mode); }
    ~PlannerDit() { if (raw_) Api<T>::dit_destroy(raw_); }
    PlannerDit(PlannerDit&& o) noexcept : raw_(o.raw_) { o.raw_ = nullptr; }
    PlannerDit(const PlannerDit&) = delete;
    PlannerDit& operator=(const PlannerDit&) = delete;
    const typename Api<T>::Dit* raw() const { return raw_; }
    typename Api<T>::Dit* raw_mut() const { return raw_; }
    std::size_t num_points() const { return Api<T>::dit_size(raw_); }
    /// additive: the pass decomposition and kernels the planner chose
    std::string describe() const { return Api<T>::dit_describe(raw_); }
    /// additive: size the device workspace for calls of up to `batch` transforms now
    void reserve(std::size_t batch) const { check(Api<T>::dit_reserve(raw_, batch)); }
  private:
    typename Api<T>::Dit* raw_ = nullptr;
};

/// planner.rs:164-212
template <typename T>
class PlannerR2c {
  public:
    explicit PlannerR2c(std::size_t n, int device = 0) { check(Api<T>::r2c_create(n, device, &raw_)); }
    ~PlannerR2c() { if (raw_) Api<T>::r2c_destroy(raw_); }
    PlannerR2c(PlannerR2c&& o) noexcept : raw_(o.raw_) { o.raw_ = nullptr; }
    PlannerR2c(const PlannerR2c&) = delete;
    PlannerR2c& operator=(const PlannerR2c&) = delete;
    const typename Api<T>::R2c* raw() const { return raw_; }
    /// additive: the c2r path calls of `batch` transforms take (describe_batch; batch 1 = describe)
    std::string describe(std::size_t batch = 1) const { return Api<T>::r2c_describe(raw_, batch); }
    /// additive: make every allocation a batched call of `batch` transforms would make now
    void reserve(std::size_t batch) const { check(Api<T>::r2c_reserve(raw_, batch)); }
    /// additive: `batch` r2c transforms on device pointers, member b at b * in_stride reals / b * out_stride bins
    void r2c_batch_dev(const T* d_in, std::size_t in_stride, T* d_out_re, T* d_out_im, std::size_t out_stride, std::size_t batch,
                       void* stream = nullptr) const {
        check(Api<T>::r2c_batch_dev(raw_, d_in, in_stride, d_out_re, d_out_im, out_stride, batch, stream));
    }
    /// additive: `batch` c2r transforms; scratch batch * N/2 each, dense, or both null for the plan's own
    void c2r_batch_dev(const T* d_in_re, const T* d_in_im, std::size_t in_stride, T* d_out, std::size_t out_stride, std::size_t batch,
                       T* d_scratch_re = nullptr, T* d_scratch_im = nullptr, void* stream = nullptr) const {
        check(Api<T>::c2r_batch_dev(raw_, d_in_re, d_in_im, in_stride, d_out, out_stride, d_scratch_re, d_scratch_im, batch, stream));
    }
  private:
    typename Api<T>::R2c* raw_ = nullptr;
};

/// How a length that is not a power of two is transformed (PHASTFT_ANY_*).  Auto takes Mixed for every eligible length
/// (2^a 3^b 5^c 7^d below 2^30 whose odd part fits one or two odd passes) and Bluestein otherwise, from the factorisation alone.
enum class AnyAlgo : int { Bluestein = PHASTFT_ANY_BLUESTEIN, Mixed = PHASTFT_ANY_MIXED, Auto = PHASTFT_ANY_AUTO };

/// additive: a complex FFT of any length (a power of two runs the c2c plan; any other length up to 2^29 - 1 Bluestein's
/// algorithm, or with AnyAlgo::Mixed / AnyAlgo::Auto the mixed-radix path for smooth lengths below 2^30)
template <typename T>
class PlannerAny {
  public:
    explicit PlannerAny(std::size_t num_points, int device = 0, AnyAlgo algo = AnyAlgo::Bluestein) {
        check(Api<T>::any_create(num_points, device, static_cast<int>(algo), &raw_));
    }
    ~PlannerAny() { if (raw_) Api<T>::any_destroy(raw_); }
    PlannerAny(PlannerAny&& o) noexcept : raw_(o.raw_) { o.raw_ = nullptr; }
    PlannerAny(const PlannerAny&) = delete;
    PlannerAny& operator=(const PlannerAny&) = delete;
    std::size_t num_points() const { return Api<T>::any_size(raw_); }
    /// "power of two", "Bluestein M=2^m" or "mixed 2^a x Q_a[ x Q_b]", then the inner plan's description
    std::string describe() const { return Api<T>::any_describe(raw_); }
    /// make every allocation a call of `batch` transforms would make now
    void reserve(std::size_t batch) const { check(Api<T>::any_reserve(raw_, batch)); }
    /// in place on planar host vectors; forward unscaled, reverse scaled by 1/N
    void fft(std::vector<T>& reals, std::vector<T>& imags, Direction d) const {
        check(Api<T>::any_host(raw_, reals.data(), reals.size(), imags.data(), imags.size(), (int)d));
    }
    /// `batch` transforms on device pointers, transform b at b * batch_stride; stream-ordered on `stream`
    void fft_device(T* d_reals, T* d_imags, Direction d, std::size_t batch, std::size_t batch_stride, void* stream = nullptr) const {
        check(Api<T>::any_dev(raw_, d_reals, d_imags, (int)d, batch, batch_stride, stream));
    }
    /// in place on `len` interleaved host values (len == N, else the length panic); the same results as fft()
    void fft_interleaved(std::complex<T>* signal, std::size_t len, Direction d) const {
        check(Api<T>::any_il_host(raw_, reinterpret_cast<T*>(signal), len, (int)d));
    }
    /// `batch` transforms on an interleaved device array, transform b at complex element b * batch_stride
    void fft_interleaved_device(std::complex<T>* d_signal, Direction d, std::size_t batch, std::size_t batch_stride,
                                void* stream = nullptr) const {
        check(Api<T>::any_il_dev(raw_, reinterpret_cast<T*>(d_signal), (int)d, batch, batch_stride, stream));
    }
  private:
    typename Api<T>::Any* raw_ = nullptr;
};

/// additive: real-input FFTs of any length (a power of two >= 4 runs the r2c plan; an even length up to 2^30 - 2 Bluestein of
/// N/2, an odd one up to 2^29 - 1 Bluestein of N, or with AnyAlgo::Mixed / AnyAlgo::Auto the mixed-radix path of N/2 or N when
/// that length is eligible)
template <typename T>
class PlannerR2cAny {
  public:
    explicit PlannerR2cAny(std::size_t n, int device = 0, AnyAlgo algo = AnyAlgo::Bluestein) {
        check(Api<T>::r2c_any_create(n, device, static_cast<int>(algo), &raw_));
    }
    ~PlannerR2cAny() { if (raw_) Api<T>::r2c_any_destroy(raw_); }
    PlannerR2cAny(PlannerR2cAny&& o) noexcept : raw_(o.raw_) { o.raw_ = nullptr; }
    PlannerR2cAny(const PlannerR2cAny&) = delete;
    PlannerR2cAny& operator=(const PlannerR2cAny&) = delete;
    std::size_t n() const { return Api<T>::r2c_any_size(raw_); }
    /// "power of two", or "halved" / "direct" with "Bluestein L=<L> M=2^m" or "mixed 2^a x Q_a[ x Q_b]", then the inner plan's
    /// description
    std::string describe() const { return Api<T>::r2c_any_describe(raw_); }
    /// make every allocation a call of `batch` members would make now
    void reserve(std::size_t batch) const { check(Api<T>::r2c_any_reserve(raw_, batch)); }
    /// N reals in, N/2 + 1 bins out (N/2 rounded down), forward unscaled, on host vectors
    void r2c(const std::vector<T>& input, std::vector<T>& out_re, std::vector<T>& out_im) const {
        check(Api<T>::r2c_any_host(raw_, input.data(), input.size(), out_re.data(), out_re.size(), out_im.data(), out_im.size()));
    }
    /// N/2 + 1 bins in, N reals out, scaled so that c2r(r2c(x)) == x
    void c2r(const std::vector<T>& in_re, const std::vector<T>& in_im, std::vector<T>& output) const {
        check(Api<T>::c2r_any_host(raw_, in_re.data(), in_re.size(), in_im.data(), in_im.size(), output.data(), output.size()));
    }
    /// `batch` r2c transforms on device pointers, member b at b * in_stride reals / b * out_stride bins
    void r2c_batch_dev(const T* d_in, std::size_t in_stride, T* d_out_re, T* d_out_im, std::size_t out_stride, std::size_t batch,
                       void* stream = nullptr) const {
        check(Api<T>::r2c_any_dev(raw_, d_in, in_stride, d_out_re, d_out_im, out_stride, batch, stream));
    }
    /// `batch` c2r transforms on device pointers, member b at b * in_stride bins / b * out_stride reals
    void c2r_batch_dev(const T* d_in_re, const T* d_in_im, std::size_t in_stride, T* d_out, std::size_t out_stride, std::size_t batch,
                       void* stream = nullptr) const {
        check(Api<T>::c2r_any_dev(raw_, d_in_re, d_in_im, in_stride, d_out, out_stride, batch, stream));
    }
    /// r2c() with the N/2 + 1 bins as one interleaved host vector (its size the length checked); the planar call's results
    void r2c_interleaved(const std::vector<T>& input, std::vector<std::complex<T>>& output) const {
        check(Api<T>::r2c_il_host(raw_, input.data(), input.size(), reinterpret_cast<T*>(output.data()), output.size()));
    }
    /// c2r() from one interleaved host vector of N/2 + 1 bins
    void c2r_interleaved(const std::vector<std::complex<T>>& input, std::vector<T>& output) const {
        check(Api<T>::c2r_il_host(raw_, reinterpret_cast<const T*>(input.data()), input.size(), output.data(), output.size()));
    }
    /// `batch` r2c transforms on device pointers, member b at b * in_stride reals / complex element b * out_stride
    void r2c_interleaved_device(const T* d_in, std::size_t in_stride, std::complex<T>* d_out, std::size_t out_stride, std::size_t batch,
                                void* stream = nullptr) const {
        check(Api<T>::r2c_il_dev(raw_, d_in, in_stride, reinterpret_cast<T*>(d_out), out_stride, batch, stream));
    }
    /// `batch` c2r transforms on device pointers, member b at complex element b * in_stride / b * out_stride reals
    void c2r_interleaved_device(const std::complex<T>* d_in, std::size_t in_stride, T* d_out, std::size_t out_stride, std::size_t batch,
                                void* stream = nullptr) const {
        check(Api<T>::c2r_il_dev(raw_, reinterpret_cast<const T*>(d_in), in_stride, d_out, out_stride, batch, stream));
    }
  private:
    typename Api<T>::R2cAny* raw_ = nullptr;
};

/// additive: DCT / DST types 2 and 3 of any length with scipy.fft's definitions and norms, over an N-point real plan built with
/// `algo`; R2rKind::Dct3 with the inverse norm is scipy's idct of type 2
enum class R2rKind : int { Dct2 = PHASTFT_R2R_DCT2, Dct3 = PHASTFT_R2R_DCT3, Dst2 = PHASTFT_R2R_DST2, Dst3 = PHASTFT_R2R_DST3 };
enum class R2rNorm : int { Backward = PHASTFT_NORM_BACKWARD, Ortho = PHASTFT_NORM_ORTHO, Forward = PHASTFT_NORM_FORWARD };
template <typename T>
class PlannerDct {
  public:
    explicit PlannerDct(std::size_t n, int device = 0, AnyAlgo algo = AnyAlgo::Auto) {
        check(Api<T>::dct_create(n, device, static_cast<int>(algo), &raw_));
    }
    ~PlannerDct() { if (raw_) Api<T>::dct_destroy(raw_); }
    PlannerDct(PlannerDct&& o) noexcept : raw_(o.raw_) { o.raw_ = nullptr; }
    PlannerDct(const PlannerDct&) = delete;
    PlannerDct& operator=(const PlannerDct&) = delete;
    std::size_t n() const { return Api<T>::dct_size(raw_); }
    /// "n=<N> <prec> dct | " followed by the inner real plan's description
    std::string describe() const { return Api<T>::dct_describe(raw_); }
    /// make every allocation a call of `batch` members would make now
    void reserve(std::size_t batch) const { check(Api<T>::dct_reserve(raw_, batch)); }
    /// N reals in, N out, on host vectors (`output` may be `input`)
    void transform(R2rKind kind, R2rNorm norm, const std::vector<T>& input, std::vector<T>& output) const {
        check(Api<T>::dct_host(raw_, static_cast<int>(kind), static_cast<int>(norm), input.data(), input.size(), output.data(), output.size()));
    }
    /// `batch` transforms on device pointers, member b at b * in_stride / b * out_stride (strides >= N, any offsets)
    void transform_device(R2rKind kind, R2rNorm norm, const T* d_in, std::size_t in_stride, T* d_out, std::size_t out_stride,
                          std::size_t batch, void* stream = nullptr) const {
        check(Api<T>::dct_dev(raw_, static_cast<int>(kind), static_cast<int>(norm), d_in, in_stride, d_out, out_stride, batch, stream));
    }
  private:
    typename Api<T>::Dct* raw_ = nullptr;
};

/// additive: linear convolution and cross-correlation (scipy.signal.fftconvolve / correlate) of n_x values with n_h values,
/// real or complex, over an L-point transform, L = 2^ceil(log2(n_x + n_h - 1)) but at least 4
enum class ConvMode : int { Full = PHASTFT_CONV_FULL, Same = PHASTFT_CONV_SAME, Valid = PHASTFT_CONV_VALID };
inline std::size_t conv_out_len(std::size_t n_x, std::size_t n_h, ConvMode mode) { return phastft_conv_out_len(n_x, n_h, static_cast<int>(mode)); }
template <typename T>
class PlannerConv {
  public:
    /// `complex_domain`: the operands are std::complex<T> (interleaved (re, im) pairs)
    PlannerConv(std::size_t n_x, std::size_t n_h, int device = 0, bool complex_domain = false) : n_x_(n_x), n_h_(n_h), cplx_(complex_domain) {
        check(Api<T>::conv_create(n_x, n_h, complex_domain ? PHASTFT_CONV_COMPLEX : PHASTFT_CONV_REAL, device, &raw_));
    }
    ~PlannerConv() { if (raw_) Api<T>::conv_destroy(raw_); }
    PlannerConv(PlannerConv&& o) noexcept : raw_(o.raw_), n_x_(o.n_x_), n_h_(o.n_h_), cplx_(o.cplx_) { o.raw_ = nullptr; }
    PlannerConv(const PlannerConv&) = delete;
    PlannerConv& operator=(const PlannerConv&) = delete;
    std::size_t n_x() const { return n_x_; }
    std::size_t n_h() const { return n_h_; }
    bool complex_domain() const { return cplx_; }
    std::size_t fft_len() const { return Api<T>::conv_fft_len(raw_); }
    std::size_t out_len(ConvMode mode) const { return conv_out_len(n_x_, n_h_, mode); }
    /// "n_x=<n_x> n_h=<n_h> <prec> conv <real|complex> L=2^<k> | " followed by the inner plan's description
    std::string describe() const { return Api<T>::conv_describe(raw_); }
    /// make every allocation a call of `batch` pairwise members would make now
    void reserve(std::size_t batch) const { check(Api<T>::conv_reserve(raw_, batch)); }
    /// real operands on host vectors: y gets the mode's window (y.size() == out_len(mode)).  Throws Panic on a length
    /// mismatch, and when the planner was built for complex operands (the library would read and write twice the vectors).
    void convolve(const std::vector<T>& x, const std::vector<T>& h, std::vector<T>& y, ConvMode mode = ConvMode::Full) const {
        check_domain(false);
        check(Api<T>::conv_host(raw_, PHASTFT_CONV_CONVOLVE, static_cast<int>(mode), x.data(), x.size(), h.data(), h.size(), y.data(), y.size()));
    }
    void correlate(const std::vector<T>& x, const std::vector<T>& h, std::vector<T>& y, ConvMode mode = ConvMode::Full) const {
        check_domain(false);
        check(Api<T>::conv_host(raw_, PHASTFT_CONV_CORRELATE, static_cast<int>(mode), x.data(), x.size(), h.data(), h.size(), y.data(), y.size()));
    }
    /// complex operands on host vectors; throws Panic when the planner was built for real operands
    void convolve(const std::vector<std::complex<T>>& x, const std::vector<std::complex<T>>& h, std::vector<std::complex<T>>& y,
                  ConvMode mode = ConvMode::Full) const {
        check_domain(true);
        check(Api<T>::conv_host(raw_, PHASTFT_CONV_CONVOLVE, static_cast<int>(mode), reinterpret_cast<const T*>(x.data()), x.size(),
                                reinterpret_cast<const T*>(h.data()), h.size(), reinterpret_cast<T*>(y.data()), y.size()));
    }
    void correlate(const std::vector<std::complex<T>>& x, const std::vector<std::complex<T>>& h, std::vector<std::complex<T>>& y,
                   ConvMode mode = ConvMode::Full) const {
        check_domain(true);
        check(Api<T>::conv_host(raw_, PHASTFT_CONV_CORRELATE, static_cast<int>(mode), reinterpret_cast<const T*>(x.data()), x.size(),
                                reinterpret_cast<const T*>(h.data()), h.size(), reinterpret_cast<T*>(y.data()), y.size()));
    }
    /// `batch` members on device pointers: x at b * x_stride, h at b * h_stride (0: one filter), y at b * y_stride, in values
    /// (complex ones, as T pairs aligned to 2 * sizeof(T), for a complex plan)
    void convolve_device(const T* d_x, std::size_t x_stride, const T* d_h, std::size_t h_stride, T* d_y, std::size_t y_stride,
                         std::size_t batch, ConvMode mode = ConvMode::Full, void* stream = nullptr) const {
        check(Api<T>::conv_dev(raw_, PHASTFT_CONV_CONVOLVE, static_cast<int>(mode), d_x, x_stride, d_h, h_stride, d_y, y_stride, batch, stream));
    }
    void correlate_device(const T* d_x, std::size_t x_stride, const T* d_h, std::size_t h_stride, T* d_y, std::size_t y_stride,
                          std::size_t batch, ConvMode mode = ConvMode::Full, void* stream = nullptr) const {
        check(Api<T>::conv_dev(raw_, PHASTFT_CONV_CORRELATE, static_cast<int>(mode), d_x, x_stride, d_h, h_stride, d_y, y_stride, batch, stream));
    }
  private:
    // the host entry counts lengths in values of the planner's domain, so vectors of the other domain must not reach it
    void check_domain(bool complex_operands) const {
        if (complex_operands != cplx_)
            throw Panic(PHASTFT_ERR_INVALID_ARG, std::string("PlannerConv domain mismatch: the planner was built for ") +
                                                     (cplx_ ? "complex" : "real") + " operands, the vectors are " +
                                                     (complex_operands ? "complex" : "real"));
    }
    typename Api<T>::Conv* raw_ = nullptr;
    std::size_t n_x_ = 0, n_h_ = 0;
    bool cplx_ = false;
};

/// additive: the short-time Fourier transform and its inverse (torch.stft(..., return_complex=True) / torch.istft(..., length=n))
/// of signals of n values, real or complex, over the n_fft-point plan: frames hop apart, the window's win_length values (empty:
/// ones) centred in n_fft, and with `center` n_fft / 2 values of reflect or zero padding on each side
enum class StftPad : int { Reflect = PHASTFT_STFT_PAD_REFLECT, Constant = PHASTFT_STFT_PAD_CONSTANT };
template <typename T>
class PlannerStft {
  public:
    /// `window` of win_length values, or empty for ones of win_length (0: n_fft); `complex_domain`: the signals are
    /// std::complex<T> and the frames two-sided
    PlannerStft(std::size_t n, std::size_t n_fft, std::size_t hop, const std::vector<T>& window = {}, std::size_t win_length = 0,
                bool center = true, StftPad pad = StftPad::Reflect, int device = 0, bool complex_domain = false)
        : n_(n), cplx_(complex_domain) {
        const std::size_t wl = window.empty() ? (win_length ? win_length : n_fft) : window.size();
        check(Api<T>::stft_create(n, n_fft, hop, window.empty() ? nullptr : window.data(), wl, center ? 1 : 0, static_cast<int>(pad),
                                  complex_domain ? PHASTFT_STFT_COMPLEX : PHASTFT_STFT_REAL, device, &raw_));
    }
    ~PlannerStft() { if (raw_) Api<T>::stft_destroy(raw_); }
    PlannerStft(PlannerStft&& o) noexcept : raw_(o.raw_), n_(o.n_), cplx_(o.cplx_) { o.raw_ = nullptr; }
    PlannerStft(const PlannerStft&) = delete;
    PlannerStft& operator=(const PlannerStft&) = delete;
    std::size_t n() const { return n_; }
    bool complex_domain() const { return cplx_; }
    std::size_t frames() const { return Api<T>::stft_frames(raw_); }
    std::size_t bins() const { return Api<T>::stft_bins(raw_); }
    /// "n=<n> n_fft=<n_fft> hop=<hop> <prec> stft <real|complex> F=<F> | " followed by the inner plan's description
    std::string describe() const { return Api<T>::stft_describe(raw_); }
    /// make every allocation a call of `batch` signals would make now
    void reserve(std::size_t batch) const { check(Api<T>::stft_reserve(raw_, batch)); }
    /// real signal on host vectors: spec gets frames() x bins() values, frame-major (spec.size() == frames() * bins()).
    /// Throws Panic on a length mismatch, and when the planner was built for complex signals.
    void stft(const std::vector<T>& x, std::vector<std::complex<T>>& spec, bool normalized = false) const {
        check_domain(false);
        check(Api<T>::stft_host(raw_, normalized, x.data(), x.size(), reinterpret_cast<T*>(spec.data()), spec.size()));
    }
    void stft(const std::vector<std::complex<T>>& x, std::vector<std::complex<T>>& spec, bool normalized = false) const {
        check_domain(true);
        check(Api<T>::stft_host(raw_, normalized, reinterpret_cast<const T*>(x.data()), x.size(), reinterpret_cast<T*>(spec.data()),
                                spec.size()));
    }
    /// the inverse of frame-major frames() x bins() values into n() values
    void istft(const std::vector<std::complex<T>>& spec, std::vector<T>& y, bool normalized = false) const {
        check_domain(false);
        check(Api<T>::istft_host(raw_, normalized, reinterpret_cast<const T*>(spec.data()), spec.size(), y.data(), y.size()));
    }
    void istft(const std::vector<std::complex<T>>& spec, std::vector<std::complex<T>>& y, bool normalized = false) const {
        check_domain(true);
        check(Api<T>::istft_host(raw_, normalized, reinterpret_cast<const T*>(spec.data()), spec.size(), reinterpret_cast<T*>(y.data()),
                                 y.size()));
    }
    /// `batch` signals on device pointers: member b at d_x + b * x_stride values (complex ones, as T pairs aligned to
    /// 2 * sizeof(T), for a complex planner), frame f of member b at d_spec + (b * frames() + f) * frame_stride complex values
    void stft_device(const T* d_x, std::size_t x_stride, T* d_spec, std::size_t frame_stride, std::size_t batch, bool normalized = false,
                     void* stream = nullptr) const {
        check(Api<T>::stft_dev(raw_, normalized, d_x, x_stride, d_spec, frame_stride, batch, stream));
    }
    void istft_device(const T* d_spec, std::size_t frame_stride, T* d_y, std::size_t y_stride, std::size_t batch, bool normalized = false,
                      void* stream = nullptr) const {
        check(Api<T>::istft_dev(raw_, normalized, d_spec, frame_stride, d_y, y_stride, batch, stream));
    }
  private:
    // the host entry counts signal lengths in values of the planner's domain, so vectors of the other domain must not reach it
    void check_domain(bool complex_signal) const {
        if (complex_signal != cplx_)
            throw Panic(PHASTFT_ERR_INVALID_ARG, std::string("PlannerStft domain mismatch: the planner was built for ") +
                                                     (cplx_ ? "complex" : "real") + " signals, the vector is " +
                                                     (complex_signal ? "complex" : "real"));
    }
    typename Api<T>::Stft* raw_ = nullptr;
    std::size_t n_ = 0;
    bool cplx_ = false;
};
}  // namespace detail

using PlannerDit64 = detail::PlannerDit<double>;
using PlannerDit32 = detail::PlannerDit<float>;
using PlannerR2c64 = detail::PlannerR2c<double>;
using PlannerR2c32 = detail::PlannerR2c<float>;
using AnyAlgo = detail::AnyAlgo;
using PlannerAny64 = detail::PlannerAny<double>;
using PlannerAny32 = detail::PlannerAny<float>;
using PlannerR2cAny64 = detail::PlannerR2cAny<double>;
using PlannerR2cAny32 = detail::PlannerR2cAny<float>;
using R2rKind = detail::R2rKind;
using R2rNorm = detail::R2rNorm;
using PlannerDct64 = detail::PlannerDct<double>;
using PlannerDct32 = detail::PlannerDct<float>;
using ConvMode = detail::ConvMode;
using PlannerConv64 = detail::PlannerConv<double>;
using PlannerConv32 = detail::PlannerConv<float>;
using detail::conv_out_len;
using StftPad = detail::StftPad;
using PlannerStft64 = detail::PlannerStft<double>;
using PlannerStft32 = detail::PlannerStft<float>;

// ---- c2c (lib.rs:143-226, algorithms/dit.rs:263,338): in place on planar vectors -----------------------
inline void fft_64_dit_with_planner_and_opts(std::vector<double>& reals, std::vector<double>& imags, Direction d, const PlannerDit64& p, const Options&) {
    check(detail::Api<double>::fft_host(p.raw(), reals.data(), reals.size(), imags.data(), imags.size(), (int)d));
}
inline void fft_64_dit_with_planner(std::vector<double>& reals, std::vector<double>& imags, Direction d, const PlannerDit64& p) {
    fft_64_dit_with_planner_and_opts(reals, imags, d, p, Options::guess_options(reals.size()));
}
inline void fft_64_dit(std::vector<double>& reals, std::vector<double>& imags, Direction d) {
    // lib.rs:181: a planner per call; the library keeps the latest one for the next same-size call
    check(phastft_fft_dit_f64_oneshot(reals.data(), reals.size(), imags.data(), imags.size(), (int)d, 0));
}
inline void fft_32_dit_with_planner_and_opts(std::vector<float>& reals, std::vector<float>& imags, Direction d, const PlannerDit32& p, const Options&) {
    check(detail::Api<float>::fft_host(p.raw(), reals.data(), reals.size(), imags.data(), imags.size(), (int)d));
}
inline void fft_32_dit_with_planner(std::vector<float>& reals, std::vector<float>& imags, Direction d, const PlannerDit32& p) {
    fft_32_dit_with_planner_and_opts(reals, imags, d, p, Options::guess_options(reals.size()));
}
inline void fft_32_dit(std::vector<float>& reals, std::vector<float>& imags, Direction d) {
    check(phastft_fft_dit_f32_oneshot(reals.data(), reals.size(), imags.data(), imags.size(), (int)d, 0));
}

// ---- additive: batches and device-resident data (the reference's batch is a caller loop sharing one planner,
// examples/benchmark.rs:24-36; here it is one call) -------------------------------------------------------------
template <typename T>
inline void fft_dit_batch(std::vector<T>& reals, std::vector<T>& imags, Direction d, const detail::PlannerDit<T>& p, std::size_t batch, std::size_t batch_stride) {
    if (reals.size() != imags.size()) check(1);
    const std::size_t n = p.num_points();
    if (batch_stride < n || (batch && reals.size() < (batch - 1) * batch_stride + n)) check(13);
    typename detail::Api<T>::Dit* one[1] = {p.raw_mut()};
    check(detail::Api<T>::fft_batch_host(one, 1, reals.data(), imags.data(), batch, batch_stride, (int)d));
}
inline void fft_64_dit_batch(std::vector<double>& re, std::vector<double>& im, Direction d, const PlannerDit64& p, std::size_t batch, std::size_t stride) { fft_dit_batch<double>(re, im, d, p, batch, stride); }
inline void fft_32_dit_batch(std::vector<float>& re, std::vector<float>& im, Direction d, const PlannerDit32& p, std::size_t batch, std::size_t stride) { fft_dit_batch<float>(re, im, d, p, batch, stride); }
/// Device pointers on the planner's device; stream-ordered on `stream` (cudaStream_t, nullptr = default stream), no allocation, no host sync.
inline void fft_64_dit_device(double* d_reals, double* d_imags, Direction d, const PlannerDit64& p, std::size_t batch, std::size_t batch_stride, void* stream) {
    check(detail::Api<double>::fft_dev(p.raw(), d_reals, d_imags, (int)d, batch, batch_stride, stream));
}
inline void fft_32_dit_device(float* d_reals, float* d_imags, Direction d, const PlannerDit32& p, std::size_t batch, std::size_t batch_stride, void* stream) {
    check(detail::Api<float>::fft_dev(p.raw(), d_reals, d_imags, (int)d, batch, batch_stride, stream));
}

// ---- r2c / c2r (algorithms/r2c.rs:521-895) --------------------------------------------------------------
inline void r2c_fft_f64_with_planner(const std::vector<double>& in, std::vector<double>& ore, std::vector<double>& oim, const PlannerR2c64& p) {
    check(detail::Api<double>::r2c_host(p.raw(), in.data(), in.size(), ore.data(), ore.size(), oim.data(), oim.size()));
}
inline void r2c_fft_f64(const std::vector<double>& in, std::vector<double>& ore, std::vector<double>& oim) {
    // r2c.rs:522: a planner per call; the library keeps the latest one for the next same-size call
    check(detail::Api<double>::r2c_oneshot(in.data(), in.size(), ore.data(), ore.size(), oim.data(), oim.size()));
}
inline void c2r_fft_f64_with_planner_and_scratch(const std::vector<double>& ire, const std::vector<double>& iim, std::vector<double>& out,
                                                 const PlannerR2c64& p, std::vector<double>& sre, std::vector<double>& sim) {
    check(detail::Api<double>::c2r_host(p.raw(), ire.data(), ire.size(), iim.data(), iim.size(), out.data(), out.size(), sre.data(), sre.size(), sim.data(), sim.size()));
}
inline void c2r_fft_f64_with_planner(const std::vector<double>& ire, const std::vector<double>& iim, std::vector<double>& out, const PlannerR2c64& p) {
    check(detail::Api<double>::c2r_host(p.raw(), ire.data(), ire.size(), iim.data(), iim.size(), out.data(), out.size(), nullptr, 0, nullptr, 0));
}
inline void c2r_fft_f64(const std::vector<double>& ire, const std::vector<double>& iim, std::vector<double>& out) {
    check(detail::Api<double>::c2r_oneshot(ire.data(), ire.size(), iim.data(), iim.size(), out.data(), out.size()));
}
inline void r2c_fft_f32_with_planner(const std::vector<float>& in, std::vector<float>& ore, std::vector<float>& oim, const PlannerR2c32& p) {
    check(detail::Api<float>::r2c_host(p.raw(), in.data(), in.size(), ore.data(), ore.size(), oim.data(), oim.size()));
}
inline void r2c_fft_f32(const std::vector<float>& in, std::vector<float>& ore, std::vector<float>& oim) {
    check(detail::Api<float>::r2c_oneshot(in.data(), in.size(), ore.data(), ore.size(), oim.data(), oim.size()));
}
inline void c2r_fft_f32_with_planner_and_scratch(const std::vector<float>& ire, const std::vector<float>& iim, std::vector<float>& out,
                                                 const PlannerR2c32& p, std::vector<float>& sre, std::vector<float>& sim) {
    check(detail::Api<float>::c2r_host(p.raw(), ire.data(), ire.size(), iim.data(), iim.size(), out.data(), out.size(), sre.data(), sre.size(), sim.data(), sim.size()));
}
inline void c2r_fft_f32_with_planner(const std::vector<float>& ire, const std::vector<float>& iim, std::vector<float>& out, const PlannerR2c32& p) {
    check(detail::Api<float>::c2r_host(p.raw(), ire.data(), ire.size(), iim.data(), iim.size(), out.data(), out.size(), nullptr, 0, nullptr, 0));
}
inline void c2r_fft_f32(const std::vector<float>& ire, const std::vector<float>& iim, std::vector<float>& out) {
    check(detail::Api<float>::c2r_oneshot(ire.data(), ire.size(), iim.data(), iim.size(), out.data(), out.size()));
}

}  // namespace phastft
