//! `planner.rs` of the reference: `Direction`, `PlannerMode`, `PlannerDit{64,32}`, `PlannerR2c{64,32}`.
//! The planners own an opaque handle to the CUDA plan (device twiddle tables, workspace, stream) and free
//! it on drop.  They stay `Send + Sync` like the reference's (plain `Vec` fields there): the C library
//! serialises workspace use inside the plan.
use crate::{check, device, ffi};

/// `planner.rs:10-16`
#[derive(Copy, Clone)]
pub enum Direction {
    Forward = 1,
    Reverse = -1,
}

/// `planner.rs:25-32`.  The reference accepts the mode and ignores it (`planner.rs:65`); here `Tune` is real: the
/// planner builds a handful of pass decompositions / tile widths around the heuristic one, times them on the device
/// and keeps the fastest.
#[derive(Copy, Clone, Debug, Default)]
pub enum PlannerMode {
    #[default]
    Heuristic,
    Tune,
}

macro_rules! impl_planner_dit {
    ($name:ident, $raw:ty, $create:ident, $destroy:ident, $size:ident, $describe:ident, $reserve:ident) => {
        pub struct $name {
            pub(crate) raw: *mut $raw,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// `planner.rs:55`: panics unless `num_points` is a non-zero power of two.
            pub fn new(num_points: usize) -> Self {
                Self::with_mode(num_points, PlannerMode::Heuristic)
            }
            /// `planner.rs:65`
            pub fn with_mode(num_points: usize, mode: PlannerMode) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create(num_points, device(), mode as i32, &mut raw) });
                Self { raw }
            }
            /// Number of points the planner was built for.
            pub fn num_points(&self) -> usize {
                unsafe { ffi::$size(self.raw) }
            }
            /// Additive: the pass decomposition and kernels the planner chose, e.g.
            /// `"n=2^20 f64: COL R=1024(32x32) C=8 NT=256 | TRANS R=1024(32x32) C=8 NT=256"`.
            pub fn describe(&self) -> String {
                unsafe { std::ffi::CStr::from_ptr(ffi::$describe(self.raw)) }.to_string_lossy().into_owned()
            }
            /// Additive: size the device workspace for calls of up to `batch` transforms now (otherwise the first larger
            /// batched call grows it, synchronising the device).
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_dit!(PlannerDit64, ffi::phastft_plan_dit_f64, phastft_plan_dit_f64_create, phastft_plan_dit_f64_destroy,
                  phastft_plan_dit_f64_size, phastft_plan_dit_f64_describe, phastft_plan_dit_f64_reserve);
impl_planner_dit!(PlannerDit32, ffi::phastft_plan_dit_f32, phastft_plan_dit_f32_create, phastft_plan_dit_f32_destroy,
                  phastft_plan_dit_f32_size, phastft_plan_dit_f32_describe, phastft_plan_dit_f32_reserve);

macro_rules! impl_planner_r2c {
    ($name:ident, $raw:ty, $create:ident, $destroy:ident, $reserve:ident) => {
        pub struct $name {
            pub(crate) raw: *mut $raw,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// `planner.rs:194`: panics with "n must be a power of 2 >= 4".
            pub fn new(n: usize) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create(n, device(), &mut raw) });
                Self { raw }
            }
            /// Additive: makes every allocation a batched call of `batch` transforms would make (the inner plan's workspace,
            /// the plan's c2r scratch when that batch takes the separate sweep), so such calls can be captured in a CUDA graph.
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_r2c!(PlannerR2c64, ffi::phastft_plan_r2c_f64, phastft_plan_r2c_f64_create, phastft_plan_r2c_f64_destroy,
                  phastft_plan_r2c_f64_reserve);
impl_planner_r2c!(PlannerR2c32, ffi::phastft_plan_r2c_f32, phastft_plan_r2c_f32_create, phastft_plan_r2c_f32_destroy,
                  phastft_plan_r2c_f32_reserve);

/// How a length that is not a power of two is transformed (`PHASTFT_ANY_*`).  `Auto` takes `Mixed` for every eligible length
/// (2^a 3^b 5^c 7^d below 2^30 whose odd part fits one or two odd passes) and `Bluestein` otherwise, from the factorisation alone.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(i32)]
pub enum AnyAlgo {
    Bluestein = 0,
    Mixed = 1,
    Auto = 2,
}

macro_rules! impl_planner_any {
    ($name:ident, $raw:ty, $create:ident, $create_with:ident, $destroy:ident, $size:ident, $describe:ident, $reserve:ident) => {
        /// Additive (the reference accepts powers of two only): a complex FFT of any length.  A power of two runs the c2c plan
        /// as it is; any other length up to 2^29 - 1 runs Bluestein's algorithm over a power-of-two plan.
        pub struct $name {
            pub(crate) raw: *mut $raw,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// Panics for `num_points == 0` or a length above 2^29 - 1 that is not a power of two.
            pub fn new(num_points: usize) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create(num_points, device(), &mut raw) });
                Self { raw }
            }
            /// `new` with the algorithm chosen.  Panics as `new` does, and for `AnyAlgo::Mixed` on a length that is not eligible.
            pub fn with_algo(num_points: usize, algo: AnyAlgo) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create_with(num_points, device(), algo as std::os::raw::c_int, &mut raw) });
                Self { raw }
            }
            /// Number of points the planner was built for.
            pub fn num_points(&self) -> usize {
                unsafe { ffi::$size(self.raw) }
            }
            /// `"n=1000 f64 any: Bluestein M=2^11 | inner: ..."`, `"n=1000 f64 any: mixed 2^3 x 125 | inner: ..."` or `"n=2^20 f64 any: power of two | inner: ..."`.
            pub fn describe(&self) -> String {
                unsafe { std::ffi::CStr::from_ptr(ffi::$describe(self.raw)) }.to_string_lossy().into_owned()
            }
            /// Makes every allocation a call of `batch` transforms would make, so such calls can be captured in a CUDA graph.
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_any!(PlannerAny64, ffi::phastft_plan_any_f64, phastft_plan_any_f64_create, phastft_plan_any_f64_create_with, phastft_plan_any_f64_destroy,
                  phastft_plan_any_f64_size, phastft_plan_any_f64_describe, phastft_plan_any_f64_reserve);
impl_planner_any!(PlannerAny32, ffi::phastft_plan_any_f32, phastft_plan_any_f32_create, phastft_plan_any_f32_create_with, phastft_plan_any_f32_destroy,
                  phastft_plan_any_f32_size, phastft_plan_any_f32_describe, phastft_plan_any_f32_reserve);

macro_rules! impl_planner_r2c_any {
    ($name:ident, $raw:ty, $create:ident, $create_with:ident, $destroy:ident, $size:ident, $describe:ident, $reserve:ident) => {
        /// Additive (the reference's r2c accepts powers of two >= 4 only): real-input FFTs of any length.  A power of two
        /// from 4 runs the r2c plan as it is; an even length up to 2^30 - 2 runs Bluestein's algorithm on N/2 complex
        /// points, an odd one up to 2^29 - 1 on N.  `with_algo` selects the mixed-radix path of N/2 or N instead.
        pub struct $name {
            pub(crate) raw: *mut $raw,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// Panics for `n == 0` or a length above the limits.
            pub fn new(n: usize) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create(n, device(), &mut raw) });
                Self { raw }
            }
            /// `new` with the algorithm chosen (`Mixed` / `Auto`: the mixed-radix path of N/2 for even N up to 2^31 - 2, of N for
            /// odd N, when that length is eligible).  Panics as `new` does, and for `AnyAlgo::Mixed` on a length that is not eligible.
            pub fn with_algo(n: usize, algo: AnyAlgo) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create_with(n, device(), algo as std::os::raw::c_int, &mut raw) });
                Self { raw }
            }
            /// Number of real points the planner was built for.
            pub fn n(&self) -> usize {
                unsafe { ffi::$size(self.raw) }
            }
            /// `"n=44100 f64 r2c any: halved, Bluestein L=22050 M=2^16 | inner: ..."`, `"... halved, mixed 2^1 x 105 x 105 | ..."`,
            /// `"... direct, ..."` or `"n=2^20 f64 r2c any: power of two | ..."`.
            pub fn describe(&self) -> String {
                unsafe { std::ffi::CStr::from_ptr(ffi::$describe(self.raw)) }.to_string_lossy().into_owned()
            }
            /// Makes every allocation a call of `batch` members would make, so such calls can be captured in a CUDA graph.
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_r2c_any!(PlannerR2cAny64, ffi::phastft_plan_r2c_any_f64, phastft_plan_r2c_any_f64_create,
                      phastft_plan_r2c_any_f64_create_with, phastft_plan_r2c_any_f64_destroy,
                      phastft_plan_r2c_any_f64_size, phastft_plan_r2c_any_f64_describe, phastft_plan_r2c_any_f64_reserve);
impl_planner_r2c_any!(PlannerR2cAny32, ffi::phastft_plan_r2c_any_f32, phastft_plan_r2c_any_f32_create,
                      phastft_plan_r2c_any_f32_create_with, phastft_plan_r2c_any_f32_destroy,
                      phastft_plan_r2c_any_f32_size, phastft_plan_r2c_any_f32_describe, phastft_plan_r2c_any_f32_reserve);

macro_rules! impl_planner_dct {
    ($name:ident, $raw:ty, $create_with:ident, $destroy:ident, $size:ident, $describe:ident, $reserve:ident) => {
        /// Additive: DCT / DST types 2 and 3 of any length (scipy.fft.dct / dst) over an N-point real plan.
        pub struct $name {
            pub(crate) raw: *mut $raw,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// `algo` as for `PlannerR2cAny*::with_algo`, with its limits.  Panics for `n == 0` or a length above them.
            pub fn new(n: usize, algo: AnyAlgo) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create_with(n, device(), algo as std::os::raw::c_int, &mut raw) });
                Self { raw }
            }
            /// Number of points the planner was built for.
            pub fn n(&self) -> usize {
                unsafe { ffi::$size(self.raw) }
            }
            /// `"n=<N> f64 dct | "` followed by the inner real plan's describe().
            pub fn describe(&self) -> String {
                unsafe { std::ffi::CStr::from_ptr(ffi::$describe(self.raw)) }.to_string_lossy().into_owned()
            }
            /// Makes every allocation a call of `batch` members would make, so such calls can be captured in a CUDA graph.
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_dct!(PlannerDct64, ffi::phastft_plan_dct_f64, phastft_plan_dct_f64_create_with, phastft_plan_dct_f64_destroy,
                  phastft_plan_dct_f64_size, phastft_plan_dct_f64_describe, phastft_plan_dct_f64_reserve);
impl_planner_dct!(PlannerDct32, ffi::phastft_plan_dct_f32, phastft_plan_dct_f32_create_with, phastft_plan_dct_f32_destroy,
                  phastft_plan_dct_f32_size, phastft_plan_dct_f32_describe, phastft_plan_dct_f32_reserve);

macro_rules! impl_planner_conv {
    ($name:ident, $raw:ty, $create:ident, $destroy:ident, $fft_len:ident, $describe:ident, $reserve:ident) => {
        /// Additive: linear convolution and cross-correlation (scipy.signal.fftconvolve / correlate) of `n_x` values with
        /// `n_h` values, real or complex, over an L-point transform, L = 2^ceil(log2(n_x + n_h - 1)) but at least 4.
        pub struct $name {
            pub(crate) raw: *mut $raw,
            n_x: usize,
            n_h: usize,
            complex: bool,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// `complex`: the operands are interleaved complex values.  Panics for `n_x == 0`, `n_h == 0`, or L above 2^31
            /// (real) / 2^30 (complex).
            pub fn new(n_x: usize, n_h: usize, complex: bool) -> Self {
                let mut raw = std::ptr::null_mut();
                check(unsafe { ffi::$create(n_x, n_h, complex as std::os::raw::c_int, device(), &mut raw) });
                Self { raw, n_x, n_h, complex }
            }
            pub fn n_x(&self) -> usize {
                self.n_x
            }
            pub fn n_h(&self) -> usize {
                self.n_h
            }
            pub fn is_complex(&self) -> bool {
                self.complex
            }
            /// L, the length of the transforms the planner runs.
            pub fn fft_len(&self) -> usize {
                unsafe { ffi::$fft_len(self.raw) }
            }
            /// The output length of `mode`: n_x + n_h - 1, n_x or |n_x - n_h| + 1.
            pub fn out_len(&self, mode: crate::ConvMode) -> usize {
                unsafe { ffi::phastft_conv_out_len(self.n_x, self.n_h, mode as std::os::raw::c_int) }
            }
            /// `"n_x=<n_x> n_h=<n_h> f64 conv real L=2^<k> | "` followed by the inner plan's describe().
            pub fn describe(&self) -> String {
                unsafe { std::ffi::CStr::from_ptr(ffi::$describe(self.raw)) }.to_string_lossy().into_owned()
            }
            /// Makes every allocation a call of `batch` pairwise members would make, so such calls can be captured in a CUDA
            /// graph.
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_conv!(PlannerConv64, ffi::phastft_plan_conv_f64, phastft_plan_conv_f64_create, phastft_plan_conv_f64_destroy,
                   phastft_plan_conv_f64_fft_len, phastft_plan_conv_f64_describe, phastft_plan_conv_f64_reserve);
impl_planner_conv!(PlannerConv32, ffi::phastft_plan_conv_f32, phastft_plan_conv_f32_create, phastft_plan_conv_f32_destroy,
                   phastft_plan_conv_f32_fft_len, phastft_plan_conv_f32_describe, phastft_plan_conv_f32_reserve);

/// The padding of `PlannerStft*` with centring: reflection (torch's default) or zeros.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(i32)]
pub enum StftPad {
    Reflect = 0,
    Constant = 1,
}

macro_rules! impl_planner_stft {
    ($name:ident, $t:ty, $raw:ty, $create:ident, $destroy:ident, $frames:ident, $bins:ident, $describe:ident, $reserve:ident) => {
        /// Additive: the short-time Fourier transform and its inverse (torch.stft(..., return_complex=True) /
        /// torch.istft(..., length=n)) of signals of `n` values, real or complex, over the `n_fft`-point plan.
        pub struct $name {
            pub(crate) raw: *mut $raw,
            n: usize,
            complex: bool,
        }
        unsafe impl Send for $name {}
        unsafe impl Sync for $name {}
        impl $name {
            /// Frames `hop` apart; `window` holds the window's values (empty: ones of `n_fft`), centred in `n_fft`;
            /// `center` pads `n_fft / 2` values on each side with `pad`.  Panics where the library refuses the plan
            /// (hop 0, a window longer than n_fft, reflect padding of n_fft / 2 >= n, n < n_fft without centring, ...).
            pub fn new(n: usize, n_fft: usize, hop: usize, window: &[$t], center: bool, pad: StftPad, complex: bool) -> Self {
                let mut raw = std::ptr::null_mut();
                let (w, wl) = if window.is_empty() { (std::ptr::null(), n_fft) } else { (window.as_ptr(), window.len()) };
                check(unsafe {
                    ffi::$create(n, n_fft, hop, w, wl, center as std::os::raw::c_int, pad as std::os::raw::c_int,
                                 complex as std::os::raw::c_int, device(), &mut raw)
                });
                Self { raw, n, complex }
            }
            pub fn n(&self) -> usize {
                self.n
            }
            pub fn is_complex(&self) -> bool {
                self.complex
            }
            /// F, the frames per signal.
            pub fn frames(&self) -> usize {
                unsafe { ffi::$frames(self.raw) }
            }
            /// The bins per frame: n_fft / 2 + 1 (real signals) or n_fft (complex).
            pub fn bins(&self) -> usize {
                unsafe { ffi::$bins(self.raw) }
            }
            /// `"n=<n> n_fft=<n_fft> hop=<hop> f64 stft real F=<F> | "` followed by the inner plan's describe().
            pub fn describe(&self) -> String {
                unsafe { std::ffi::CStr::from_ptr(ffi::$describe(self.raw)) }.to_string_lossy().into_owned()
            }
            /// Makes every allocation a call of `batch` signals would make, so such calls can be captured in a CUDA graph.
            pub fn reserve(&self, batch: usize) {
                check(unsafe { ffi::$reserve(self.raw, batch) });
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { ffi::$destroy(self.raw) }
            }
        }
    };
}
impl_planner_stft!(PlannerStft64, f64, ffi::phastft_plan_stft_f64, phastft_plan_stft_f64_create, phastft_plan_stft_f64_destroy,
                   phastft_plan_stft_f64_frames, phastft_plan_stft_f64_bins, phastft_plan_stft_f64_describe, phastft_plan_stft_f64_reserve);
impl_planner_stft!(PlannerStft32, f32, ffi::phastft_plan_stft_f32, phastft_plan_stft_f32_create, phastft_plan_stft_f32_destroy,
                   phastft_plan_stft_f32_frames, phastft_plan_stft_f32_bins, phastft_plan_stft_f32_describe, phastft_plan_stft_f32_reserve);
