//! PhastFT's public API, unchanged, over `libphastft_cuda.so` (H100 / sm_90a).
//!
//! Every item below keeps the name, signature and panic behaviour of the reference crate
//! (QuState/PhastFT @ 8cd3a39; the `file:line` in each doc comment is the item it replaces), so a user
//! switches by changing the dependency, not the call sites:
//!
//! ```ignore
//! use phastft::{fft_64_dit, planner::Direction};
//! let mut reals = vec![1.0, 0.0, 0.0, 0.0];
//! let mut imags = vec![0.0; 4];
//! fft_64_dit(&mut reals, &mut imags, Direction::Forward);   // runs on cuda:0
//! ```
//!
//! The wrappers are deliberately thin: length checks that the reference performs with `assert!` happen
//! inside the C ABI, which returns a status code; `check()` turns a non-zero code back into a `panic!`
//! carrying the reference's message, so `#[should_panic(expected = "...")]` tests carry over.
//! The device is chosen with the `PHASTFT_DEVICE` environment variable (default 0).
pub mod ffi;
pub mod options;
pub mod planner;

use options::Options;
use planner::{Direction, PlannerAny32, PlannerAny64, PlannerConv32, PlannerConv64, PlannerDit32, PlannerDit64, PlannerDct32, PlannerDct64,
              PlannerR2c32, PlannerR2c64, PlannerR2cAny32, PlannerR2cAny64, PlannerStft32, PlannerStft64};

/// Reference panic texts by status code (include/phastft_status.h).
#[track_caller]
pub(crate) fn check(code: i32) {
    let msg = match code {
        0 => return,
        1 => "assertion `left == right` failed: reals.len() == imags.len()",
        2 => "assertion failed: length must be a non-zero power of two",
        3 => "assertion `left == right` failed: log_n == planner.log_n",
        4 => "n must be a power of 2 >= 4",
        5 => "input length must match planner size",
        6 => "output_re must have length N/2 + 1",
        7 => "output_im must have length N/2 + 1",
        8 => "output length must match planner size",
        9 => "input_re must have length N/2 + 1",
        10 => "input_im must have length N/2 + 1",
        11 => "scratch_re must have length N/2",
        12 => "scratch_im must have length N/2",
        _ => {
            let detail = unsafe { std::ffi::CStr::from_ptr(ffi::phastft_last_error()) }.to_string_lossy().into_owned();
            panic!("phastft_cuda error {code}: {detail}");
        }
    };
    panic!("{msg}");
}

/// Page-lock a long-lived buffer so the host-slice calls copy at full PCIe speed (~52 GB/s instead of ~13 GB/s
/// from pageable memory). Additive: the reference has no analogue. Undo with [`host_unregister`] before the
/// buffer is freed.
pub fn host_register<T>(buf: &mut [T]) {
    check(unsafe { ffi::phastft_host_register(buf.as_mut_ptr() as *mut std::os::raw::c_void, std::mem::size_of_val(buf)) });
}
pub fn host_unregister<T>(buf: &mut [T]) {
    check(unsafe { ffi::phastft_host_unregister(buf.as_mut_ptr() as *mut std::os::raw::c_void) });
}

pub(crate) fn device() -> i32 {
    std::env::var("PHASTFT_DEVICE").ok().and_then(|s| s.parse().ok()).unwrap_or(0)
}

fn c_opts(o: &Options) -> ffi::phastft_options {
    ffi::phastft_options {
        multithreaded_bit_reversal: o.multithreaded_bit_reversal as i32,
        smallest_parallel_chunk_size: o.smallest_parallel_chunk_size,
    }
}

// ------------------------------------------------------------------------------------------------
// c2c, planar
// ------------------------------------------------------------------------------------------------

/// `algorithms/dit.rs:263` -- in place on planar slices; panics like the reference on length
/// mismatch, non-power-of-two length, or a planner built for another size.
pub fn fft_64_dit_with_planner_and_opts(reals: &mut [f64], imags: &mut [f64], direction: Direction, planner: &PlannerDit64, opts: &Options) {
    let o = c_opts(opts);
    check(unsafe {
        ffi::phastft_fft_dit_f64_host(planner.raw, reals.as_mut_ptr(), reals.len(), imags.as_mut_ptr(), imags.len(), direction as i32, &o)
    });
}

/// `algorithms/dit.rs:338`
pub fn fft_32_dit_with_planner_and_opts(reals: &mut [f32], imags: &mut [f32], direction: Direction, planner: &PlannerDit32, opts: &Options) {
    let o = c_opts(opts);
    check(unsafe {
        ffi::phastft_fft_dit_f32_host(planner.raw, reals.as_mut_ptr(), reals.len(), imags.as_mut_ptr(), imags.len(), direction as i32, &o)
    });
}

/// `lib.rs:143`
pub fn fft_64_dit_with_planner(reals: &mut [f64], imags: &mut [f64], direction: Direction, planner: &PlannerDit64) {
    let opts = Options::guess_options(reals.len());
    fft_64_dit_with_planner_and_opts(reals, imags, direction, planner, &opts);
}

/// `lib.rs:180` -- plans per call, like the reference.
pub fn fft_64_dit(reals: &mut [f64], imags: &mut [f64], direction: Direction) {
    // a planner per call, as in the reference; the library keeps the latest one for the next same-size call
    check(unsafe {
        ffi::phastft_fft_dit_f64_oneshot(reals.as_mut_ptr(), reals.len(), imags.as_mut_ptr(), imags.len(), direction as i32, device())
    });
}

/// `lib.rs:186`
pub fn fft_32_dit_with_planner(reals: &mut [f32], imags: &mut [f32], direction: Direction, planner: &PlannerDit32) {
    let opts = Options::guess_options(reals.len());
    fft_32_dit_with_planner_and_opts(reals, imags, direction, planner, &opts);
}

/// `lib.rs:223`
pub fn fft_32_dit(reals: &mut [f32], imags: &mut [f32], direction: Direction) {
    check(unsafe {
        ffi::phastft_fft_dit_f32_oneshot(reals.as_mut_ptr(), reals.len(), imags.as_mut_ptr(), imags.len(), direction as i32, device())
    });
}

// ------------------------------------------------------------------------------------------------
// Additive: batches and device-resident data.  The reference has no batch API -- a batch is a caller loop sharing one
// planner (examples/benchmark.rs:24-36); on a GPU the loop is one call, and the data can stay in device memory.
// ------------------------------------------------------------------------------------------------

macro_rules! impl_batch {
    ($batch:ident, $sharded:ident, $device:ident, $t:ty, $planner:ident, $ffi_sharded:ident, $ffi_dev:ident) => {
        /// `batch` transforms of `planner.num_points()` points, transform `b` at `[b * batch_stride ..][.. n]` of the planar
        /// host slices, in place; equivalent to calling the `_with_planner` function on every transform.  Host memory is
        /// streamed through a three-slot H2D / FFT / D2H pipeline (page-lock it with [`host_register`] for full PCIe speed).
        pub fn $batch(reals: &mut [$t], imags: &mut [$t], direction: Direction, planner: &$planner, batch: usize, batch_stride: usize) {
            $sharded(reals, imags, direction, &[planner], batch, batch_stride);
        }
        /// The same batch sharded over several devices from one process: transforms `[g*batch/G, (g+1)*batch/G)` run on
        /// `planners[g]` (one planner per device).  No data-path collective.
        pub fn $sharded(reals: &mut [$t], imags: &mut [$t], direction: Direction, planners: &[&$planner], batch: usize, batch_stride: usize) {
            assert!(!planners.is_empty(), "at least one planner");
            let n = planners[0].num_points();
            assert_eq!(reals.len(), imags.len(), "reals.len() == imags.len()");
            assert!(batch_stride >= n && (batch == 0 || reals.len() >= (batch - 1) * batch_stride + n), "slices shorter than batch * batch_stride");
            let raw: Vec<*mut _> = planners.iter().map(|p| p.raw).collect();
            check(unsafe { ffi::$ffi_sharded(raw.as_ptr(), raw.len() as i32, reals.as_mut_ptr(), imags.as_mut_ptr(), batch, batch_stride, direction as i32) });
        }
        /// Device-resident planar data: stream-ordered on `stream` (a `cudaStream_t`, null = the default stream), no
        /// allocation, no host synchronisation.
        ///
        /// # Safety
        /// `d_reals` / `d_imags` must be device pointers valid for `(batch - 1) * batch_stride + n` elements on the
        /// planner's device, and must not be used by other work on other streams until this call's work has completed.
        pub unsafe fn $device(d_reals: *mut $t, d_imags: *mut $t, direction: Direction, planner: &$planner, batch: usize, batch_stride: usize,
                              stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_dev(planner.raw, d_reals, d_imags, direction as i32, batch, batch_stride, stream));
        }
    };
}
impl_batch!(fft_64_dit_batch, fft_64_dit_batch_sharded, fft_64_dit_device, f64, PlannerDit64, phastft_fft_dit_f64_batch_sharded_host, phastft_fft_dit_f64_dev);
impl_batch!(fft_32_dit_batch, fft_32_dit_batch_sharded, fft_32_dit_device, f32, PlannerDit32, phastft_fft_dit_f32_batch_sharded_host, phastft_fft_dit_f32_dev);

/// Number of CUDA devices the library sees (0 without a driver; every transform then panics with the NO_DEVICE message).
pub fn device_count() -> usize {
    let mut n: std::os::raw::c_int = 0;
    unsafe { ffi::phastft_device_count(&mut n) };
    n.max(0) as usize
}

/// Device-resident real transforms (`r2c.rs:535`, `:740` on device pointers).
///
/// # Safety
/// Device pointers on the planner's device: `d_input` N reals, `d_out_*` N/2 + 1 each.
pub unsafe fn r2c_fft_f64_device(d_input: *const f64, d_out_re: *mut f64, d_out_im: *mut f64, planner: &PlannerR2c64, stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_r2c_f64_dev(planner.raw, d_input, d_out_re, d_out_im, stream));
}
/// # Safety
/// As [`r2c_fft_f64_device`]; `d_scratch_*` are N/2 each or both null (the plan's own scratch is then used).
pub unsafe fn c2r_fft_f64_device(d_in_re: *const f64, d_in_im: *const f64, d_output: *mut f64, planner: &PlannerR2c64,
                                 d_scratch_re: *mut f64, d_scratch_im: *mut f64, stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_c2r_f64_dev(planner.raw, d_in_re, d_in_im, d_output, d_scratch_re, d_scratch_im, stream));
}
/// # Safety
/// As [`r2c_fft_f64_device`].
pub unsafe fn r2c_fft_f32_device(d_input: *const f32, d_out_re: *mut f32, d_out_im: *mut f32, planner: &PlannerR2c32, stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_r2c_f32_dev(planner.raw, d_input, d_out_re, d_out_im, stream));
}
/// # Safety
/// Additive: `batch` r2c transforms in one call.  Member b reads N reals at `d_input + b * in_stride` (in_stride >= N, even)
/// and writes N/2 + 1 bins at `d_out_* + b * out_stride` (out_stride >= N/2 + 1).  Batch 1 is [`r2c_fft_f64_device`].
pub unsafe fn r2c_fft_f64_device_batch(d_input: *const f64, in_stride: usize, d_out_re: *mut f64, d_out_im: *mut f64, out_stride: usize,
                                       batch: usize, planner: &PlannerR2c64, stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_r2c_f64_batch_dev(planner.raw, d_input, in_stride, d_out_re, d_out_im, out_stride, batch, stream));
}

/// Additive: `batch` c2r transforms in one call.  Member b reads N/2 + 1 bins at `d_in_* + b * in_stride` (in_stride >= N/2 + 1)
/// and writes N reals at `d_output + b * out_stride` (out_stride >= N, even); `d_scratch_*` hold batch * N/2 each, dense, or are
/// both null (the plan's own scratch).  Batch 1 is [`c2r_fft_f64_device`].
pub unsafe fn c2r_fft_f64_device_batch(d_in_re: *const f64, d_in_im: *const f64, in_stride: usize, d_output: *mut f64, out_stride: usize,
                                       batch: usize, planner: &PlannerR2c64, d_scratch_re: *mut f64, d_scratch_im: *mut f64,
                                       stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_c2r_f64_batch_dev(planner.raw, d_in_re, d_in_im, in_stride, d_output, out_stride, d_scratch_re, d_scratch_im,
                                         batch, stream));
}

/// As [`r2c_fft_f64_device_batch`].
pub unsafe fn r2c_fft_f32_device_batch(d_input: *const f32, in_stride: usize, d_out_re: *mut f32, d_out_im: *mut f32, out_stride: usize,
                                       batch: usize, planner: &PlannerR2c32, stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_r2c_f32_batch_dev(planner.raw, d_input, in_stride, d_out_re, d_out_im, out_stride, batch, stream));
}

/// As [`c2r_fft_f64_device_batch`].
pub unsafe fn c2r_fft_f32_device_batch(d_in_re: *const f32, d_in_im: *const f32, in_stride: usize, d_output: *mut f32, out_stride: usize,
                                       batch: usize, planner: &PlannerR2c32, d_scratch_re: *mut f32, d_scratch_im: *mut f32,
                                       stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_c2r_f32_batch_dev(planner.raw, d_in_re, d_in_im, in_stride, d_output, out_stride, d_scratch_re, d_scratch_im,
                                         batch, stream));
}

/// As [`c2r_fft_f64_device`].
pub unsafe fn c2r_fft_f32_device(d_in_re: *const f32, d_in_im: *const f32, d_output: *mut f32, planner: &PlannerR2c32,
                                 d_scratch_re: *mut f32, d_scratch_im: *mut f32, stream: *mut std::os::raw::c_void) {
    check(ffi::phastft_c2r_f32_dev(planner.raw, d_in_re, d_in_im, d_output, d_scratch_re, d_scratch_im, stream));
}

// ------------------------------------------------------------------------------------------------
// Additive: complex FFTs of any length (the reference accepts powers of two only)
// ------------------------------------------------------------------------------------------------
macro_rules! impl_any {
    ($with_planner:ident, $device_batch:ident, $t:ty, $planner:ident, $ffi_host:ident, $ffi_dev:ident) => {
        /// In place on planar host slices of `planner.num_points()` points, any length; forward unscaled, reverse scaled by
        /// 1/N.  Panics on a length mismatch or a planner built for another size.
        pub fn $with_planner(reals: &mut [$t], imags: &mut [$t], direction: Direction, planner: &$planner) {
            check(unsafe { ffi::$ffi_host(planner.raw, reals.as_mut_ptr(), reals.len(), imags.as_mut_ptr(), imags.len(), direction as i32) });
        }
        /// Device-resident planar data, `batch` transforms at `b * batch_stride` (batch_stride >= N), stream-ordered on
        /// `stream`; allocates only when the plan's workspace must grow (see `reserve`).
        ///
        /// # Safety
        /// `d_reals` / `d_imags` must be device pointers valid for `(batch - 1) * batch_stride + n` elements on the
        /// planner's device, and must not be used by other work on other streams until this call's work has completed.
        pub unsafe fn $device_batch(d_reals: *mut $t, d_imags: *mut $t, direction: Direction, planner: &$planner, batch: usize,
                                    batch_stride: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_dev(planner.raw, d_reals, d_imags, direction as i32, batch, batch_stride, stream));
        }
    };
}
impl_any!(fft_64_any_with_planner, fft_64_any_device_batch, f64, PlannerAny64, phastft_fft_any_f64_host, phastft_fft_any_f64_dev);
impl_any!(fft_32_any_with_planner, fft_32_any_device_batch, f32, PlannerAny32, phastft_fft_any_f32_host, phastft_fft_any_f32_dev);

// ------------------------------------------------------------------------------------------------
// Additive: real-input FFTs of any length (the reference's r2c / c2r accept powers of two >= 4 only)
// ------------------------------------------------------------------------------------------------
macro_rules! impl_r2c_any {
    ($r2c:ident, $c2r:ident, $r2c_dev:ident, $c2r_dev:ident, $t:ty, $planner:ident, $ffi_r2c_host:ident, $ffi_c2r_host:ident,
     $ffi_r2c_dev:ident, $ffi_c2r_dev:ident) => {
        /// `planner.n()` reals in, `n / 2 + 1` bins out (rounded down), forward unscaled.  Panics on a length mismatch.
        pub fn $r2c(input: &[$t], output_re: &mut [$t], output_im: &mut [$t], planner: &$planner) {
            check(unsafe { ffi::$ffi_r2c_host(planner.raw, input.as_ptr(), input.len(), output_re.as_mut_ptr(), output_re.len(),
                                              output_im.as_mut_ptr(), output_im.len()) });
        }
        /// `n / 2 + 1` bins in, `planner.n()` reals out, scaled so that c2r(r2c(x)) == x.  Panics on a length mismatch.
        pub fn $c2r(input_re: &[$t], input_im: &[$t], output: &mut [$t], planner: &$planner) {
            check(unsafe { ffi::$ffi_c2r_host(planner.raw, input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(),
                                              output.as_mut_ptr(), output.len()) });
        }
        /// `batch` r2c transforms on device data: member b reads n reals at `d_input + b * in_stride` and writes the bins at
        /// `b * out_stride`; stream-ordered on `stream`.
        ///
        /// # Safety
        /// The pointers must be device pointers valid for the members on the planner's device, and for even n the input must
        /// be aligned to two elements with an even `in_stride`.
        pub unsafe fn $r2c_dev(d_input: *const $t, in_stride: usize, d_out_re: *mut $t, d_out_im: *mut $t, out_stride: usize,
                               planner: &$planner, batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_r2c_dev(planner.raw, d_input, in_stride, d_out_re, d_out_im, out_stride, batch, stream));
        }
        /// `batch` c2r transforms on device data, the mirror of the r2c call.
        ///
        /// # Safety
        /// As for the r2c call, with the alignment rule on the output.
        pub unsafe fn $c2r_dev(d_in_re: *const $t, d_in_im: *const $t, in_stride: usize, d_output: *mut $t, out_stride: usize,
                               planner: &$planner, batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_c2r_dev(planner.raw, d_in_re, d_in_im, in_stride, d_output, out_stride, batch, stream));
        }
    };
}
impl_r2c_any!(r2c_fft_f64_any_with_planner, c2r_fft_f64_any_with_planner, r2c_fft_f64_any_device_batch, c2r_fft_f64_any_device_batch,
              f64, PlannerR2cAny64, phastft_r2c_any_f64_host, phastft_c2r_any_f64_host, phastft_r2c_any_f64_dev, phastft_c2r_any_f64_dev);
impl_r2c_any!(r2c_fft_f32_any_with_planner, c2r_fft_f32_any_with_planner, r2c_fft_f32_any_device_batch, c2r_fft_f32_any_device_batch,
              f32, PlannerR2cAny32, phastft_r2c_any_f32_host, phastft_c2r_any_f32_host, phastft_r2c_any_f32_dev, phastft_c2r_any_f32_dev);

// ------------------------------------------------------------------------------------------------
// Additive: DCT / DST types 2 and 3 of any length (scipy.fft.dct / dst)
// ------------------------------------------------------------------------------------------------
/// The transforms of `PlannerDct*`, with scipy.fft's definitions; `Dct3` with the inverse norm is scipy's idct of type 2.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(i32)]
pub enum R2rKind {
    Dct2 = 0,
    Dct3 = 1,
    Dst2 = 2,
    Dst3 = 3,
}
/// scipy.fft's `norm`: no scale, 1/sqrt(2N) with the orthogonalising factor on the first (DCT) or last (DST) element, or 1/(2N).
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(i32)]
pub enum R2rNorm {
    Backward = 0,
    Ortho = 1,
    Forward = 2,
}
macro_rules! impl_dct {
    ($host:ident, $dev:ident, $t:ty, $planner:ident, $ffi_host:ident, $ffi_dev:ident) => {
        /// `planner.n()` reals in, as many out.  Panics on a length mismatch.
        pub fn $host(kind: R2rKind, norm: R2rNorm, input: &[$t], output: &mut [$t], planner: &$planner) {
            check(unsafe { ffi::$ffi_host(planner.raw, kind as i32, norm as i32, input.as_ptr(), input.len(), output.as_mut_ptr(),
                                          output.len()) });
        }
        /// `batch` transforms on device data: member b reads n reals at `d_in + b * in_stride` and writes n at
        /// `d_out + b * out_stride` (any strides >= n and offsets; `d_out == d_in` with equal strides in place), stream-ordered.
        ///
        /// # Safety
        /// The pointers must be device pointers valid for the members on the planner's device.
        pub unsafe fn $dev(kind: R2rKind, norm: R2rNorm, d_in: *const $t, in_stride: usize, d_out: *mut $t, out_stride: usize,
                           planner: &$planner, batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_dev(planner.raw, kind as i32, norm as i32, d_in, in_stride, d_out, out_stride, batch, stream));
        }
    };
}
impl_dct!(dct_f64_with_planner, dct_f64_device_batch, f64, PlannerDct64, phastft_dct_f64_host, phastft_dct_f64_dev);
impl_dct!(dct_f32_with_planner, dct_f32_device_batch, f32, PlannerDct32, phastft_dct_f32_host, phastft_dct_f32_dev);

// ------------------------------------------------------------------------------------------------
// Additive: linear convolution and cross-correlation (scipy.signal.fftconvolve / correlate)
// ------------------------------------------------------------------------------------------------
/// The output window of `PlannerConv*`: the whole linear convolution (n_x + n_h - 1 values), its centre n_x values from
/// (n_h - 1) / 2, or the |n_x - n_h| + 1 values that need no zero padding, from min(n_x, n_h) - 1.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(i32)]
pub enum ConvMode {
    Full = 0,
    Same = 1,
    Valid = 2,
}
const CONV_CONVOLVE: i32 = 0;
const CONV_CORRELATE: i32 = 1;
/// The safe host functions pass slice lengths in values of the slice's element type, and the library reads and writes as many
/// values of the planner's domain: a real slice given to a complex planner would be overrun, a complex one given to a real
/// planner misread.  So they panic on a domain mismatch before any call.
#[track_caller]
fn check_conv_domain(planner_complex: bool, slices_complex: bool) {
    if planner_complex != slices_complex {
        panic!("PlannerConv domain mismatch: the planner was built for {} operands, the slices are {}",
               if planner_complex { "complex" } else { "real" }, if slices_complex { "complex" } else { "real" });
    }
}
macro_rules! impl_conv {
    ($conv:ident, $corr:ident, $conv_dev:ident, $corr_dev:ident, $t:ty, $planner:ident, $ffi_host:ident, $ffi_dev:ident) => {
        /// Real operands of a real planner: `y` gets the window of `mode` of x * h.  Panics on a length mismatch, and when
        /// the planner was built for complex operands.
        pub fn $conv(x: &[$t], h: &[$t], y: &mut [$t], mode: ConvMode, planner: &$planner) {
            check_conv_domain(planner.is_complex(), false);
            check(unsafe { ffi::$ffi_host(planner.raw, CONV_CONVOLVE, mode as i32, x.as_ptr(), x.len(), h.as_ptr(), h.len(),
                                          y.as_mut_ptr(), y.len()) });
        }
        /// The cross-correlation of x with h (convolution with h reversed), as the convolution, with its panics.
        pub fn $corr(x: &[$t], h: &[$t], y: &mut [$t], mode: ConvMode, planner: &$planner) {
            check_conv_domain(planner.is_complex(), false);
            check(unsafe { ffi::$ffi_host(planner.raw, CONV_CORRELATE, mode as i32, x.as_ptr(), x.len(), h.as_ptr(), h.len(),
                                          y.as_mut_ptr(), y.len()) });
        }
        /// `batch` convolutions on device data: member b reads x at `d_x + b * x_stride`, h at `d_h + b * h_stride`
        /// (`h_stride == 0`: one filter for every member) and writes the window at `d_y + b * y_stride`, stream-ordered.
        /// Strides count values (complex ones, as `$t` pairs aligned to their size, for a complex planner).
        ///
        /// # Safety
        /// The pointers must be device pointers valid for the members on the planner's device, counted in values of the
        /// planner's domain (two `$t` per value for a complex planner).
        pub unsafe fn $conv_dev(d_x: *const $t, x_stride: usize, d_h: *const $t, h_stride: usize, d_y: *mut $t, y_stride: usize,
                                mode: ConvMode, planner: &$planner, batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_dev(planner.raw, CONV_CONVOLVE, mode as i32, d_x, x_stride, d_h, h_stride, d_y, y_stride, batch, stream));
        }
        /// The cross-correlation form of the device batch.
        ///
        /// # Safety
        /// As for the convolution.
        pub unsafe fn $corr_dev(d_x: *const $t, x_stride: usize, d_h: *const $t, h_stride: usize, d_y: *mut $t, y_stride: usize,
                                mode: ConvMode, planner: &$planner, batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$ffi_dev(planner.raw, CONV_CORRELATE, mode as i32, d_x, x_stride, d_h, h_stride, d_y, y_stride, batch, stream));
        }
    };
}
impl_conv!(convolve_f64_with_planner, correlate_f64_with_planner, convolve_f64_device_batch, correlate_f64_device_batch, f64,
           PlannerConv64, phastft_conv_f64_host, phastft_conv_f64_dev);
impl_conv!(convolve_f32_with_planner, correlate_f32_with_planner, convolve_f32_device_batch, correlate_f32_device_batch, f32,
           PlannerConv32, phastft_conv_f32_host, phastft_conv_f32_dev);

// ------------------------------------------------------------------------------------------------
// Additive: the short-time Fourier transform and its inverse (torch.stft / torch.istft)
// ------------------------------------------------------------------------------------------------
/// The safe host functions pass slice lengths in values of the slice's element type, and the library reads and writes as many
/// values of the planner's domain, so they panic on a domain mismatch before any call (as the convolution's do).
#[track_caller]
fn check_stft_domain(planner_complex: bool, signal_complex: bool) {
    if planner_complex != signal_complex {
        panic!("PlannerStft domain mismatch: the planner was built for {} signals, the slice is {}",
               if planner_complex { "complex" } else { "real" }, if signal_complex { "complex" } else { "real" });
    }
}
macro_rules! impl_stft {
    ($stft:ident, $istft:ident, $stft_dev:ident, $istft_dev:ident, $t:ty, $planner:ident, $host_f:ident, $host_i:ident, $dev_f:ident,
     $dev_i:ident) => {
        /// Real signal of a real planner: `spec` gets `frames() * bins()` interleaved (re, im) pairs as `$t` (`2 *` that
        /// many values), frame-major.  Panics on a length mismatch, and when the planner was built for complex signals.
        pub fn $stft(x: &[$t], spec: &mut [$t], normalized: bool, planner: &$planner) {
            check_stft_domain(planner.is_complex(), false);
            check(unsafe { ffi::$host_f(planner.raw, normalized as i32, x.as_ptr(), x.len(), spec.as_mut_ptr(), spec.len() / 2) });
        }
        /// The inverse of a real planner's frame-major spectrum into `n()` reals, with the forward form's panics.
        pub fn $istft(spec: &[$t], y: &mut [$t], normalized: bool, planner: &$planner) {
            check_stft_domain(planner.is_complex(), false);
            check(unsafe { ffi::$host_i(planner.raw, normalized as i32, spec.as_ptr(), spec.len() / 2, y.as_mut_ptr(), y.len()) });
        }
        /// `batch` signals on device data: member b reads `n()` values at `d_x + b * x_stride` and frame f of it goes to
        /// `d_spec + (b * frames() + f) * frame_stride` complex values, stream-ordered.
        ///
        /// # Safety
        /// The pointers must be device pointers valid for the members on the planner's device, counted in values of the
        /// planner's domain (two `$t` per value for a complex planner), `d_spec` aligned to `2 * size_of::<$t>()`.
        pub unsafe fn $stft_dev(d_x: *const $t, x_stride: usize, d_spec: *mut $t, frame_stride: usize, normalized: bool, planner: &$planner,
                                batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$dev_f(planner.raw, normalized as i32, d_x, x_stride, d_spec, frame_stride, batch, stream));
        }
        /// The inverse device batch: frames at `d_spec + (b * frames() + f) * frame_stride`, signals at `d_y + b * y_stride`.
        ///
        /// # Safety
        /// As for the forward form.
        pub unsafe fn $istft_dev(d_spec: *const $t, frame_stride: usize, d_y: *mut $t, y_stride: usize, normalized: bool, planner: &$planner,
                                 batch: usize, stream: *mut std::os::raw::c_void) {
            check(ffi::$dev_i(planner.raw, normalized as i32, d_spec, frame_stride, d_y, y_stride, batch, stream));
        }
    };
}
impl_stft!(stft_f64_with_planner, istft_f64_with_planner, stft_f64_device_batch, istft_f64_device_batch, f64, PlannerStft64,
           phastft_stft_f64_host, phastft_istft_f64_host, phastft_stft_f64_dev, phastft_istft_f64_dev);
impl_stft!(stft_f32_with_planner, istft_f32_with_planner, stft_f32_device_batch, istft_f32_device_batch, f32, PlannerStft32,
           phastft_stft_f32_host, phastft_istft_f32_host, phastft_stft_f32_dev, phastft_istft_f32_dev);

// ------------------------------------------------------------------------------------------------
// r2c / c2r  (algorithms/r2c.rs:521-895)
// ------------------------------------------------------------------------------------------------

/// `r2c.rs:535`
pub fn r2c_fft_f64_with_planner(input_re: &[f64], output_re: &mut [f64], output_im: &mut [f64], planner: &PlannerR2c64) {
    check(unsafe {
        ffi::phastft_r2c_f64_host(planner.raw, input_re.as_ptr(), input_re.len(), output_re.as_mut_ptr(), output_re.len(),
                                  output_im.as_mut_ptr(), output_im.len())
    });
}

/// `r2c.rs:521`
pub fn r2c_fft_f64(input_re: &[f64], output_re: &mut [f64], output_im: &mut [f64]) {
    // a planner per call, as in the reference; the library keeps the latest one for the next same-size call
    check(unsafe {
        ffi::phastft_r2c_f64_oneshot(input_re.as_ptr(), input_re.len(), output_re.as_mut_ptr(), output_re.len(),
                                     output_im.as_mut_ptr(), output_im.len(), device())
    });
}

/// `r2c.rs:607`
pub fn r2c_fft_f32_with_planner(input_re: &[f32], output_re: &mut [f32], output_im: &mut [f32], planner: &PlannerR2c32) {
    check(unsafe {
        ffi::phastft_r2c_f32_host(planner.raw, input_re.as_ptr(), input_re.len(), output_re.as_mut_ptr(), output_re.len(),
                                  output_im.as_mut_ptr(), output_im.len())
    });
}

/// `r2c.rs:598`
pub fn r2c_fft_f32(input_re: &[f32], output_re: &mut [f32], output_im: &mut [f32]) {
    check(unsafe {
        ffi::phastft_r2c_f32_oneshot(input_re.as_ptr(), input_re.len(), output_re.as_mut_ptr(), output_re.len(),
                                     output_im.as_mut_ptr(), output_im.len(), device())
    });
}

/// `r2c.rs:740` -- caller scratch is length-checked like the reference; the work happens in device memory.
pub fn c2r_fft_f64_with_planner_and_scratch(input_re: &[f64], input_im: &[f64], output: &mut [f64], planner: &PlannerR2c64,
                                            scratch_re: &mut [f64], scratch_im: &mut [f64]) {
    check(unsafe {
        ffi::phastft_c2r_f64_host(planner.raw, input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(),
                                  output.as_mut_ptr(), output.len(), scratch_re.as_mut_ptr(), scratch_re.len(),
                                  scratch_im.as_mut_ptr(), scratch_im.len())
    });
}

/// `r2c.rs:708` -- the reference allocates two N/2 Vecs here; the CUDA plan owns device scratch instead.
pub fn c2r_fft_f64_with_planner(input_re: &[f64], input_im: &[f64], output: &mut [f64], planner: &PlannerR2c64) {
    check(unsafe {
        ffi::phastft_c2r_f64_host(planner.raw, input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(),
                                  output.as_mut_ptr(), output.len(), std::ptr::null_mut(), 0, std::ptr::null_mut(), 0)
    });
}

/// `r2c.rs:695`
pub fn c2r_fft_f64(input_re: &[f64], input_im: &[f64], output: &mut [f64]) {
    check(unsafe {
        ffi::phastft_c2r_f64_oneshot(input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(), output.as_mut_ptr(), output.len(), device())
    });
}

/// `r2c.rs:835`
pub fn c2r_fft_f32_with_planner_and_scratch(input_re: &[f32], input_im: &[f32], output: &mut [f32], planner: &PlannerR2c32,
                                            scratch_re: &mut [f32], scratch_im: &mut [f32]) {
    check(unsafe {
        ffi::phastft_c2r_f32_host(planner.raw, input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(),
                                  output.as_mut_ptr(), output.len(), scratch_re.as_mut_ptr(), scratch_re.len(),
                                  scratch_im.as_mut_ptr(), scratch_im.len())
    });
}

/// `r2c.rs:813`
pub fn c2r_fft_f32_with_planner(input_re: &[f32], input_im: &[f32], output: &mut [f32], planner: &PlannerR2c32) {
    check(unsafe {
        ffi::phastft_c2r_f32_host(planner.raw, input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(),
                                  output.as_mut_ptr(), output.len(), std::ptr::null_mut(), 0, std::ptr::null_mut(), 0)
    });
}

/// `r2c.rs:804`
pub fn c2r_fft_f32(input_re: &[f32], input_im: &[f32], output: &mut [f32]) {
    check(unsafe {
        ffi::phastft_c2r_f32_oneshot(input_re.as_ptr(), input_re.len(), input_im.as_ptr(), input_im.len(), output.as_mut_ptr(), output.len(), device())
    });
}

// ------------------------------------------------------------------------------------------------
// interleaved Complex<T> API (lib.rs:41-140, feature `complex-nums`)
// ------------------------------------------------------------------------------------------------
#[cfg(feature = "complex-nums")]
mod interleaved {
    use super::*;
    use num_complex::Complex;

    /// `lib.rs:41-60`: the reference deinterleaves into two Vecs, transforms, re-interleaves; here the
    /// AoS <-> planar conversion is fused into the first pass's load and the last pass's store.
    pub fn fft_64_interleaved_with_planner_and_opts(signal: &mut [Complex<f64>], direction: Direction, planner: &PlannerDit64, _opts: &Options) {
        check(unsafe { ffi::phastft_fft_interleaved_f64_host(planner.raw, signal.as_mut_ptr() as *mut f64, signal.len(), direction as i32) });
    }
    pub fn fft_32_interleaved_with_planner_and_opts(signal: &mut [Complex<f32>], direction: Direction, planner: &PlannerDit32, _opts: &Options) {
        check(unsafe { ffi::phastft_fft_interleaved_f32_host(planner.raw, signal.as_mut_ptr() as *mut f32, signal.len(), direction as i32) });
    }
    /// `lib.rs:77-97`
    pub fn fft_64_interleaved_with_planner(signal: &mut [Complex<f64>], direction: Direction, planner: &PlannerDit64) {
        let opts = Options::guess_options(signal.len());
        fft_64_interleaved_with_planner_and_opts(signal, direction, planner, &opts);
    }
    pub fn fft_32_interleaved_with_planner(signal: &mut [Complex<f32>], direction: Direction, planner: &PlannerDit32) {
        let opts = Options::guess_options(signal.len());
        fft_32_interleaved_with_planner_and_opts(signal, direction, planner, &opts);
    }
    /// `lib.rs:113-140`
    pub fn fft_64_interleaved(signal: &mut [Complex<f64>], direction: Direction) {
        let planner = PlannerDit64::new(signal.len());
        fft_64_interleaved_with_planner(signal, direction, &planner);
    }
    pub fn fft_32_interleaved(signal: &mut [Complex<f32>], direction: Direction) {
        let planner = PlannerDit32::new(signal.len());
        fft_32_interleaved_with_planner(signal, direction, &planner);
    }

    // Additive: interleaved transforms of any length on the any-length planners
    macro_rules! impl_interleaved_any {
        ($with_planner:ident, $device_batch:ident, $t:ty, $planner:ident, $ffi_host:ident, $ffi_dev:ident) => {
            /// In place on `planner.num_points()` interleaved host values, any length; forward unscaled, reverse scaled by 1/N.
            /// Bluestein and mixed-radix plans give the planar call's results bit for bit.  Panics on a length mismatch.
            pub fn $with_planner(signal: &mut [Complex<$t>], direction: Direction, planner: &$planner) {
                check(unsafe { ffi::$ffi_host(planner.raw, signal.as_mut_ptr() as *mut $t, signal.len(), direction as i32) });
            }
            /// Device-resident interleaved data, `batch` transforms at complex element `b * batch_stride` (batch_stride >= N),
            /// stream-ordered on `stream`; allocates only when the plan's workspace must grow (see `reserve`).
            ///
            /// # Safety
            /// `d_signal` must be a device pointer, aligned to `Complex<T>`, valid for `(batch - 1) * batch_stride + n` complex
            /// values on the planner's device, and must not be used by other work on other streams until this call's work has
            /// completed.
            pub unsafe fn $device_batch(d_signal: *mut Complex<$t>, direction: Direction, planner: &$planner, batch: usize,
                                        batch_stride: usize, stream: *mut std::os::raw::c_void) {
                check(ffi::$ffi_dev(planner.raw, d_signal as *mut $t, direction as i32, batch, batch_stride, stream));
            }
        };
    }
    impl_interleaved_any!(fft_64_interleaved_any_with_planner, fft_64_interleaved_any_device_batch, f64, PlannerAny64,
                          phastft_fft_interleaved_any_f64_host, phastft_fft_interleaved_any_f64_dev);
    impl_interleaved_any!(fft_32_interleaved_any_with_planner, fft_32_interleaved_any_device_batch, f32, PlannerAny32,
                          phastft_fft_interleaved_any_f32_host, phastft_fft_interleaved_any_f32_dev);

    // Additive: real transforms of any length with the spectrum as interleaved bins
    macro_rules! impl_real_interleaved_any {
        ($r2c:ident, $c2r:ident, $r2c_dev:ident, $c2r_dev:ident, $t:ty, $planner:ident, $ffi_r2c_host:ident, $ffi_c2r_host:ident,
         $ffi_r2c_dev:ident, $ffi_c2r_dev:ident) => {
            /// N reals in, the floor(N/2) + 1 bins out as `Complex<T>`, forward unscaled; the planar call's results bit for bit.
            /// Panics on a length mismatch.
            pub fn $r2c(input: &[$t], output: &mut [Complex<$t>], planner: &$planner) {
                check(unsafe { ffi::$ffi_r2c_host(planner.raw, input.as_ptr(), input.len(), output.as_mut_ptr() as *mut $t, output.len()) });
            }
            /// floor(N/2) + 1 `Complex<T>` bins in, N reals out, scaled so that c2r(r2c(x)) == x; the input is not written.
            pub fn $c2r(input: &[Complex<$t>], output: &mut [$t], planner: &$planner) {
                check(unsafe { ffi::$ffi_c2r_host(planner.raw, input.as_ptr() as *const $t, input.len(), output.as_mut_ptr(), output.len()) });
            }
            /// Device-resident: member b reads N reals at `d_input + b * in_stride` and writes its bins at complex element
            /// `b * out_stride` of `d_out`, stream-ordered on `stream`.
            ///
            /// # Safety
            /// Both pointers must be device pointers on the planner's device, valid for `batch` members at those strides
            /// (`d_out` aligned to `Complex<T>`; for even N `d_input` aligned to 2 * size_of::<T>() and `in_stride` even), and
            /// must not be used by other work on other streams until this call's work has completed.
            pub unsafe fn $r2c_dev(d_input: *const $t, in_stride: usize, d_out: *mut Complex<$t>, out_stride: usize, planner: &$planner,
                                   batch: usize, stream: *mut std::os::raw::c_void) {
                check(ffi::$ffi_r2c_dev(planner.raw, d_input, in_stride, d_out as *mut $t, out_stride, batch, stream));
            }
            /// The mirror of the r2c batch: member b reads its bins at complex element `b * in_stride` of `d_in` and writes N
            /// reals at `d_output + b * out_stride`.
            ///
            /// # Safety
            /// As the r2c batch, with `d_in` aligned to `Complex<T>` and, for even N, `d_output` pair-aligned with an even stride.
            pub unsafe fn $c2r_dev(d_in: *const Complex<$t>, in_stride: usize, d_output: *mut $t, out_stride: usize, planner: &$planner,
                                   batch: usize, stream: *mut std::os::raw::c_void) {
                check(ffi::$ffi_c2r_dev(planner.raw, d_in as *const $t, in_stride, d_output, out_stride, batch, stream));
            }
        };
    }
    impl_real_interleaved_any!(r2c_fft_f64_interleaved_any_with_planner, c2r_fft_f64_interleaved_any_with_planner,
                               r2c_fft_f64_interleaved_any_device_batch, c2r_fft_f64_interleaved_any_device_batch, f64, PlannerR2cAny64,
                               phastft_r2c_interleaved_any_f64_host, phastft_c2r_interleaved_any_f64_host,
                               phastft_r2c_interleaved_any_f64_dev, phastft_c2r_interleaved_any_f64_dev);
    impl_real_interleaved_any!(r2c_fft_f32_interleaved_any_with_planner, c2r_fft_f32_interleaved_any_with_planner,
                               r2c_fft_f32_interleaved_any_device_batch, c2r_fft_f32_interleaved_any_device_batch, f32, PlannerR2cAny32,
                               phastft_r2c_interleaved_any_f32_host, phastft_c2r_interleaved_any_f32_host,
                               phastft_r2c_interleaved_any_f32_dev, phastft_c2r_interleaved_any_f32_dev);

    macro_rules! impl_conv_complex {
        ($conv:ident, $corr:ident, $t:ty, $planner:ident, $ffi_host:ident) => {
            /// Complex operands of a complex planner: `y` gets the window of `mode` of x * h.  Panics on a length mismatch,
            /// and when the planner was built for real operands.
            pub fn $conv(x: &[Complex<$t>], h: &[Complex<$t>], y: &mut [Complex<$t>], mode: ConvMode, planner: &$planner) {
                check_conv_domain(planner.is_complex(), true);
                check(unsafe { ffi::$ffi_host(planner.raw, CONV_CONVOLVE, mode as i32, x.as_ptr() as *const $t, x.len(),
                                              h.as_ptr() as *const $t, h.len(), y.as_mut_ptr() as *mut $t, y.len()) });
            }
            /// The cross-correlation of x with h (convolution with conj(h) reversed), as the convolution, with its panics.
            pub fn $corr(x: &[Complex<$t>], h: &[Complex<$t>], y: &mut [Complex<$t>], mode: ConvMode, planner: &$planner) {
                check_conv_domain(planner.is_complex(), true);
                check(unsafe { ffi::$ffi_host(planner.raw, CONV_CORRELATE, mode as i32, x.as_ptr() as *const $t, x.len(),
                                              h.as_ptr() as *const $t, h.len(), y.as_mut_ptr() as *mut $t, y.len()) });
            }
        };
    }
    impl_conv_complex!(convolve_complex_f64_with_planner, correlate_complex_f64_with_planner, f64, PlannerConv64, phastft_conv_f64_host);
    impl_conv_complex!(convolve_complex_f32_with_planner, correlate_complex_f32_with_planner, f32, PlannerConv32, phastft_conv_f32_host);

    macro_rules! impl_stft_complex {
        ($stft:ident, $istft:ident, $t:ty, $planner:ident, $host_f:ident, $host_i:ident) => {
            /// Real or complex signal: `spec` gets `frames() * bins()` bins, frame-major.  Panics on a length mismatch, and
            /// when the signal's domain is not the planner's.
            pub fn $stft(x: &[Complex<$t>], spec: &mut [Complex<$t>], normalized: bool, planner: &$planner) {
                check_stft_domain(planner.is_complex(), true);
                check(unsafe { ffi::$host_f(planner.raw, normalized as i32, x.as_ptr() as *const $t, x.len(), spec.as_mut_ptr() as *mut $t,
                                            spec.len()) });
            }
            /// The inverse of a complex planner's frame-major spectrum into `n()` complex values, with the forward form's panics.
            pub fn $istft(spec: &[Complex<$t>], y: &mut [Complex<$t>], normalized: bool, planner: &$planner) {
                check_stft_domain(planner.is_complex(), true);
                check(unsafe { ffi::$host_i(planner.raw, normalized as i32, spec.as_ptr() as *const $t, spec.len(), y.as_mut_ptr() as *mut $t,
                                            y.len()) });
            }
        };
    }
    impl_stft_complex!(stft_complex_f64_with_planner, istft_complex_f64_with_planner, f64, PlannerStft64, phastft_stft_f64_host,
                       phastft_istft_f64_host);
    impl_stft_complex!(stft_complex_f32_with_planner, istft_complex_f32_with_planner, f32, PlannerStft32, phastft_stft_f32_host,
                       phastft_istft_f32_host);
}
#[cfg(feature = "complex-nums")]
pub use interleaved::*;
