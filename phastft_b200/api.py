"""Host-side mirror of PhastFT's public API over libphastft_cuda.so.

Same names, argument meaning and error behaviour as the reference crate
(the reference's src/lib.rs:33-226, planner.rs, options.rs, algorithms/r2c.rs:521-895), so the
parity tests read like the reference's own tests:

    fft_64_dit(reals, imags, Direction.Forward)          # lib.rs:180
    planner = PlannerDit64(n); fft_64_dit_with_planner(reals, imags, Direction.Reverse, planner)
    r2c_fft_f64(x, out_re, out_im); c2r_fft_f64(out_re, out_im, y)

Arrays: numpy arrays (host slices -> `*_host` entry points: H2D, kernels, D2H, synchronous,
in place) or torch CUDA tensors (device-resident -> `*_dev` entry points on torch's current
stream, asynchronous, nothing copied).  Where the reference panics these raise `PhastFTPanic`
(an AssertionError) whose message starts with the reference's panic text.

The Rust crate that keeps the exact Rust signatures over the same C ABI is rust/src/lib.rs.
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import PhastFTPanic, check, fn

__all__ = [
    "Direction", "PlannerMode", "Options", "PhastFTPanic",
    "PlannerDit64", "PlannerDit32", "PlannerR2c64", "PlannerR2c32",
    "fft_64_dit", "fft_64_dit_with_planner", "fft_64_dit_with_planner_and_opts",
    "fft_32_dit", "fft_32_dit_with_planner", "fft_32_dit_with_planner_and_opts",
    "fft_64_interleaved", "fft_64_interleaved_with_planner", "fft_64_interleaved_with_planner_and_opts",
    "fft_32_interleaved", "fft_32_interleaved_with_planner", "fft_32_interleaved_with_planner_and_opts",
    "r2c_fft_f64", "r2c_fft_f64_with_planner", "c2r_fft_f64", "c2r_fft_f64_with_planner",
    "c2r_fft_f64_with_planner_and_scratch",
    "r2c_fft_f32", "r2c_fft_f32_with_planner", "c2r_fft_f32", "c2r_fft_f32_with_planner",
    "c2r_fft_f32_with_planner_and_scratch",
    "fft_dit_batch", "fft_dit_batch_sharded", "host_register", "host_unregister",
    "r2c_batch", "c2r_batch",
    "PlannerAny64", "PlannerAny32", "fft_64_any_with_planner", "fft_32_any_with_planner", "fft_any_batch",
]


class Direction(enum.IntEnum):
    """planner.rs:10-16"""
    Forward = 1
    Reverse = -1


class PlannerMode(enum.IntEnum):
    """planner.rs:25-32 (accepted; the reference ignores it, planner.rs:65)"""
    Heuristic = 0
    Tune = 1


@dataclass
class Options:
    """options.rs:10-43.  Hints only on the GPU (kept for source compatibility)."""
    multithreaded_bit_reversal: bool = False
    smallest_parallel_chunk_size: int = 16384

    @staticmethod
    def guess_options(input_size: int) -> "Options":
        o = _lib.Options()
        _lib.lib.phastft_options_guess(int(input_size), C.byref(o))
        return Options(bool(o.multithreaded_bit_reversal), int(o.smallest_parallel_chunk_size))


# ----------------------------------------------------------------------------------------------
# array plumbing
# ----------------------------------------------------------------------------------------------
def _is_torch(a) -> bool:
    return type(a).__module__.startswith("torch")


def _np_ptr(a: np.ndarray, dtype, writable: bool):
    if not isinstance(a, np.ndarray):
        raise TypeError("expected a numpy array or a torch CUDA tensor")
    if a.dtype != dtype:
        raise TypeError(f"expected dtype {np.dtype(dtype)}, got {a.dtype}")
    if a.ndim != 1 or not a.flags.c_contiguous:
        raise ValueError("slices must be 1-D and contiguous")
    if writable and not a.flags.writeable:
        raise ValueError("output slice is read-only")
    return a.ctypes.data_as(C.c_void_p), a.size


def _torch_ptr(t, dtype):
    import torch
    want = torch.float64 if np.dtype(dtype) == np.float64 else torch.float32
    if not t.is_cuda:
        raise TypeError("torch tensors must live on a CUDA device (use numpy arrays for host slices)")
    if t.dtype != want or t.dim() != 1 or not t.is_contiguous():
        raise TypeError("expected a contiguous 1-D tensor of the planner's precision")
    return C.c_void_p(t.data_ptr()), t.numel()


def _pair_aligned(t) -> bool:
    """r2c reads its real input and c2r writes its real output as (re, im) pairs, so those device pointers must be aligned
    to 2 * sizeof(T); a view of a real tensor can start at any element, e.g. x[1:]."""
    return t.data_ptr() % (2 * t.element_size()) == 0


def _torch_stream(t):
    import torch
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


# ----------------------------------------------------------------------------------------------
# planners
# ----------------------------------------------------------------------------------------------
class _PlannerDit:
    _sfx = ""
    _dtype = None

    def __init__(self, num_points: int, device: int = 0, mode: PlannerMode = PlannerMode.Heuristic):
        """PlannerDit{64,32}::new / with_mode (planner.rs:55-100): panics unless num_points is a
        non-zero power of two."""
        self._h = C.c_void_p()
        self.device = int(device)
        check(fn("phastft_plan_dit_{s}_create", self._sfx)(int(num_points), self.device, int(mode), C.byref(self._h)))
        self.num_points = int(num_points)

    @classmethod
    def new(cls, num_points: int, device: int = 0):
        return cls(num_points, device)

    @classmethod
    def with_mode(cls, num_points: int, mode: PlannerMode, device: int = 0):
        return cls(num_points, device, mode)

    def describe(self) -> str:
        return fn("phastft_plan_dit_{s}_describe", self._sfx)(self._h).decode()

    # planner-table blob, for the one init-time broadcast of a multi-GPU job
    def reserve(self, batch: int) -> None:
        """Size the device workspace for calls of up to `batch` transforms now (otherwise the first larger call grows
        it, synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_dit_{s}_reserve", self._sfx)(self._h, int(batch)))

    def tables_bytes(self) -> int:
        return int(fn("phastft_plan_dit_{s}_tables_bytes", self._sfx)(self._h))

    def tables_export(self, dst_tensor) -> None:
        check(fn("phastft_plan_dit_{s}_tables_export", self._sfx)(self._h, C.c_void_p(dst_tensor.data_ptr()),
                                                                  _torch_stream(dst_tensor)))

    def tables_import(self, src_tensor) -> None:
        check(fn("phastft_plan_dit_{s}_tables_import", self._sfx)(self._h, C.c_void_p(src_tensor.data_ptr()),
                                                                  _torch_stream(src_tensor)))

    def broadcast_tables(self, src: int = 0, group=None) -> None:
        """One collective at init: rank `src`'s twiddle tables to every rank (torch.distributed,
        NCCL on GPUs).  After this no call communicates."""
        import torch
        import torch.distributed as dist
        buf = torch.empty(self.tables_bytes(), dtype=torch.uint8, device=f"cuda:{self.device}")
        self.tables_export(buf)
        dist.broadcast(buf, src=src, group=group)
        self.tables_import(buf)
        torch.cuda.current_stream(buf.device).synchronize()

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_dit_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerDit64(_PlannerDit):
    _sfx, _dtype = "f64", np.float64


class PlannerDit32(_PlannerDit):
    _sfx, _dtype = "f32", np.float32


class _PlannerR2c:
    _sfx = ""
    _dtype = None

    def __init__(self, n: int, device: int = 0):
        """PlannerR2c{64,32}::new (planner.rs:194-206): panics with "n must be a power of 2 >= 4"."""
        self._h = C.c_void_p()
        self.device = int(device)
        check(fn("phastft_plan_r2c_{s}_create", self._sfx)(int(n), self.device, C.byref(self._h)))
        self.n = int(n)

    @classmethod
    def new(cls, n: int, device: int = 0):
        return cls(n, device)

    def describe(self, batch: int = 1) -> str:
        """The c2r path calls of `batch` transforms take under the current environment (fused on load or the separate
        sweep, and why), the c2r build of the first pass they run, and the inner N/2-point plan's describe()."""
        if batch == 1:
            return fn("phastft_plan_r2c_{s}_describe", self._sfx)(self._h).decode()
        return fn("phastft_plan_r2c_{s}_describe_batch", self._sfx)(self._h, int(batch)).decode()

    def reserve(self, batch: int) -> None:
        """Make every allocation a batched call of `batch` transforms would make now: the inner plan's workspace and, when
        that batch's c2r takes the separate sweep, the plan-owned scratch (otherwise the first such call makes them,
        synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_r2c_{s}_reserve", self._sfx)(self._h, int(batch)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_r2c_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerR2c64(_PlannerR2c):
    _sfx, _dtype = "f64", np.float64


class PlannerR2c32(_PlannerR2c):
    _sfx, _dtype = "f32", np.float32


class _PlannerAny:
    _sfx = ""
    _dtype = None

    def __init__(self, num_points: int, device: int = 0):
        """A complex FFT of any length num_points >= 1 (the reference accepts powers of two only): a power of two runs the
        c2c plan as it is, any other length up to 2^29 - 1 Bluestein's algorithm over a power-of-two plan.  Other lengths
        raise PhastFTPanic(13) before the device is touched."""
        self._h = C.c_void_p()
        self.device = int(device)
        check(fn("phastft_plan_any_{s}_create", self._sfx)(int(num_points), self.device, C.byref(self._h)))
        self.num_points = int(num_points)

    @classmethod
    def new(cls, num_points: int, device: int = 0):
        return cls(num_points, device)

    def describe(self) -> str:
        """"power of two" or "Bluestein M=2^m" (the convolution length), then the inner plan's describe()."""
        return fn("phastft_plan_any_{s}_describe", self._sfx)(self._h).decode()

    def reserve(self, batch: int) -> None:
        """Make every allocation a call of `batch` transforms would make now (otherwise the first larger call makes them,
        synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_any_{s}_reserve", self._sfx)(self._h, int(batch)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_any_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerAny64(_PlannerAny):
    _sfx, _dtype = "f64", np.float64


class PlannerAny32(_PlannerAny):
    _sfx, _dtype = "f32", np.float32


# The convenience functions plan per call like the reference (lib.rs:180-183); building a plan and allocating its workspace
# per call costs far more than the transform, and destroying a plan while its kernels are still queued relies on cudaFree's
# implicit synchronisation -- so the most recent one-shot planner per (class, size, device) is kept, like the C library
# does for host slices (phastft_*_oneshot).
_ONESHOT_PLANNERS: dict = {}


def _oneshot_planner(cls, n: int, device: int):
    key = (cls.__name__, device)
    hit = _ONESHOT_PLANNERS.get(key)
    if hit is not None and hit[0] == n:
        return hit[1]
    planner = cls(n, device)           # raises the reference's panic for an invalid size before anything is cached
    if hit is not None and _is_torch_available():
        import torch
        torch.cuda.synchronize(device)     # the replaced planner may still have work queued
    _ONESHOT_PLANNERS[key] = (n, planner)
    return planner


def _is_torch_available() -> bool:
    try:
        import torch  # noqa: F401
        return True
    except Exception:  # noqa: BLE001
        return False


def oneshot_cache_clear() -> None:
    """Drop the planners kept for the convenience functions (here and inside the C library)."""
    _ONESHOT_PLANNERS.clear()
    _lib.lib.phastft_oneshot_cache_clear()


# ----------------------------------------------------------------------------------------------
# c2c
# ----------------------------------------------------------------------------------------------
def _fft_dit_with_planner(sfx, dtype, reals, imags, direction, planner, opts=None):
    if planner._sfx != sfx:
        raise TypeError("planner precision does not match the function")
    if _is_torch(reals):
        pr, nr = _torch_ptr(reals, dtype)
        pi, ni = _torch_ptr(imags, dtype)
        # the asserts of algorithms/dit.rs:284-289, in the reference's order
        if nr != ni:
            raise PhastFTPanic(1)
        if nr == 0 or nr & (nr - 1):
            raise PhastFTPanic(2)
        if nr != planner.num_points:
            raise PhastFTPanic(3)
        check(fn("phastft_fft_dit_{s}_dev", sfx)(planner._h, pr, pi, int(direction), 1, nr, _torch_stream(reals)))
    else:
        pr, nr = _np_ptr(reals, dtype, True)
        pi, ni = _np_ptr(imags, dtype, True)
        o = None
        if opts is not None:
            o = _lib.Options(int(opts.multithreaded_bit_reversal), int(opts.smallest_parallel_chunk_size))
        check(fn("phastft_fft_dit_{s}_host", sfx)(planner._h, pr, nr, pi, ni, int(direction),
                                                  C.byref(o) if o is not None else None))


def _fft_dit(sfx, dtype, planner_cls, reals, imags, direction, device=0):
    # lib.rs:180-183: a planner per call
    if not _is_torch(reals):
        # host slices: the library's one-shot entry (it keeps the latest plan for the next same-size call)
        pr, nr = _np_ptr(reals, dtype, True)
        pi, ni = _np_ptr(imags, dtype, True)
        check(fn("phastft_fft_dit_{s}_oneshot", sfx)(pr, nr, pi, ni, int(direction), int(device)))
        return
    planner = _oneshot_planner(planner_cls, reals.numel(), reals.device.index or 0)
    _fft_dit_with_planner(sfx, dtype, reals, imags, direction, planner)


def fft_64_dit(reals, imags, direction: Direction, device: int = 0) -> None:
    """lib.rs:180"""
    _fft_dit("f64", np.float64, PlannerDit64, reals, imags, direction, device)


def fft_64_dit_with_planner(reals, imags, direction: Direction, planner: PlannerDit64) -> None:
    """lib.rs:143"""
    _fft_dit_with_planner("f64", np.float64, reals, imags, direction, planner)


def fft_64_dit_with_planner_and_opts(reals, imags, direction: Direction, planner: PlannerDit64, opts: Options) -> None:
    """algorithms/dit.rs:263"""
    _fft_dit_with_planner("f64", np.float64, reals, imags, direction, planner, opts)


def fft_32_dit(reals, imags, direction: Direction, device: int = 0) -> None:
    """lib.rs:223"""
    _fft_dit("f32", np.float32, PlannerDit32, reals, imags, direction, device)


def fft_32_dit_with_planner(reals, imags, direction: Direction, planner: PlannerDit32) -> None:
    """lib.rs:186"""
    _fft_dit_with_planner("f32", np.float32, reals, imags, direction, planner)


def fft_32_dit_with_planner_and_opts(reals, imags, direction: Direction, planner: PlannerDit32, opts: Options) -> None:
    """algorithms/dit.rs:338"""
    _fft_dit_with_planner("f32", np.float32, reals, imags, direction, planner, opts)


def fft_dit_batch(reals, imags, direction: Direction, planner, batch: int, batch_stride: int | None = None) -> None:
    """Batched device-resident transform: `batch` signals of planner.num_points, transform b at
    offset b*batch_stride of the planar torch CUDA tensors.  (The reference has no batch API; a
    batch is a caller loop sharing one planner, examples/benchmark.rs:24-36.)"""
    n = planner.num_points
    stride = n if batch_stride is None else int(batch_stride)
    pr, nr = _torch_ptr(reals, planner._dtype)
    pi, ni = _torch_ptr(imags, planner._dtype)
    if nr != ni:
        raise PhastFTPanic(1)
    if batch < 1 or nr < (batch - 1) * stride + n:
        raise PhastFTPanic(13, "tensors shorter than batch * batch_stride")
    check(fn("phastft_fft_dit_{s}_dev", planner._sfx)(planner._h, pr, pi, int(direction), int(batch), stride,
                                                      _torch_stream(reals)))


def fft_dit_batch_sharded(reals: np.ndarray, imags: np.ndarray, direction: Direction, planners, batch: int,
                          batch_stride: int | None = None) -> None:
    """Host planar batch sharded over several devices from ONE process (one planner per device)."""
    sfx, dtype = planners[0]._sfx, planners[0]._dtype
    n = planners[0].num_points
    stride = n if batch_stride is None else int(batch_stride)
    pr, nr = _np_ptr(reals, dtype, True)
    pi, ni = _np_ptr(imags, dtype, True)
    if nr != ni:
        raise PhastFTPanic(1)
    if nr < (batch - 1) * stride + n:
        raise PhastFTPanic(13, "arrays shorter than batch * batch_stride")
    arr = (C.c_void_p * len(planners))(*[p._h for p in planners])
    check(fn("phastft_fft_dit_{s}_batch_sharded_host", sfx)(arr, len(planners), pr, pi, int(batch), stride, int(direction)))


def host_register(array: np.ndarray) -> None:
    """Page-lock a numpy array in place (cudaHostRegister) so the host-slice calls copy at full PCIe speed
    (~52 GB/s instead of ~13 GB/s from pageable memory); undo with host_unregister before freeing it."""
    check(_lib.lib.phastft_host_register(array.ctypes.data_as(C.c_void_p), array.nbytes))


def host_unregister(array: np.ndarray) -> None:
    check(_lib.lib.phastft_host_unregister(array.ctypes.data_as(C.c_void_p)))


# ----------------------------------------------------------------------------------------------
# interleaved Complex<T> API (lib.rs:41-140, feature `complex-nums`)
# ----------------------------------------------------------------------------------------------
def _interleaved(sfx, dtype, cdtype, signal, direction, planner):
    if _is_torch(signal):
        import torch
        if not signal.is_cuda or signal.dtype != (torch.complex128 if sfx == "f64" else torch.complex64):
            raise TypeError("expected a CUDA complex tensor of the planner's precision")
        n = signal.numel()
        if n == 0 or n & (n - 1):
            raise PhastFTPanic(2)
        if n != planner.num_points:
            raise PhastFTPanic(3)
        # (torch keeps a complex tensor's storage offset in whole elements, so its pointer is pair-aligned)
        check(fn("phastft_fft_interleaved_{s}_dev", sfx)(planner._h, C.c_void_p(signal.data_ptr()), int(direction), 1, n,
                                                          _torch_stream(signal)))
    else:
        if signal.dtype != cdtype or signal.ndim != 1 or not signal.flags.c_contiguous:
            raise TypeError(f"expected a contiguous 1-D {np.dtype(cdtype)} array")
        check(fn("phastft_fft_interleaved_{s}_host", sfx)(planner._h, signal.ctypes.data_as(C.c_void_p), signal.size,
                                                           int(direction)))


def fft_64_interleaved_with_planner_and_opts(signal, direction, planner: PlannerDit64, opts: Options | None = None):
    _interleaved("f64", np.float64, np.complex128, signal, direction, planner)


def fft_64_interleaved_with_planner(signal, direction, planner: PlannerDit64):
    _interleaved("f64", np.float64, np.complex128, signal, direction, planner)


def fft_64_interleaved(signal, direction, device: int = 0):
    n = signal.numel() if _is_torch(signal) else signal.size
    _interleaved("f64", np.float64, np.complex128, signal, direction, _oneshot_planner(PlannerDit64, n, device))


def fft_32_interleaved_with_planner_and_opts(signal, direction, planner: PlannerDit32, opts: Options | None = None):
    _interleaved("f32", np.float32, np.complex64, signal, direction, planner)


def fft_32_interleaved_with_planner(signal, direction, planner: PlannerDit32):
    _interleaved("f32", np.float32, np.complex64, signal, direction, planner)


def fft_32_interleaved(signal, direction, device: int = 0):
    n = signal.numel() if _is_torch(signal) else signal.size
    _interleaved("f32", np.float32, np.complex64, signal, direction, _oneshot_planner(PlannerDit32, n, device))


# ----------------------------------------------------------------------------------------------
# r2c / c2r
# ----------------------------------------------------------------------------------------------
def _r2c_with_planner(sfx, dtype, x, out_re, out_im, planner):
    if _is_torch(x):
        px, nx = _torch_ptr(x, dtype)
        pr, nr = _torch_ptr(out_re, dtype)
        pi, ni = _torch_ptr(out_im, dtype)
        half = planner.n // 2
        if nx != planner.n:
            raise PhastFTPanic(5)
        if nr != half + 1:
            raise PhastFTPanic(6)
        if ni != half + 1:
            raise PhastFTPanic(7)
        if not _pair_aligned(x):                                  # the input is read as pairs: an aligned copy
            x = x.clone()
            px = C.c_void_p(x.data_ptr())
        check(fn("phastft_r2c_{s}_dev", sfx)(planner._h, px, pr, pi, _torch_stream(x)))
    else:
        px, nx = _np_ptr(x, dtype, False)
        pr, nr = _np_ptr(out_re, dtype, True)
        pi, ni = _np_ptr(out_im, dtype, True)
        check(fn("phastft_r2c_{s}_host", sfx)(planner._h, px, nx, pr, nr, pi, ni))


def _c2r_with_planner(sfx, dtype, in_re, in_im, out, planner, scratch_re=None, scratch_im=None):
    if _is_torch(out):
        import torch
        pr, nr = _torch_ptr(in_re, dtype)
        pi, ni = _torch_ptr(in_im, dtype)
        po, no = _torch_ptr(out, dtype)
        half = planner.n // 2
        if no != planner.n:
            raise PhastFTPanic(8)
        if nr != half + 1:
            raise PhastFTPanic(9)
        if ni != half + 1:
            raise PhastFTPanic(10)
        psr = psi = None
        if scratch_re is not None or scratch_im is not None:
            psr, nsr = _torch_ptr(scratch_re, dtype)
            psi, nsi = _torch_ptr(scratch_im, dtype)
            if nsr != half:
                raise PhastFTPanic(11)
            if nsi != half:
                raise PhastFTPanic(12)
        work = out if _pair_aligned(out) else torch.empty_like(out)    # the output is written as pairs: an aligned temporary
        check(fn("phastft_c2r_{s}_dev", sfx)(planner._h, pr, pi, C.c_void_p(work.data_ptr()), psr, psi, _torch_stream(out)))
        if work is not out:
            out.copy_(work)
    else:
        pr, nr = _np_ptr(in_re, dtype, False)
        pi, ni = _np_ptr(in_im, dtype, False)
        po, no = _np_ptr(out, dtype, True)
        if scratch_re is None and scratch_im is None:
            psr, nsr, psi, nsi = None, 0, None, 0
        else:
            psr, nsr = _np_ptr(scratch_re, dtype, True)
            psi, nsi = _np_ptr(scratch_im, dtype, True)
        check(fn("phastft_c2r_{s}_host", sfx)(planner._h, pr, nr, pi, ni, po, no, psr, nsr, psi, nsi))


def _len(a):
    return a.numel() if _is_torch(a) else a.size


def _dev_of(a, device):
    return (a.device.index or 0) if _is_torch(a) else device


def r2c_fft_f64(input_re, output_re, output_im, device: int = 0) -> None:
    """r2c.rs:521: PlannerR2c64::new(input_re.len()) then the planner path."""
    if not _is_torch(input_re):
        px, nx = _np_ptr(input_re, np.float64, False)
        pr, nr = _np_ptr(output_re, np.float64, True)
        pi, ni = _np_ptr(output_im, np.float64, True)
        check(fn("phastft_r2c_{s}_oneshot", "f64")(px, nx, pr, nr, pi, ni, int(device)))
        return
    _r2c_with_planner("f64", np.float64, input_re, output_re, output_im, _oneshot_planner(PlannerR2c64, _len(input_re), _dev_of(input_re, device)))


def r2c_fft_f64_with_planner(input_re, output_re, output_im, planner: PlannerR2c64) -> None:
    """r2c.rs:535"""
    _r2c_with_planner("f64", np.float64, input_re, output_re, output_im, planner)


def c2r_fft_f64(input_re, input_im, output, device: int = 0) -> None:
    """r2c.rs:695: PlannerR2c64::new(output.len())"""
    if not _is_torch(output):
        pr, nr = _np_ptr(input_re, np.float64, False)
        pi, ni = _np_ptr(input_im, np.float64, False)
        po, no = _np_ptr(output, np.float64, True)
        check(fn("phastft_c2r_{s}_oneshot", "f64")(pr, nr, pi, ni, po, no, int(device)))
        return
    _c2r_with_planner("f64", np.float64, input_re, input_im, output, _oneshot_planner(PlannerR2c64, _len(output), _dev_of(output, device)))


def c2r_fft_f64_with_planner(input_re, input_im, output, planner: PlannerR2c64) -> None:
    """r2c.rs:708"""
    _c2r_with_planner("f64", np.float64, input_re, input_im, output, planner)


def c2r_fft_f64_with_planner_and_scratch(input_re, input_im, output, planner: PlannerR2c64, scratch_re, scratch_im) -> None:
    """r2c.rs:740"""
    _c2r_with_planner("f64", np.float64, input_re, input_im, output, planner, scratch_re, scratch_im)


def r2c_fft_f32(input_re, output_re, output_im, device: int = 0) -> None:
    """r2c.rs:598"""
    if not _is_torch(input_re):
        px, nx = _np_ptr(input_re, np.float32, False)
        pr, nr = _np_ptr(output_re, np.float32, True)
        pi, ni = _np_ptr(output_im, np.float32, True)
        check(fn("phastft_r2c_{s}_oneshot", "f32")(px, nx, pr, nr, pi, ni, int(device)))
        return
    _r2c_with_planner("f32", np.float32, input_re, output_re, output_im, _oneshot_planner(PlannerR2c32, _len(input_re), _dev_of(input_re, device)))


def r2c_fft_f32_with_planner(input_re, output_re, output_im, planner: PlannerR2c32) -> None:
    """r2c.rs:607"""
    _r2c_with_planner("f32", np.float32, input_re, output_re, output_im, planner)


def c2r_fft_f32(input_re, input_im, output, device: int = 0) -> None:
    """r2c.rs:804"""
    if not _is_torch(output):
        pr, nr = _np_ptr(input_re, np.float32, False)
        pi, ni = _np_ptr(input_im, np.float32, False)
        po, no = _np_ptr(output, np.float32, True)
        check(fn("phastft_c2r_{s}_oneshot", "f32")(pr, nr, pi, ni, po, no, int(device)))
        return
    _c2r_with_planner("f32", np.float32, input_re, input_im, output, _oneshot_planner(PlannerR2c32, _len(output), _dev_of(output, device)))


def c2r_fft_f32_with_planner(input_re, input_im, output, planner: PlannerR2c32) -> None:
    """r2c.rs:813"""
    _c2r_with_planner("f32", np.float32, input_re, input_im, output, planner)


def c2r_fft_f32_with_planner_and_scratch(input_re, input_im, output, planner: PlannerR2c32, scratch_re, scratch_im) -> None:
    """r2c.rs:835"""
    _c2r_with_planner("f32", np.float32, input_re, input_im, output, planner, scratch_re, scratch_im)


# ----------------------------------------------------------------------------------------------
# batched r2c / c2r (device-resident; the reference has no batch API)
# ----------------------------------------------------------------------------------------------
def _check_batch_len(what: str, have: int, batch: int, stride: int, length: int) -> None:
    if batch < 0:
        raise PhastFTPanic(13, "batch < 0")
    if batch and have < (batch - 1) * stride + length:
        raise PhastFTPanic(13, f"{what} shorter than (batch - 1) * stride + {length}")


def r2c_batch(x, out_re, out_im, planner, batch: int, in_stride: int | None = None, out_stride: int | None = None) -> None:
    """`batch` r2c transforms in one call on flat 1-D torch CUDA tensors: member b reads N reals at x[b * in_stride:] and
    writes N/2 + 1 bins at out_re / out_im[b * out_stride:] (defaults: N and N/2 + 1).  In-stride must be even (the input is
    read as (re, im) pairs); a misaligned x is read through an aligned copy."""
    n, half = planner.n, planner.n // 2
    in_stride = n if in_stride is None else int(in_stride)
    out_stride = half + 1 if out_stride is None else int(out_stride)
    px, nx = _torch_ptr(x, planner._dtype)
    pr, nr = _torch_ptr(out_re, planner._dtype)
    pi, ni = _torch_ptr(out_im, planner._dtype)
    _check_batch_len("input", nx, batch, in_stride, n)
    _check_batch_len("output_re", nr, batch, out_stride, half + 1)
    _check_batch_len("output_im", ni, batch, out_stride, half + 1)
    if not _pair_aligned(x):
        x = x.clone()
        px = C.c_void_p(x.data_ptr())
    check(fn("phastft_r2c_{s}_batch_dev", planner._sfx)(planner._h, px, in_stride, pr, pi, out_stride, int(batch), _torch_stream(x)))


def c2r_batch(in_re, in_im, out, planner, batch: int, in_stride: int | None = None, out_stride: int | None = None,
              scratch_re=None, scratch_im=None) -> None:
    """`batch` c2r transforms in one call on flat 1-D torch CUDA tensors: member b reads N/2 + 1 bins at
    in_re / in_im[b * in_stride:] and writes N reals at out[b * out_stride:] (defaults: N/2 + 1 and N), normalised so that
    c2r(r2c(x)) == x.  scratch_re / scratch_im: batch * N/2 each, or neither (the planner's own).  Out-stride must be even
    (the output is written as (re, im) pairs); a misaligned out is written through an aligned copy."""
    n, half = planner.n, planner.n // 2
    in_stride = half + 1 if in_stride is None else int(in_stride)
    out_stride = n if out_stride is None else int(out_stride)
    pr, nr = _torch_ptr(in_re, planner._dtype)
    pi, ni = _torch_ptr(in_im, planner._dtype)
    _, no = _torch_ptr(out, planner._dtype)
    _check_batch_len("input_re", nr, batch, in_stride, half + 1)
    _check_batch_len("input_im", ni, batch, in_stride, half + 1)
    _check_batch_len("output", no, batch, out_stride, n)
    psr = psi = None
    if scratch_re is not None or scratch_im is not None:
        psr, nsr = _torch_ptr(scratch_re, planner._dtype)
        psi, nsi = _torch_ptr(scratch_im, planner._dtype)
        if nsr < batch * half or nsi < batch * half:
            raise PhastFTPanic(13, "scratch shorter than batch * N/2")
    work = out if _pair_aligned(out) else out.clone()      # the clone keeps what lies between the members
    check(fn("phastft_c2r_{s}_batch_dev", planner._sfx)(planner._h, pr, pi, in_stride, C.c_void_p(work.data_ptr()), out_stride,
                                                        psr, psi, int(batch), _torch_stream(out)))
    if work is not out:
        out.copy_(work)


# ----------------------------------------------------------------------------------------------
# complex FFTs of any length (the reference accepts powers of two only)
# ----------------------------------------------------------------------------------------------
def _fft_any_with_planner(sfx, dtype, reals, imags, direction, planner):
    if planner._sfx != sfx:
        raise TypeError("planner precision does not match the function")
    if _is_torch(reals):
        pr, nr = _torch_ptr(reals, dtype)
        pi, ni = _torch_ptr(imags, dtype)
        if nr != ni:
            raise PhastFTPanic(1)
        if nr != planner.num_points:
            raise PhastFTPanic(3)
        check(fn("phastft_fft_any_{s}_dev", sfx)(planner._h, pr, pi, int(direction), 1, nr, _torch_stream(reals)))
    else:
        pr, nr = _np_ptr(reals, dtype, True)
        pi, ni = _np_ptr(imags, dtype, True)
        check(fn("phastft_fft_any_{s}_host", sfx)(planner._h, pr, nr, pi, ni, int(direction)))


def fft_64_any_with_planner(reals, imags, direction: Direction, planner: PlannerAny64) -> None:
    """fft_64_dit_with_planner for any length: numpy arrays (synchronous) or torch CUDA tensors (torch's current stream)."""
    _fft_any_with_planner("f64", np.float64, reals, imags, direction, planner)


def fft_32_any_with_planner(reals, imags, direction: Direction, planner: PlannerAny32) -> None:
    _fft_any_with_planner("f32", np.float32, reals, imags, direction, planner)


def fft_any_batch(reals, imags, direction: Direction, planner, batch: int, batch_stride: int | None = None) -> None:
    """fft_dit_batch for any length: `batch` signals of planner.num_points, transform b at offset b * batch_stride of the planar
    torch CUDA tensors."""
    n = planner.num_points
    stride = n if batch_stride is None else int(batch_stride)
    pr, nr = _torch_ptr(reals, planner._dtype)
    pi, ni = _torch_ptr(imags, planner._dtype)
    if nr != ni:
        raise PhastFTPanic(1)
    _check_batch_len("tensors", nr, batch, stride, n)
    check(fn("phastft_fft_any_{s}_dev", planner._sfx)(planner._h, pr, pi, int(direction), int(batch), stride,
                                                      _torch_stream(reals)))
