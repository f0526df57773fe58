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
    "AnyAlgo", "PlannerAny64", "PlannerAny32", "fft_64_any_with_planner", "fft_32_any_with_planner", "fft_any_batch",
    "PlannerR2cAny64", "PlannerR2cAny32", "r2c_fft_f64_any_with_planner", "r2c_fft_f32_any_with_planner",
    "c2r_fft_f64_any_with_planner", "c2r_fft_f32_any_with_planner", "r2c_any_batch", "c2r_any_batch",
    "fft_64_interleaved_any_with_planner", "fft_32_interleaved_any_with_planner", "fft_interleaved_any_batch",
    "r2c_fft_f64_interleaved_any_with_planner", "r2c_fft_f32_interleaved_any_with_planner",
    "c2r_fft_f64_interleaved_any_with_planner", "c2r_fft_f32_interleaved_any_with_planner",
    "r2c_interleaved_any_batch", "c2r_interleaved_any_batch",
    "PlannerDct64", "PlannerDct32", "dct_f64_with_planner", "dct_f32_with_planner", "dst_f64_with_planner", "dst_f32_with_planner",
    "dct_batch", "dst_batch",
    "PlannerConv64", "PlannerConv32", "convolve_with_planner", "correlate_with_planner", "convolve_batch", "correlate_batch",
    "PlannerStft64", "PlannerStft32", "stft_with_planner", "istft_with_planner", "stft_batch", "istft_batch",
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


class AnyAlgo(enum.IntEnum):
    """How a length that is not a power of two is transformed (include/phastft_cuda.h, PHASTFT_ANY_*).  Auto picks Mixed for
    every eligible length (2^a 3^b 5^c 7^d below 2^30 whose odd part fits one or two odd passes) and Bluestein otherwise, from
    the factorisation of the length alone: pass it unless one algorithm is wanted."""
    Bluestein = 0
    Mixed = 1
    Auto = 2


class _PlannerAny:
    _sfx = ""
    _dtype = None

    def __init__(self, num_points: int, device: int = 0, algo: AnyAlgo = AnyAlgo.Bluestein):
        """A complex FFT of any length num_points >= 1 (the reference accepts powers of two only): a power of two runs the
        c2c plan as it is, any other length up to 2^29 - 1 Bluestein's algorithm over a power-of-two plan, or with
        AnyAlgo.Mixed / AnyAlgo.Auto the mixed-radix path for smooth lengths below 2^30.  Other lengths (and AnyAlgo.Mixed on
        a length that is not eligible) raise PhastFTPanic(13) before the device is touched."""
        self._h = C.c_void_p()
        self.device = int(device)
        check(fn("phastft_plan_any_{s}_create_with", self._sfx)(int(num_points), self.device, int(algo), C.byref(self._h)))
        self.num_points = int(num_points)

    @classmethod
    def new(cls, num_points: int, device: int = 0):
        return cls(num_points, device)

    @classmethod
    def with_algo(cls, num_points: int, algo: AnyAlgo, device: int = 0):
        return cls(num_points, device, algo)

    def describe(self) -> str:
        """"power of two", "Bluestein M=2^m" (the convolution length) or "mixed 2^a x Q_a[ x Q_b]", then the inner plan's
        describe()."""
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


class _PlannerR2cAny:
    _sfx = ""
    _dtype = None

    def __init__(self, n: int, device: int = 0, algo: AnyAlgo = AnyAlgo.Bluestein):
        """Real-input FFTs of any length n (the reference's r2c accepts powers of two >= 4 only): a power of two from 4 to
        2^31 runs the r2c plan as it is, an even n up to 2^30 - 2 Bluestein of n/2 ("halved"), an odd n up to 2^29 - 1
        Bluestein of n ("direct").  With AnyAlgo.Mixed / AnyAlgo.Auto the halved and direct paths run the mixed-radix
        transform of n/2 (even n up to 2^31 - 2) or n instead when that length is eligible.  Other lengths (and
        AnyAlgo.Mixed on a length that is not eligible) raise PhastFTPanic(13) before the device is touched."""
        self._h = C.c_void_p()
        self.device = int(device)
        check(fn("phastft_plan_r2c_any_{s}_create_with", self._sfx)(int(n), self.device, int(algo), C.byref(self._h)))
        self.n = int(n)

    @classmethod
    def new(cls, n: int, device: int = 0):
        return cls(n, device)

    @classmethod
    def with_algo(cls, n: int, algo: AnyAlgo, device: int = 0):
        return cls(n, device, algo)

    def describe(self) -> str:
        """"power of two | <the r2c plan's describe()>", or "halved" / "direct", then "Bluestein L=<L> M=2^m" or
        "mixed 2^a x Q_a[ x Q_b]", then the inner plan's describe()."""
        return fn("phastft_plan_r2c_any_{s}_describe", self._sfx)(self._h).decode()

    def reserve(self, batch: int) -> None:
        """Make every allocation a call of `batch` members would make now (otherwise the first larger call makes them,
        synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_r2c_any_{s}_reserve", self._sfx)(self._h, int(batch)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_r2c_any_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerR2cAny64(_PlannerR2cAny):
    _sfx, _dtype = "f64", np.float64


class PlannerR2cAny32(_PlannerR2cAny):
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


def _complex_any_ptr(sfx, signal, planner, host, writable=True):
    """The pointer and length of an interleaved complex signal for planner (a PlannerAny or PlannerR2cAny of precision sfx): a
    torch CUDA complex tensor, or with host=True also a numpy array (writable unless `writable` is False).  Raises before
    anything reaches the library."""
    if planner._sfx != sfx:
        raise TypeError("planner precision does not match the function")
    if _is_torch(signal):
        import torch
        if not signal.is_cuda or signal.dtype != (torch.complex128 if sfx == "f64" else torch.complex64):
            raise TypeError("expected a CUDA complex tensor of the planner's precision")
        if signal.dim() != 1 or not signal.is_contiguous():
            raise TypeError("expected a contiguous 1-D tensor")
        # (torch keeps a complex tensor's storage offset in whole elements, so its pointer is pair-aligned)
        return C.c_void_p(signal.data_ptr()), signal.numel()
    if not host:
        raise TypeError("expected a torch CUDA complex tensor")
    cdtype = np.complex128 if sfx == "f64" else np.complex64
    if not isinstance(signal, np.ndarray) or signal.dtype != cdtype or signal.ndim != 1 or not signal.flags.c_contiguous:
        raise TypeError(f"expected a contiguous 1-D {np.dtype(cdtype)} array or a torch CUDA complex tensor")
    if writable and not signal.flags.writeable:
        raise ValueError("signal is read-only")
    return signal.ctypes.data_as(C.c_void_p), signal.size


def _fft_interleaved_any_with_planner(sfx, signal, direction, planner):
    p, n = _complex_any_ptr(sfx, signal, planner, True)
    if n != planner.num_points:
        raise PhastFTPanic(3)
    if _is_torch(signal):
        check(fn("phastft_fft_interleaved_any_{s}_dev", sfx)(planner._h, p, int(direction), 1, n, _torch_stream(signal)))
    else:
        check(fn("phastft_fft_interleaved_any_{s}_host", sfx)(planner._h, p, n, int(direction)))


def fft_64_interleaved_any_with_planner(signal, direction: Direction, planner: PlannerAny64) -> None:
    """fft_64_any_with_planner on interleaved complex128 values, in place: a numpy array (synchronous) or a torch CUDA tensor
    (torch's current stream).  Bluestein and mixed-radix plans give the planar call's results bit for bit."""
    _fft_interleaved_any_with_planner("f64", signal, direction, planner)


def fft_32_interleaved_any_with_planner(signal, direction: Direction, planner: PlannerAny32) -> None:
    _fft_interleaved_any_with_planner("f32", signal, direction, planner)


def fft_interleaved_any_batch(signal, direction: Direction, planner, batch: int, batch_stride: int | None = None) -> None:
    """fft_any_batch on a flat 1-D torch CUDA complex tensor: `batch` signals of planner.num_points, transform b at complex
    element b * batch_stride (default planner.num_points)."""
    n = planner.num_points
    stride = n if batch_stride is None else int(batch_stride)
    p, total = _complex_any_ptr(planner._sfx, signal, planner, False)
    _check_batch_len("tensor", total, batch, stride, n)
    check(fn("phastft_fft_interleaved_any_{s}_dev", planner._sfx)(planner._h, p, int(direction), int(batch), stride,
                                                                  _torch_stream(signal)))


# ----------------------------------------------------------------------------------------------
# real-input FFTs of any length (the reference's r2c / c2r accept powers of two >= 4 only)
# ----------------------------------------------------------------------------------------------
def _r2c_any(sfx, x, out_re, out_im, planner, batch, in_stride, out_stride):
    if planner._sfx != sfx:
        raise TypeError("planner precision does not match the function")
    n, bins = planner.n, planner.n // 2 + 1
    in_stride = n if in_stride is None else int(in_stride)
    out_stride = bins if out_stride is None else int(out_stride)
    px, nx = _torch_ptr(x, planner._dtype)
    pr, nr = _torch_ptr(out_re, planner._dtype)
    pi, ni = _torch_ptr(out_im, planner._dtype)
    _check_batch_len("input", nx, batch, in_stride, n)
    _check_batch_len("output_re", nr, batch, out_stride, bins)
    _check_batch_len("output_im", ni, batch, out_stride, bins)
    if n % 2 == 0 and not _pair_aligned(x):                   # even n reads the input as pairs: an aligned copy
        x = x.clone()
        px = C.c_void_p(x.data_ptr())
    check(fn("phastft_r2c_any_{s}_dev", sfx)(planner._h, px, in_stride, pr, pi, out_stride, int(batch), _torch_stream(x)))


def _c2r_any(sfx, in_re, in_im, out, planner, batch, in_stride, out_stride):
    if planner._sfx != sfx:
        raise TypeError("planner precision does not match the function")
    n, bins = planner.n, planner.n // 2 + 1
    in_stride = bins if in_stride is None else int(in_stride)
    out_stride = n if out_stride is None else int(out_stride)
    pr, nr = _torch_ptr(in_re, planner._dtype)
    pi, ni = _torch_ptr(in_im, planner._dtype)
    _, no = _torch_ptr(out, planner._dtype)
    _check_batch_len("input_re", nr, batch, in_stride, bins)
    _check_batch_len("input_im", ni, batch, in_stride, bins)
    _check_batch_len("output", no, batch, out_stride, n)
    work = out if n % 2 or _pair_aligned(out) else out.clone()   # even n writes pairs; the clone keeps what lies between members
    check(fn("phastft_c2r_any_{s}_dev", sfx)(planner._h, pr, pi, in_stride, C.c_void_p(work.data_ptr()), out_stride, int(batch),
                                             _torch_stream(out)))
    if work is not out:
        out.copy_(work)


def _r2c_any_with_planner(sfx, dtype, x, out_re, out_im, planner):
    if _is_torch(x):
        bins = planner.n // 2 + 1
        if x.numel() != planner.n:
            raise PhastFTPanic(5)
        if out_re.numel() != bins:
            raise PhastFTPanic(6)
        if out_im.numel() != bins:
            raise PhastFTPanic(7)
        _r2c_any(sfx, x, out_re, out_im, planner, 1, None, None)
    else:
        if planner._sfx != sfx:
            raise TypeError("planner precision does not match the function")
        px, nx = _np_ptr(x, dtype, False)
        pr, nr = _np_ptr(out_re, dtype, True)
        pi, ni = _np_ptr(out_im, dtype, True)
        check(fn("phastft_r2c_any_{s}_host", sfx)(planner._h, px, nx, pr, nr, pi, ni))


def _c2r_any_with_planner(sfx, dtype, in_re, in_im, out, planner):
    if _is_torch(out):
        bins = planner.n // 2 + 1
        if out.numel() != planner.n:
            raise PhastFTPanic(8)
        if in_re.numel() != bins:
            raise PhastFTPanic(9)
        if in_im.numel() != bins:
            raise PhastFTPanic(10)
        _c2r_any(sfx, in_re, in_im, out, planner, 1, None, None)
    else:
        if planner._sfx != sfx:
            raise TypeError("planner precision does not match the function")
        pr, nr = _np_ptr(in_re, dtype, False)
        pi, ni = _np_ptr(in_im, dtype, False)
        po, no = _np_ptr(out, dtype, True)
        check(fn("phastft_c2r_any_{s}_host", sfx)(planner._h, pr, nr, pi, ni, po, no))


def r2c_fft_f64_any_with_planner(input_re, output_re, output_im, planner: PlannerR2cAny64) -> None:
    """r2c_fft_f64_with_planner for any length: N reals in, N/2 + 1 bins out (N/2 rounded down); numpy arrays (synchronous) or
    torch CUDA tensors (torch's current stream)."""
    _r2c_any_with_planner("f64", np.float64, input_re, output_re, output_im, planner)


def r2c_fft_f32_any_with_planner(input_re, output_re, output_im, planner: PlannerR2cAny32) -> None:
    _r2c_any_with_planner("f32", np.float32, input_re, output_re, output_im, planner)


def c2r_fft_f64_any_with_planner(input_re, input_im, output, planner: PlannerR2cAny64) -> None:
    """c2r_fft_f64_with_planner for any length: N/2 + 1 bins in, N reals out, normalised so that c2r(r2c(x)) == x."""
    _c2r_any_with_planner("f64", np.float64, input_re, input_im, output, planner)


def c2r_fft_f32_any_with_planner(input_re, input_im, output, planner: PlannerR2cAny32) -> None:
    _c2r_any_with_planner("f32", np.float32, input_re, input_im, output, planner)


def r2c_any_batch(x, out_re, out_im, planner, batch: int, in_stride: int | None = None, out_stride: int | None = None) -> None:
    """r2c_batch for any length: member b reads N reals at x[b * in_stride:] and writes N/2 + 1 bins at
    out_re / out_im[b * out_stride:] (defaults: N and N/2 + 1).  For even N the in-stride must be even (the input is read as
    pairs); a misaligned x is read through an aligned copy."""
    _r2c_any(planner._sfx, x, out_re, out_im, planner, int(batch), in_stride, out_stride)


def c2r_any_batch(in_re, in_im, out, planner, batch: int, in_stride: int | None = None, out_stride: int | None = None) -> None:
    """c2r_batch for any length: member b reads N/2 + 1 bins at in_re / in_im[b * in_stride:] and writes N reals at
    out[b * out_stride:] (defaults: N/2 + 1 and N).  For even N the out-stride must be even (the output is written as pairs)."""
    _c2r_any(planner._sfx, in_re, in_im, out, planner, int(batch), in_stride, out_stride)


# ----------------------------------------------------------------------------------------------
# real-input FFTs of any length with the spectrum as interleaved complex bins (torch.fft.rfft / irfft's layout)
# ----------------------------------------------------------------------------------------------
def _r2c_interleaved_any(sfx, x, out, planner, batch, in_stride, out_stride):
    po, no = _complex_any_ptr(sfx, out, planner, False)
    n, bins = planner.n, planner.n // 2 + 1
    in_stride = n if in_stride is None else int(in_stride)
    out_stride = bins if out_stride is None else int(out_stride)
    px, nx = _torch_ptr(x, planner._dtype)
    _check_batch_len("input", nx, batch, in_stride, n)
    _check_batch_len("output", no, batch, out_stride, bins)
    if n % 2 == 0 and not _pair_aligned(x):                   # even n reads the input as pairs: an aligned copy
        x = x.clone()
        px = C.c_void_p(x.data_ptr())
    check(fn("phastft_r2c_interleaved_any_{s}_dev", sfx)(planner._h, px, in_stride, po, out_stride, int(batch), _torch_stream(x)))


def _c2r_interleaved_any(sfx, spec, out, planner, batch, in_stride, out_stride):
    ps, ns = _complex_any_ptr(sfx, spec, planner, False)
    n, bins = planner.n, planner.n // 2 + 1
    in_stride = bins if in_stride is None else int(in_stride)
    out_stride = n if out_stride is None else int(out_stride)
    _, no = _torch_ptr(out, planner._dtype)
    _check_batch_len("input", ns, batch, in_stride, bins)
    _check_batch_len("output", no, batch, out_stride, n)
    work = out if n % 2 or _pair_aligned(out) else out.clone()   # even n writes pairs; the clone keeps what lies between members
    check(fn("phastft_c2r_interleaved_any_{s}_dev", sfx)(planner._h, ps, in_stride, C.c_void_p(work.data_ptr()), out_stride,
                                                         int(batch), _torch_stream(out)))
    if work is not out:
        out.copy_(work)


def _r2c_interleaved_any_with_planner(sfx, dtype, x, out, planner):
    if _is_torch(x):
        _, no = _complex_any_ptr(sfx, out, planner, False)
        if x.numel() != planner.n:
            raise PhastFTPanic(5)
        if no != planner.n // 2 + 1:
            raise PhastFTPanic(6)
        _r2c_interleaved_any(sfx, x, out, planner, 1, None, None)
    else:
        if _is_torch(out):
            raise TypeError("numpy input with a torch output: pass both as numpy arrays or both as torch CUDA tensors")
        po, no = _complex_any_ptr(sfx, out, planner, True)
        px, nx = _np_ptr(x, dtype, False)
        check(fn("phastft_r2c_interleaved_any_{s}_host", sfx)(planner._h, px, nx, po, no))


def _c2r_interleaved_any_with_planner(sfx, dtype, spec, out, planner):
    if _is_torch(out):
        _, ns = _complex_any_ptr(sfx, spec, planner, False)
        if out.numel() != planner.n:
            raise PhastFTPanic(8)
        if ns != planner.n // 2 + 1:
            raise PhastFTPanic(9)
        _c2r_interleaved_any(sfx, spec, out, planner, 1, None, None)
    else:
        if _is_torch(spec):
            raise TypeError("torch input with a numpy output: pass both as numpy arrays or both as torch CUDA tensors")
        ps, ns = _complex_any_ptr(sfx, spec, planner, True, writable=False)
        po, no = _np_ptr(out, dtype, True)
        check(fn("phastft_c2r_interleaved_any_{s}_host", sfx)(planner._h, ps, ns, po, no))


def r2c_fft_f64_interleaved_any_with_planner(input_re, output, planner: PlannerR2cAny64) -> None:
    """r2c_fft_f64_any_with_planner with the N/2 + 1 bins (N/2 rounded down) as one complex128 array: a float64 / complex128 numpy
    pair (synchronous) or torch CUDA tensors (torch's current stream), the layout of torch.fft.rfft.  Bit-identical to the planar
    call on the same plan."""
    _r2c_interleaved_any_with_planner("f64", np.float64, input_re, output, planner)


def r2c_fft_f32_interleaved_any_with_planner(input_re, output, planner: PlannerR2cAny32) -> None:
    _r2c_interleaved_any_with_planner("f32", np.float32, input_re, output, planner)


def c2r_fft_f64_interleaved_any_with_planner(input, output, planner: PlannerR2cAny64) -> None:
    """c2r_fft_f64_any_with_planner from N/2 + 1 complex128 bins (torch.fft.irfft(spec, n=N)'s input), normalised so that
    c2r(r2c(x)) == x; the input is never written."""
    _c2r_interleaved_any_with_planner("f64", np.float64, input, output, planner)


def c2r_fft_f32_interleaved_any_with_planner(input, output, planner: PlannerR2cAny32) -> None:
    _c2r_interleaved_any_with_planner("f32", np.float32, input, output, planner)


def r2c_interleaved_any_batch(x, out, planner, batch: int, in_stride: int | None = None, out_stride: int | None = None) -> None:
    """r2c_any_batch into a flat 1-D complex torch CUDA tensor: member b reads N reals at x[b * in_stride:] and writes N/2 + 1
    bins at out[b * out_stride:] (complex values; defaults: N and N/2 + 1)."""
    _r2c_interleaved_any(planner._sfx, x, out, planner, int(batch), in_stride, out_stride)


def c2r_interleaved_any_batch(spec, out, planner, batch: int, in_stride: int | None = None, out_stride: int | None = None) -> None:
    """c2r_any_batch from a flat 1-D complex torch CUDA tensor: member b reads N/2 + 1 bins at spec[b * in_stride:] (complex
    values) and writes N reals at out[b * out_stride:] (defaults: N/2 + 1 and N)."""
    _c2r_interleaved_any(planner._sfx, spec, out, planner, int(batch), in_stride, out_stride)


# ----------------------------------------------------------------------------------------------
# discrete cosine and sine transforms, types 2 and 3, of any length (scipy.fft.dct / dst)
# ----------------------------------------------------------------------------------------------
class _PlannerDct:
    _sfx = ""
    _dtype = None

    def __init__(self, n: int, device: int = 0, algo: AnyAlgo = AnyAlgo.Auto):
        """DCT / DST types 2 and 3 of length n >= 1 over an n-point real FFT (PlannerR2cAny's, built with `algo`, so with its
        limits and refusals: PhastFTPanic(13) before the device is touched for n = 0)."""
        self._h = C.c_void_p()
        self.device = int(device)
        check(fn("phastft_plan_dct_{s}_create_with", self._sfx)(int(n), self.device, int(algo), C.byref(self._h)))
        self.n = int(n)

    def describe(self) -> str:
        """"n=<N> <prec> dct | " followed by the inner real plan's describe()."""
        return fn("phastft_plan_dct_{s}_describe", self._sfx)(self._h).decode()

    def reserve(self, batch: int) -> None:
        """Make every allocation a call of `batch` members would make now (otherwise the first larger call makes them,
        synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_dct_{s}_reserve", self._sfx)(self._h, int(batch)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_dct_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerDct64(_PlannerDct):
    _sfx, _dtype = "f64", np.float64


class PlannerDct32(_PlannerDct):
    _sfx, _dtype = "f32", np.float32


_NORMS = {None: 0, "backward": 0, "ortho": 1, "forward": 2}


def _r2r_kind(sine: bool, type, norm):
    """(kind, norm) codes of include/phastft_cuda.h (PHASTFT_R2R_*, PHASTFT_NORM_*)"""
    if isinstance(type, bool) or not isinstance(type, (int, np.integer)) or type not in (2, 3):
        raise ValueError(f"type must be 2 or 3, got {type!r}")
    if norm not in _NORMS:
        raise ValueError(f"norm must be 'backward', 'ortho' or 'forward', got {norm!r}")
    return int(type) - 2 + 2 * sine, _NORMS[norm]


def _r2r(sine, x, out, planner, batch, type, norm, in_stride, out_stride):
    kind, nc = _r2r_kind(sine, type, norm)
    if not (_is_torch(x) and _is_torch(out)):
        raise TypeError("expected 1-D torch CUDA tensors (use dct_*_with_planner for numpy arrays)")
    n = planner.n
    in_stride = n if in_stride is None else int(in_stride)
    out_stride = n if out_stride is None else int(out_stride)
    px, nx = _torch_ptr(x, planner._dtype)
    po, no = _torch_ptr(out, planner._dtype)
    _check_batch_len("input", nx, batch, in_stride, n)
    _check_batch_len("output", no, batch, out_stride, n)
    check(fn("phastft_dct_{s}_dev", planner._sfx)(planner._h, kind, nc, px, in_stride, po, out_stride, int(batch), _torch_stream(x)))


def _r2r_with_planner(sfx, sine, x, out, planner, type, norm):
    if planner._sfx != sfx:
        raise TypeError("planner precision does not match the function")
    kind, nc = _r2r_kind(sine, type, norm)
    if _is_torch(x) != _is_torch(out):
        raise TypeError("pass the input and the output both as numpy arrays or both as torch CUDA tensors")
    if _is_torch(x):
        _torch_ptr(x, planner._dtype)
        _torch_ptr(out, planner._dtype)
        if x.numel() != planner.n:
            raise PhastFTPanic(5)
        if out.numel() != planner.n:
            raise PhastFTPanic(8)
        _r2r(sine, x, out, planner, 1, type, norm, None, None)
        return
    px, nx = _np_ptr(x, planner._dtype, False)
    po, no = _np_ptr(out, planner._dtype, True)
    if nx != planner.n:
        raise PhastFTPanic(5)
    if no != planner.n:
        raise PhastFTPanic(8)
    check(fn("phastft_dct_{s}_host", sfx)(planner._h, kind, nc, px, nx, po, no))


def dct_f64_with_planner(x, out, planner: PlannerDct64, type: int = 2, norm: str = "backward") -> None:
    """scipy.fft.dct(x, type, norm=norm) of N = planner.n values into out: float64 numpy arrays (synchronous) or 1-D torch CUDA
    tensors (torch's current stream).  out may be x.  scipy.fft.idct(X, type=2, norm=m) is type=3 with the inverse norm
    ("backward" <-> "forward", "ortho" itself), and idct of type 3 is type 2."""
    _r2r_with_planner("f64", False, x, out, planner, type, norm)


def dct_f32_with_planner(x, out, planner: PlannerDct32, type: int = 2, norm: str = "backward") -> None:
    _r2r_with_planner("f32", False, x, out, planner, type, norm)


def dst_f64_with_planner(x, out, planner: PlannerDct64, type: int = 2, norm: str = "backward") -> None:
    """scipy.fft.dst(x, type, norm=norm), as dct_f64_with_planner."""
    _r2r_with_planner("f64", True, x, out, planner, type, norm)


def dst_f32_with_planner(x, out, planner: PlannerDct32, type: int = 2, norm: str = "backward") -> None:
    _r2r_with_planner("f32", True, x, out, planner, type, norm)


def dct_batch(x, out, planner, batch: int, type: int = 2, norm: str = "backward", in_stride: int | None = None,
              out_stride: int | None = None) -> None:
    """`batch` DCTs on flat 1-D torch CUDA tensors: member b reads N values at x[b * in_stride:] and writes N at
    out[b * out_stride:] (defaults: N; any strides >= N, any offsets; out may be x with equal strides)."""
    _r2r(False, x, out, planner, int(batch), type, norm, in_stride, out_stride)


def dst_batch(x, out, planner, batch: int, type: int = 2, norm: str = "backward", in_stride: int | None = None,
              out_stride: int | None = None) -> None:
    """dct_batch for the DST."""
    _r2r(True, x, out, planner, int(batch), type, norm, in_stride, out_stride)


# ----------------------------------------------------------------------------------------------
# linear convolution and cross-correlation of real or complex signals (scipy.signal.fftconvolve / correlate)
# ----------------------------------------------------------------------------------------------
_CONV_MODES = {"full": 0, "same": 1, "valid": 2}


class _PlannerConv:
    _sfx = ""
    _dtype = None

    def __init__(self, n_x: int, n_h: int, device: int = 0, complex: bool = False):
        """Convolution and correlation of n_x values with n_h values (both >= 1), real or complex (interleaved complex128 /
        complex64), over an L-point transform, L = 2^ceil(log2(n_x + n_h - 1)) but at least 4 (`fft_len`).  n_x or n_h of 0,
        or L above 2^31 (real) / 2^30 (complex), raise PhastFTPanic(13) before the device is touched."""
        self._h = C.c_void_p()
        self.device = int(device)
        self.complex = bool(complex)
        check(fn("phastft_plan_conv_{s}_create", self._sfx)(int(n_x), int(n_h), int(self.complex), self.device, C.byref(self._h)))
        self.n_x, self.n_h = int(n_x), int(n_h)

    @property
    def fft_len(self) -> int:
        """L, the length of the transforms the plan runs."""
        return int(fn("phastft_plan_conv_{s}_fft_len", self._sfx)(self._h))

    def out_len(self, mode: str = "full") -> int:
        """The output length of `mode`: n_x + n_h - 1 (full), n_x (same) or |n_x - n_h| + 1 (valid)."""
        from ._lib import conv_out_len
        return conv_out_len(self.n_x, self.n_h, _conv_mode(mode))

    def describe(self) -> str:
        """"n_x=<n_x> n_h=<n_h> <prec> conv <real|complex> L=2^<k> | " followed by the inner plan's describe()."""
        return fn("phastft_plan_conv_{s}_describe", self._sfx)(self._h).decode()

    def reserve(self, batch: int) -> None:
        """Make every allocation a call of `batch` pairwise members would make now (otherwise the first larger call makes
        them, synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_conv_{s}_reserve", self._sfx)(self._h, int(batch)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_conv_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerConv64(_PlannerConv):
    _sfx, _dtype = "f64", np.float64


class PlannerConv32(_PlannerConv):
    _sfx, _dtype = "f32", np.float32


def _conv_mode(mode) -> int:
    if not isinstance(mode, str) or mode not in _CONV_MODES:
        raise ValueError(f"mode must be 'full', 'same' or 'valid', got {mode!r}")
    return _CONV_MODES[mode]


def _conv_operand(planner, a, what: str, on_device: bool):
    """`a` checked against the planner: a contiguous 1-D torch CUDA tensor (on_device) or numpy array of its dtype (float64 /
    float32, or complex128 / complex64 for a complex planner).  A wrong dtype raises ValueError, a wrong kind TypeError."""
    cplx = planner.complex
    if on_device:
        import torch
        if not _is_torch(a) or not a.is_cuda:
            raise TypeError(f"{what}: pass every operand as a torch CUDA tensor, or every one as a numpy array")
        want = {("f64", False): torch.float64, ("f32", False): torch.float32,
                ("f64", True): torch.complex128, ("f32", True): torch.complex64}[(planner._sfx, cplx)]
        if a.dtype != want:
            raise ValueError(f"{what}: expected dtype {want} for this planner, got {a.dtype}")
        if a.dim() != 1 or not a.is_contiguous():
            raise ValueError(f"{what}: expected a contiguous 1-D tensor")
        return a
    if not isinstance(a, np.ndarray):
        raise TypeError(f"{what}: pass every operand as a torch CUDA tensor, or every one as a numpy array")
    want = np.dtype({("f64", False): np.float64, ("f32", False): np.float32,
                     ("f64", True): np.complex128, ("f32", True): np.complex64}[(planner._sfx, cplx)])
    if a.dtype != want:
        raise ValueError(f"{what}: expected dtype {want} for this planner, got {a.dtype}")
    if a.ndim != 1 or not a.flags.c_contiguous:
        raise ValueError(f"{what}: expected a contiguous 1-D array")
    return a


def _conv_dev(op, x, h, out, planner, batch, mode, x_stride, h_stride, out_stride):
    """One device call on torch tensors; a complex operand whose pointer is not pair-aligned goes through an aligned copy."""
    def aligned(t):
        return not planner.complex or _pair_aligned(t)
    xs = x if aligned(x) else x.clone()
    hs = h if aligned(h) else h.clone()
    work = out if aligned(out) else out.clone()   # the clone keeps what lies between members
    check(fn("phastft_conv_{s}_dev", planner._sfx)(planner._h, op, mode, C.c_void_p(xs.data_ptr()), x_stride,
                                                   C.c_void_p(hs.data_ptr()), h_stride, C.c_void_p(work.data_ptr()), out_stride,
                                                   int(batch), _torch_stream(out)))
    if work is not out:
        out.copy_(work)


def _conv_with_planner(op, x, h, out, planner, mode):
    m = _conv_mode(mode)
    if not isinstance(planner, _PlannerConv):
        raise TypeError("expected a PlannerConv64 or PlannerConv32")
    on_device = _is_torch(out)
    x = _conv_operand(planner, x, "x", on_device)
    h = _conv_operand(planner, h, "h", on_device)
    out = _conv_operand(planner, out, "out", on_device)
    n_y = planner.out_len(mode)
    for what, a, n in (("x", x, planner.n_x), ("h", h, planner.n_h), ("out", out, n_y)):
        have = a.numel() if on_device else a.size
        if have != n:
            raise ValueError(f"{what} has {have} values, the planner expects {n}")
    if on_device:
        _conv_dev(op, x, h, out, planner, 1, m, planner.n_x, planner.n_h, n_y)
        return
    if not out.flags.writeable:
        raise ValueError("out is read-only")
    check(fn("phastft_conv_{s}_host", planner._sfx)(planner._h, op, m, x.ctypes.data_as(C.c_void_p), x.size,
                                                    h.ctypes.data_as(C.c_void_p), h.size, out.ctypes.data_as(C.c_void_p), out.size))


def _conv_batch(op, x, h, out, planner, batch, mode, x_stride, h_stride, out_stride):
    m = _conv_mode(mode)
    if not isinstance(planner, _PlannerConv):
        raise TypeError("expected a PlannerConv64 or PlannerConv32")
    x = _conv_operand(planner, x, "x", True)
    h = _conv_operand(planner, h, "h", True)
    out = _conv_operand(planner, out, "out", True)
    batch = int(batch)
    if batch < 0:
        raise ValueError("batch < 0")
    n_y = planner.out_len(mode)
    x_stride = planner.n_x if x_stride is None else int(x_stride)
    h_stride = planner.n_h if h_stride is None else int(h_stride)
    out_stride = n_y if out_stride is None else int(out_stride)
    for what, a, stride, n in (("x", x, x_stride, planner.n_x), ("h", h, h_stride, planner.n_h), ("out", out, out_stride, n_y)):
        if batch and a.numel() < (batch - 1) * stride + n:
            raise ValueError(f"{what} has {a.numel()} values, fewer than (batch - 1) * stride + {n}")
    _conv_dev(op, x, h, out, planner, batch, m, x_stride, h_stride, out_stride)


def convolve_with_planner(x, h, out, planner, mode: str = "full") -> None:
    """scipy.signal.fftconvolve(x, h, mode) into out: numpy arrays (synchronous) or 1-D torch CUDA tensors (torch's current
    stream) of the planner's dtype, with len(x) == planner.n_x, len(h) == planner.n_h and len(out) == planner.out_len(mode).
    out may be x or h (when the lengths allow)."""
    _conv_with_planner(0, x, h, out, planner, mode)


def correlate_with_planner(x, h, out, planner, mode: str = "full") -> None:
    """scipy.signal.correlate(x, h, mode) into out: convolve_with_planner with conj(h reversed)."""
    _conv_with_planner(1, x, h, out, planner, mode)


def convolve_batch(x, h, out, planner, batch: int, mode: str = "full", x_stride: int | None = None, h_stride: int | None = None,
                   out_stride: int | None = None) -> None:
    """`batch` convolutions on flat 1-D torch CUDA tensors: member b convolves x[b * x_stride:][:n_x] with h[b * h_stride:][:n_h]
    (h_stride 0: one filter for every member) into out[b * out_stride:][:out_len(mode)].  Defaults: n_x, n_h, out_len(mode);
    strides in values (complex ones for a complex planner)."""
    _conv_batch(0, x, h, out, planner, batch, mode, x_stride, h_stride, out_stride)


def correlate_batch(x, h, out, planner, batch: int, mode: str = "full", x_stride: int | None = None, h_stride: int | None = None,
                    out_stride: int | None = None) -> None:
    """convolve_batch for scipy.signal.correlate."""
    _conv_batch(1, x, h, out, planner, batch, mode, x_stride, h_stride, out_stride)


# ----------------------------------------------------------------------------------------------
# short-time Fourier transform and its inverse (torch.stft(..., return_complex=True) / torch.istft(..., length=n))
# ----------------------------------------------------------------------------------------------
_STFT_PAD = {"reflect": 0, "constant": 1}


class _PlannerStft:
    _sfx = ""
    _dtype = None

    def __init__(self, n: int, n_fft: int, hop_length: int | None = None, win_length: int | None = None, window=None,
                 center: bool = True, pad_mode: str = "reflect", device: int = 0, complex: bool = False):
        """torch.stft / torch.istft of signals of n values (real, or interleaved complex128 / complex64 with complex=True):
        frames of n_fft values hop_length apart (default n_fft // 4), the window's win_length values (default n_fft; window
        None: ones) centred in n_fft, and with center the signal padded by n_fft // 2 values on each side (pad_mode "reflect"
        or "constant").  n_frames frames of n_bins bins (n_fft // 2 + 1 real, n_fft complex).  A bad pad_mode or a window of
        another length raises ValueError; what the library refuses (hop 0, win_length above n_fft, reflect padding of n_fft // 2
        >= n, n < n_fft without center, ...) raises PhastFTPanic(13) before the device is touched."""
        self._h = C.c_void_p()
        n_fft = int(n_fft)
        hop_length = n_fft // 4 if hop_length is None else int(hop_length)
        win_length = n_fft if win_length is None else int(win_length)
        if not isinstance(pad_mode, str) or pad_mode not in _STFT_PAD:
            raise ValueError(f"pad_mode must be 'reflect' or 'constant', got {pad_mode!r}")
        w = None
        if window is not None:
            if _is_torch(window):
                window = window.detach().cpu().numpy()
            w = np.ascontiguousarray(np.asarray(window, dtype=self._dtype))
            if w.ndim != 1 or w.size != win_length:
                raise ValueError(f"window must be 1-D with win_length = {win_length} values, got shape {w.shape}")
        self.device = int(device)
        self.complex = bool(complex)
        check(fn("phastft_plan_stft_{s}_create", self._sfx)(int(n), n_fft, hop_length,
                                                           None if w is None else w.ctypes.data_as(C.c_void_p), win_length,
                                                           int(bool(center)), _STFT_PAD[pad_mode], int(self.complex), self.device,
                                                           C.byref(self._h)))
        self.n, self.n_fft, self.hop_length, self.win_length = int(n), n_fft, hop_length, win_length
        self.center, self.pad_mode = bool(center), pad_mode

    @property
    def n_frames(self) -> int:
        """F = 1 + (n + 2 pad - n_fft) // hop_length, pad = n_fft // 2 with center, else 0."""
        return int(fn("phastft_plan_stft_{s}_frames", self._sfx)(self._h))

    @property
    def n_bins(self) -> int:
        """n_fft // 2 + 1 (real signals) or n_fft (complex)."""
        return int(fn("phastft_plan_stft_{s}_bins", self._sfx)(self._h))

    def describe(self) -> str:
        """"n=<n> n_fft=<n_fft> hop=<hop> <prec> stft <real|complex> F=<F> | " followed by the inner plan's describe()."""
        return fn("phastft_plan_stft_{s}_describe", self._sfx)(self._h).decode()

    def reserve(self, batch: int) -> None:
        """Make every allocation a call of `batch` signals would make now (otherwise the first larger call makes them,
        synchronising the device -- an error inside a CUDA-graph capture)."""
        check(fn("phastft_plan_stft_{s}_reserve", self._sfx)(self._h, int(batch)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                fn("phastft_plan_stft_{s}_destroy", self._sfx)(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the module globals are already gone
                pass


class PlannerStft64(_PlannerStft):
    _sfx, _dtype = "f64", np.float64


class PlannerStft32(_PlannerStft):
    _sfx, _dtype = "f32", np.float32


def _stft_dtypes(planner):
    """(signal dtype, spectrum dtype) as numpy dtypes"""
    cdt = np.complex128 if planner._sfx == "f64" else np.complex64
    return np.dtype(cdt if planner.complex else planner._dtype), np.dtype(cdt)


def _torch_dtype(dt):
    import torch
    return {np.dtype(np.float64): torch.float64, np.dtype(np.float32): torch.float32,
            np.dtype(np.complex128): torch.complex128, np.dtype(np.complex64): torch.complex64}[np.dtype(dt)]


def _normalized(normalized) -> int:
    if isinstance(normalized, (bool, np.bool_)) or normalized in (0, 1):
        return int(bool(normalized))
    raise ValueError(f"normalized must be a bool, got {normalized!r}")


def _sig_stride(t, n: int):
    """member stride of a (..., n) tensor whose last dimension is unit-stride and whose leading dimensions flatten to one
    stride >= n, else None"""
    if n > 1 and t.stride(-1) != 1:
        return None
    cands, inner = [], 1
    for size, st in reversed(list(zip(t.shape[:-1], t.stride()[:-1]))):
        if size > 1:
            if st % inner:
                return None
            cands.append(st // inner)
        inner *= size
    s = cands[0] if cands else n
    return s if s >= n and all(c == s for c in cands) else None


def _frame_stride(t, bins: int, frames: int):
    """frame stride fs of a (..., bins, F) spectrum whose element (b, k, f) lies at (b F + f) fs + k (torch.stft's layout, b
    the flattened leading index, fs >= bins), else None"""
    if bins > 1 and t.stride(-2) != 1:
        return None
    cands, inner = [], frames
    if frames > 1:
        cands.append(t.stride(-1))
    for size, st in reversed(list(zip(t.shape[:-2], t.stride()[:-2]))):
        if size > 1:
            if st % inner:
                return None
            cands.append(st // inner)
        inner *= size
    fs = cands[0] if cands else bins
    return fs if fs >= bins and all(c == fs for c in cands) else None


def _stft_torch(inverse: bool, sig, spec, planner, normalized: int):
    """One device call on torch CUDA tensors sig (..., n) and spec (..., n_bins, F) with the same leading shape.  A tensor in
    another layout, or a complex one that is not aligned to its element size, goes through a temporary."""
    import torch
    sdt, cdt = _stft_dtypes(planner)
    n, bins, F = planner.n, planner.n_bins, planner.n_frames
    for what, t, want in (("signal", sig, sdt), ("spectrum", spec, cdt)):
        if not _is_torch(t) or not t.is_cuda:
            raise TypeError(f"{what}: pass both arrays as torch CUDA tensors, or both as numpy arrays")
        if t.dtype != _torch_dtype(want):
            raise ValueError(f"{what}: expected dtype {_torch_dtype(want)} for this planner, got {t.dtype}")
    if sig.dim() < 1 or sig.shape[-1] != n:
        raise ValueError(f"the signal has shape {tuple(sig.shape)}, the planner expects (..., {n})")
    lead = tuple(sig.shape[:-1])
    if tuple(spec.shape) != lead + (bins, F):
        raise ValueError(f"the spectrum has shape {tuple(spec.shape)}, the planner expects {lead + (bins, F)}")
    batch = int(np.prod(lead, dtype=np.int64)) if lead else 1

    def aligned(t):
        return not t.is_complex() or t.data_ptr() % t.element_size() == 0
    ss = _sig_stride(sig, n) if aligned(sig) else None
    fs = _frame_stride(spec, bins, F) if aligned(spec) else None
    sig_w = sig if ss is not None else torch.empty((batch, n), dtype=sig.dtype, device=sig.device)
    spec_w = spec if fs is not None else torch.empty((batch, F, bins), dtype=spec.dtype, device=spec.device).transpose(1, 2)
    if inverse and fs is None:
        spec_w.copy_(spec.reshape(batch, bins, F))
    if not inverse and ss is None:
        sig_w.copy_(sig.reshape(batch, n))
    ss = n if ss is None else ss
    fs = bins if fs is None else fs
    name = "phastft_istft_{s}_dev" if inverse else "phastft_stft_{s}_dev"
    a, b, sa, sb = (spec_w, sig_w, fs, ss) if inverse else (sig_w, spec_w, ss, fs)
    check(fn(name, planner._sfx)(planner._h, normalized, C.c_void_p(a.data_ptr()), sa, C.c_void_p(b.data_ptr()), sb, batch,
                                 _torch_stream(spec)))
    if inverse and sig_w is not sig:
        sig.copy_(sig_w.reshape(sig.shape))
    if not inverse and spec_w is not spec:
        spec.copy_(spec_w.reshape(spec.shape))


def _stft_numpy(inverse: bool, sig, spec, planner, normalized: int):
    """One synchronous host call on a 1-D numpy signal and an (n_bins, F) numpy spectrum."""
    sdt, cdt = _stft_dtypes(planner)
    n, bins, F = planner.n, planner.n_bins, planner.n_frames
    for what, a, want in (("signal", sig, sdt), ("spectrum", spec, cdt)):
        if not isinstance(a, np.ndarray):
            raise TypeError(f"{what}: pass both arrays as torch CUDA tensors, or both as numpy arrays")
        if a.dtype != want:
            raise ValueError(f"{what}: expected dtype {want} for this planner, got {a.dtype}")
    if sig.shape != (n,):
        raise ValueError(f"the signal has shape {sig.shape}, the planner expects ({n},)")
    if spec.shape != (bins, F):
        raise ValueError(f"the spectrum has shape {spec.shape}, the planner expects ({bins}, {F})")
    out = spec if not inverse else sig
    if not out.flags.writeable:
        raise ValueError("the output array is read-only")
    direct = spec.T.flags.c_contiguous
    frames = spec.T if direct else np.ascontiguousarray(spec.T)   # F x bins, dense
    s = sig if sig.flags.c_contiguous else np.ascontiguousarray(sig)
    if inverse:
        check(fn("phastft_istft_{s}_host", planner._sfx)(planner._h, normalized, frames.ctypes.data_as(C.c_void_p), frames.size,
                                                         s.ctypes.data_as(C.c_void_p), s.size))
        if s is not sig:
            sig[...] = s
    else:
        check(fn("phastft_stft_{s}_host", planner._sfx)(planner._h, normalized, s.ctypes.data_as(C.c_void_p), s.size,
                                                        frames.ctypes.data_as(C.c_void_p), frames.size))
        if not direct:
            spec[...] = frames.T


def _stft_call(inverse: bool, sig, spec, planner, normalized, batched: bool):
    if not isinstance(planner, _PlannerStft):
        raise TypeError("expected a PlannerStft64 or PlannerStft32")
    nz = _normalized(normalized)
    if _is_torch(sig) or _is_torch(spec):
        if not batched and (getattr(sig, "dim", lambda: 0)() != 1):
            raise ValueError("stft_with_planner / istft_with_planner take one signal: use stft_batch / istft_batch for more")
        _stft_torch(inverse, sig, spec, planner, nz)
    elif batched:
        raise TypeError("stft_batch / istft_batch take torch CUDA tensors")
    else:
        _stft_numpy(inverse, sig, spec, planner, nz)


def stft_with_planner(x, out, planner, normalized: bool = False) -> None:
    """torch.stft(x, ..., return_complex=True) of one signal into out: x of n values (float64 / float32, or complex128 /
    complex64 for a complex planner) and out of shape (n_bins, n_frames), complex.  numpy arrays (synchronous, through a
    staging buffer) or torch CUDA tensors (torch's current stream); out in any other layout than torch.stft's (unit bin
    stride) goes through a temporary."""
    _stft_call(False, x, out, planner, normalized, False)


def istft_with_planner(spec, out, planner, normalized: bool = False) -> None:
    """torch.istft(spec, ..., length=n) of one spectrum of shape (n_bins, n_frames) into out of n values (real, or complex for
    a complex planner); numpy arrays or torch CUDA tensors.  spec is not written.  A plan whose window fails the NOLA
    condition raises PhastFTPanic(13) naming the first sample where the overlap-add envelope is below 1e-11."""
    _stft_call(True, out, spec, planner, normalized, False)


def stft_batch(x, out, planner, normalized: bool = False) -> None:
    """stft_with_planner over torch CUDA tensors x (..., n) and out (..., n_bins, n_frames): one device call when out has
    torch.stft's layout and the leading dimensions of each flatten to one stride."""
    _stft_call(False, x, out, planner, normalized, True)


def istft_batch(spec, out, planner, normalized: bool = False) -> None:
    """istft_with_planner over torch CUDA tensors spec (..., n_bins, n_frames) and out (..., n)."""
    _stft_call(True, out, spec, planner, normalized, True)
