"""Real FFTs of any length on interleaved spectra without a GPU: the Python functions refuse bad arguments before the library
is called, and cpp/phastft.hpp's PlannerR2cAny interleaved members compile and link against the C ABI."""
import shutil
import subprocess
import types
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def pf():
    import __graft_entry__ as g
    g.build()
    import phastft_b200
    return phastft_b200


def _stand_in(sfx, n):
    """A planner-shaped object whose handle is NULL: any argument check that reached the library would fail differently."""
    return types.SimpleNamespace(_sfx=sfx, _h=None, n=n, _dtype=np.float64 if sfx == "f64" else np.float32)


def test_python_argument_errors_before_the_library(pf):
    n = 1000
    bins = n // 2 + 1
    p64, p32 = _stand_in("f64", n), _stand_in("f32", n)
    x64, s64 = np.zeros(n), np.zeros(bins, np.complex128)
    with pytest.raises(TypeError):                       # planner of the other precision
        pf.r2c_fft_f64_interleaved_any_with_planner(x64, s64, p32)
    with pytest.raises(TypeError):
        pf.c2r_fft_f64_interleaved_any_with_planner(s64, x64, p32)
    with pytest.raises(TypeError):                       # spectrum dtype of the other precision
        pf.r2c_fft_f32_interleaved_any_with_planner(np.zeros(n, np.float32), s64, p32)
    with pytest.raises(TypeError):                       # real input of the other precision
        pf.r2c_fft_f64_interleaved_any_with_planner(np.zeros(n, np.float32), s64, p64)
    with pytest.raises(TypeError):                       # a real array where the spectrum goes
        pf.r2c_fft_f64_interleaved_any_with_planner(x64, np.zeros(2 * bins), p64)
    with pytest.raises(TypeError):                       # spectrum not contiguous
        pf.c2r_fft_f64_interleaved_any_with_planner(np.zeros(2 * bins, np.complex128)[::2], x64, p64)
    with pytest.raises(TypeError):                       # spectrum not 1-D
        pf.r2c_fft_f64_interleaved_any_with_planner(x64, np.zeros((1, bins), np.complex128), p64)
    with pytest.raises(ValueError):                      # real output not contiguous
        pf.c2r_fft_f64_interleaved_any_with_planner(s64, np.zeros(2 * n)[::2], p64)
    with pytest.raises(ValueError):                      # read-only spectrum output
        ro = np.zeros(bins, np.complex128)
        ro.flags.writeable = False
        pf.r2c_fft_f64_interleaved_any_with_planner(x64, ro, p64)
    with pytest.raises(TypeError):                       # the batch functions take device tensors only
        pf.r2c_interleaved_any_batch(np.zeros(3 * n), np.zeros(3 * bins, np.complex128), p64, 3)
    with pytest.raises(TypeError):
        pf.c2r_interleaved_any_batch(np.zeros(3 * bins, np.complex128), np.zeros(3 * n), p64, 3)
    torch = pytest.importorskip("torch")
    with pytest.raises(TypeError):                       # host tensors
        pf.r2c_fft_f64_interleaved_any_with_planner(torch.zeros(n, dtype=torch.float64), torch.zeros(bins, dtype=torch.complex128), p64)
    with pytest.raises(TypeError):
        pf.c2r_interleaved_any_batch(torch.zeros(bins, dtype=torch.complex64), torch.zeros(n), p32, 1)
    with pytest.raises(TypeError):                       # numpy input with a torch output
        pf.r2c_fft_f64_interleaved_any_with_planner(x64, torch.zeros(bins, dtype=torch.complex128), p64)
    with pytest.raises(TypeError):                       # torch input with a numpy output
        pf.c2r_fft_f64_interleaved_any_with_planner(torch.zeros(bins, dtype=torch.complex128), x64, p64)


CPP = r"""
#include <complex>
#include <vector>
#include "phastft.hpp"

template <typename T>
void use(const phastft::detail::PlannerR2cAny<T>& p, const std::vector<T>& x, std::vector<std::complex<T>>& spec, std::vector<T>& y,
         const T* d_x, std::complex<T>* d_spec, T* d_y) {
    p.r2c_interleaved(x, spec);
    p.c2r_interleaved(spec, y);
    p.r2c_interleaved_device(d_x, 1000, d_spec, 501, 4, nullptr);
    p.c2r_interleaved_device(d_spec, 501, d_y, 1000, 4, nullptr);
}
template void use<double>(const phastft::PlannerR2cAny64&, const std::vector<double>&, std::vector<std::complex<double>>&,
                          std::vector<double>&, const double*, std::complex<double>*, double*);
template void use<float>(const phastft::PlannerR2cAny32&, const std::vector<float>&, std::vector<std::complex<float>>&,
                         std::vector<float>&, const float*, std::complex<float>*, float*);

int main() { return 0; }
"""


def test_cpp_interleaved_members_compile(pf, tmp_path):
    gxx = shutil.which("g++") or "/usr/bin/g++"
    src = tmp_path / "ril.cpp"
    src.write_text(CPP)
    libdir = ROOT / "phastft_b200"
    subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", "-Werror", f"-I{ROOT / 'cpp'}", "-o", str(tmp_path / "ril"), str(src),
                    f"-L{libdir}", "-lphastft_cuda", f"-Wl,-rpath,{libdir}"], check=True)
