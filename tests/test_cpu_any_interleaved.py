"""Interleaved complex FFTs of any length without a GPU: the Python functions refuse bad arguments before the library is
called, and cpp/phastft.hpp's PlannerAny interleaved members compile and link against the C ABI."""
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
    return types.SimpleNamespace(_sfx=sfx, _h=None, num_points=n, _dtype=np.float64 if sfx == "f64" else np.float32)


def test_python_argument_errors_before_the_library(pf):
    n = 1000
    p64, p32 = _stand_in("f64", n), _stand_in("f32", n)
    with pytest.raises(TypeError):                       # planner of the other precision
        pf.fft_64_interleaved_any_with_planner(np.zeros(n, np.complex128), pf.Direction.Forward, p32)
    with pytest.raises(TypeError):                       # dtype of the other precision
        pf.fft_32_interleaved_any_with_planner(np.zeros(n, np.complex128), pf.Direction.Forward, p32)
    with pytest.raises(TypeError):                       # real data
        pf.fft_64_interleaved_any_with_planner(np.zeros(n, np.float64), pf.Direction.Forward, p64)
    with pytest.raises(TypeError):                       # not contiguous
        pf.fft_64_interleaved_any_with_planner(np.zeros(2 * n, np.complex128)[::2], pf.Direction.Forward, p64)
    with pytest.raises(TypeError):                       # not 1-D
        pf.fft_64_interleaved_any_with_planner(np.zeros((2, n // 2), np.complex128), pf.Direction.Forward, p64)
    for m in (n - 1, n + 1):
        with pytest.raises(pf.PhastFTPanic) as e:
            pf.fft_32_interleaved_any_with_planner(np.zeros(m, np.complex64), pf.Direction.Forward, p32)
        assert e.value.code == 3
    with pytest.raises(TypeError):                       # the batch function takes device tensors only
        pf.fft_interleaved_any_batch(np.zeros(3 * n, np.complex128), pf.Direction.Forward, p64, 3)
    torch = pytest.importorskip("torch")
    with pytest.raises(TypeError):                       # a host tensor
        pf.fft_64_interleaved_any_with_planner(torch.zeros(n, dtype=torch.complex128), pf.Direction.Forward, p64)
    with pytest.raises(TypeError):
        pf.fft_interleaved_any_batch(torch.zeros(n, dtype=torch.complex64), pf.Direction.Forward, p32, 1)


CPP = r"""
#include <complex>
#include <vector>
#include "phastft.hpp"

template <typename T>
void use(const phastft::detail::PlannerAny<T>& p, std::vector<std::complex<T>>& host, std::complex<T>* dev) {
    p.fft_interleaved(host.data(), host.size(), phastft::Direction::Forward);
    p.fft_interleaved_device(dev, phastft::Direction::Reverse, 4, 1001, nullptr);
}
template void use<double>(const phastft::PlannerAny64&, std::vector<std::complex<double>>&, std::complex<double>*);
template void use<float>(const phastft::PlannerAny32&, std::vector<std::complex<float>>&, std::complex<float>*);

int main() { return 0; }
"""


def test_cpp_interleaved_members_compile(pf, tmp_path):
    gxx = shutil.which("g++") or "/usr/bin/g++"
    src = tmp_path / "il.cpp"
    src.write_text(CPP)
    libdir = ROOT / "phastft_b200"
    subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", "-Werror", f"-I{ROOT / 'cpp'}", "-o", str(tmp_path / "il"), str(src),
                    f"-L{libdir}", "-lphastft_cuda", f"-Wl,-rpath,{libdir}"], check=True)
