"""The radix-32 stage table of the 1024-row pass tiles.

Strided tiles whose last stage is radix 32 read W_R^(m*i) from a per-plan [m][i] table in the plan's table blob instead of
building it in registers from five loads and 26 complex products.  These tests check that the table holds exactly the values
that product chain gives (evaluated here by a small device kernel written the way the stage computed them), that the blob's
header locates it, and that export / import carries it.
"""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HEADER = "<QQQIIQ3Q3Q"          # magic, bytes, n, precision_bits, num_passes, layout_sig, tw_stage_off[3], tw32_off[3]
MAGIC = 0x3354464854534150

# The radix-32 stage's twiddles as stage_from_tile derived them in registers: W^(m*i) loaded for i = 1, 2, 4, 8, 16 from the
# pass's W_R table, every other i the product of two earlier ones (i = hi + lo, hi the top bit of i).
CHAIN_SRC = r"""
#include "fft_device.cuh"
using namespace phast;
template <typename T>
__global__ void chain32(const cx<T>* tw_stage, cx<T>* out, int ns) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= ns) return;
    cx<T> w[32];
#pragma unroll
    for (int i = 1; i < 32; ++i) {
        const int hi = 1 << (31 - __builtin_clz((unsigned)i));
        if (i == hi) w[i] = __ldg(tw_stage + m * i);
        else w[i] = ctwid<T>(w[hi], w[i - hi]);
        out[m * 32 + i] = w[i];
    }
    out[m * 32] = tw_stage[0];
}
extern "C" int chain32_run(int f64, const void* tw_stage, void* out, int ns) {
    if (f64) chain32<double><<<(ns + 127) / 128, 128>>>((const double2*)tw_stage, (double2*)out, ns);
    else chain32<float><<<(ns + 127) / 128, 128>>>((const float2*)tw_stage, (float2*)out, ns);
    cudaError_t e = cudaDeviceSynchronize();
    return e == cudaSuccess ? (int)cudaGetLastError() : (int)e;
}
"""


@pytest.fixture(scope="module")
def chain_lib(tmp_path_factory):
    import __graft_entry__ as g
    d = tmp_path_factory.mktemp("chain32")
    src = d / "chain32.cu"
    src.write_text(CHAIN_SRC)
    so = d / "chain32.so"
    subprocess.run([g._nvcc(), *g.NVCC_FLAGS, f"-I{g.CSRC}", "-shared", "-o", str(so), str(src)], check=True)
    lib = C.CDLL(str(so))
    lib.chain32_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    lib.chain32_run.restype = C.c_int
    return lib


def _export(planner):
    import torch
    buf = torch.empty(planner.tables_bytes(), dtype=torch.uint8, device="cuda:0")
    planner.tables_export(buf)
    torch.cuda.synchronize()
    return buf


def _header(buf):
    f = struct.unpack(HEADER, bytes(buf[:struct.calcsize(HEADER)].cpu().numpy()))
    return {"magic": f[0], "bytes": f[1], "n": f[2], "bits": f[3], "passes": f[4], "tw_stage_off": f[6:9], "tw32_off": f[9:12]}


def _planner(pf, sfx, n):
    return (pf.PlannerDit64 if sfx == "f64" else pf.PlannerDit32)(n, 0)


@pytest.mark.parametrize("sfx", ["f64", "f32"])
def test_table_is_the_product_chain(sfx, chain_lib):
    import torch
    import phastft_b200 as pf
    n = 1 << 20
    planner = _planner(pf, sfx, n)
    buf = _export(planner)
    h = _header(buf)
    assert h["magic"] == MAGIC and h["n"] == n and h["passes"] == 2 and h["bytes"] == buf.numel()
    elem = 16 if sfx == "f64" else 8
    R = 1024                                           # 2^20 = 1024 x 1024: both passes end in a radix-32 stage
    for p in range(2):
        assert h["tw32_off"][p] > 0, (p, planner.describe())
        tw = buf[h["tw_stage_off"][p]:h["tw_stage_off"][p] + R * elem]
        table = buf[h["tw32_off"][p]:h["tw32_off"][p] + R * elem]
        want = torch.zeros(R * elem, dtype=torch.uint8, device="cuda:0")
        assert chain_lib.chain32_run(int(sfx == "f64"), tw.data_ptr(), want.data_ptr(), R // 32) == 0
        assert torch.equal(table, want), p


@pytest.mark.parametrize("sfx", ["f64", "f32"])
def test_export_import_carries_the_table(sfx):
    import torch
    import phastft_b200 as pf
    from phastft_b200._lib import PhastFTPanic
    n = 1 << 20
    dt = np.float64 if sfx == "f64" else np.float32
    fft = pf.fft_64_dit_with_planner if sfx == "f64" else pf.fft_32_dit_with_planner
    p0, p1 = _planner(pf, sfx, n), _planner(pf, sfx, n)
    rng = np.random.default_rng(7)
    re = rng.uniform(-1, 1, n).astype(dt); im = rng.uniform(-1, 1, n).astype(dt)

    def run(planner):
        a, b = re.copy(), im.copy()
        fft(a, b, pf.Direction.Forward, planner)
        return a, b

    want = run(p0)
    good = _export(p0)
    h = _header(good)
    elem = 16 if sfx == "f64" else 8
    # the kernels read the table out of the blob: an imported blob with zeroed radix-32 tables changes the transform ...
    bad = good.clone()
    for p in range(2):
        bad[h["tw32_off"][p]:h["tw32_off"][p] + 1024 * elem] = 0
    p1.tables_import(bad)
    torch.cuda.synchronize()
    got = run(p1)
    assert not np.array_equal(got[0], want[0])
    # ... and importing the exported one gives the exporting plan's transform bit for bit
    p1.tables_import(good)
    torch.cuda.synchronize()
    got = run(p1)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    # a header that places the table elsewhere is a different layout
    moved = good.clone()
    moved[64:72] = torch.tensor(list(struct.pack("<Q", h["tw32_off"][0] + 256)), dtype=torch.uint8, device="cuda:0")
    with pytest.raises(PhastFTPanic) as err:
        p1.tables_import(moved)
    assert err.value.code == 3 and "different pass decomposition" in str(err.value)   # PHASTFT_ERR_PLAN_MISMATCH
