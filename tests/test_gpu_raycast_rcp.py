"""The ray cast divides by the cell size as a multiply by rcp.approx.ftz(cell), computed once per ray (kt_raycast.cu, rcp_approx).
That is bit-exact only because `x / cell`, compiled with the library's numerics flags (--ftz=true --prec-div=false), is itself
x * rcp(cell) whenever |cell| <= 2^126.  These tests check that premise on the device, over a seeded spread of coordinates and the
cell sizes the tracker uses, and that the ray cast refuses a cell size outside the range."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KERNEL = r"""
#include <cstdint>
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__global__ void cmp(const float* x, long long n, const float* cells, int ncell, unsigned long long* bad, long long* first)
{
    for (int k = 0; k < ncell; ++k) {
        const float c = cells[k], r = rcp_approx(c);
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
            if (__float_as_uint(x[i] / c) != __float_as_uint(__fmul_rn(x[i], r))) {
                atomicAdd(bad, 1ull);
                atomicMin(first, (long long)k * n + i);
            }
        }
    }
}
extern "C" int rcp_check(const float* x, long long n, const float* cells, int ncell, unsigned long long* bad, long long* first)
{
    cmp<<<1024, 256>>>(x, n, cells, ncell, bad, first);
    return (int)cudaDeviceSynchronize();
}
"""


def _numerics_flags():
    """-O3, the architecture and the float numerics flags of the library's build (kintinuous_b200/csrc/Makefile)."""
    mk = open(os.path.join(ROOT, "kintinuous_b200", "csrc", "Makefile")).read()
    arch = re.search(r"^ARCH := (.*)$", mk, re.M).group(1).split()
    flags = re.search(r"^NVFLAGS := (.*)$", mk, re.M).group(1).split()
    keep = [f for f in flags if f == "-O3" or f.startswith("--ftz") or f.startswith("--prec-") or f.startswith("--fmad")]
    assert any(f.startswith("--prec-div") for f in keep), flags
    return keep + arch


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    d = tmp_path_factory.mktemp("rcp")
    src, lib = d / "rcp_check.cu", d / "librcp_check.so"
    src.write_text(KERNEL)
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.check_call([nvcc, *_numerics_flags(), "-Xcompiler", "-fPIC", "-shared", "-o", str(lib), str(src)])
    f = ctypes.CDLL(str(lib)).rcp_check
    f.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return f


def _coordinates(n, cells):
    """n seeded finite floats of both signs, log-uniform in magnitude from the smallest denormal to 1e4, plus every integer multiple
    of each cell size within +-2048 cells (the floor boundaries of getVoxel) and their float neighbours."""
    rng = np.random.default_rng(20261017)
    mag = np.exp2(rng.uniform(-149.0, np.log2(1e4), n)).astype(np.float32)
    x = np.where(rng.random(n) < 0.5, -mag, mag).astype(np.float32)
    k = np.arange(-2048, 2049, dtype=np.float32)
    mult = np.concatenate([k * np.float32(c) for c in cells]).astype(np.float32)
    edge = np.concatenate([mult, np.nextafter(mult, np.float32(np.inf)), np.nextafter(mult, np.float32(-np.inf)),
                           np.array([0.0, -0.0, 1e4, -1e4, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38], np.float32)])
    return np.concatenate([x, edge.astype(np.float32)])


def test_division_by_cell_is_multiply_by_rcp_approx(checker):
    import torch
    size = np.float32(6.0)
    cells = [size / np.float32(v) for v in (128, 256, 512, 1024, 2048)]
    cells += [np.float32(s) / np.float32(512) for s in (6.0, 4.5, 3.3)]           # a non-cubic volume_size at 512^3
    cells += [size / np.float32(300)]                                             # a resolution that is not a power of two
    cells = np.array(cells, np.float32)
    x = _coordinates(10_000_000, cells)
    assert np.isfinite(x).all()
    xd = torch.from_numpy(x).cuda()
    cd = torch.from_numpy(cells).cuda()
    bad = torch.zeros(1, dtype=torch.int64, device="cuda")
    first = torch.full((1,), 2**62, dtype=torch.int64, device="cuda")
    assert checker(xd.data_ptr(), x.size, cd.data_ptr(), cells.size, bad.data_ptr(), first.data_ptr()) == 0
    nbad = int(bad.item())
    if nbad:
        f = int(first.item())
        pytest.fail(f"{nbad} quotients differ; first: x = {x[f % x.size]!r}, cell = {cells[f // x.size]!r}")


def test_raycast_refuses_a_cell_size_above_2_pow_126(built):
    import torch
    import kintinuous_b200 as kb
    rows, cols, vol = 8, 16, 2
    intr = np.array([10.0, 10.0, 8.0, 4.0], np.float32)
    tsdf = torch.zeros(vol ** 3, dtype=torch.int16, device="cuda")
    color = torch.zeros(vol ** 3 * 4, dtype=torch.uint8, device="cuda")
    vmap = torch.zeros(3 * rows * cols, dtype=torch.float32, device="cuda")
    nmap = torch.zeros_like(vmap)
    vcol = torch.zeros(rows * cols * 4, dtype=torch.uint8, device="cuda")
    vs = np.full(3, 3e38, np.float32)                                             # cell 1.5e38 > 2^126
    with pytest.raises(kb.KtError, match="cell size"):
        kb.ops.raycast(intr, np.eye(3, dtype=np.float32), np.zeros(3, np.float32), 0.1, vs, tsdf, vol, vmap, nmap, rows, cols,
                       (0, 0, 0), vcol, color)
