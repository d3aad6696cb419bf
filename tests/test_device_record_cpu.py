"""CPU-side checks of the device record API (include/loghisto_b200_device.cuh, lh_recorder in include/loghisto_b200.h):
the struct layout as C sees it, and that the device header compiles, links and allocates as a library user needs."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

needs_nvcc = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")


def test_recorder_layout_matches_ctypes(tmp_path):
    from loghisto_b200 import _lib
    cls = _lib.lh_recorder
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "loghisto_b200.h"', 'int main(void) {',
           'printf("size %zu\\n", sizeof(lh_recorder));']
    for f, _ in cls._fields_:
        src.append('printf("%s %%zu\\n", offsetof(lh_recorder, %s));' % (f, f))
    src.append('return 0; }')
    c = tmp_path / "rec.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "rec"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", INC, "-o", str(exe), str(c)],
                   check=True)
    want = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert ctypes.sizeof(cls) == int(want["size"]) == 104
    for f, _ in cls._fields_:
        assert getattr(cls, f).offset == int(want[f]), f


A_CU = r'''
#include "loghisto_b200_device.cuh"
__global__ void k_a(lh_recorder rec, const double *v, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { lh::record(rec, 0, v[i]); lh::count(rec, 1, 2); }
}
void launch_a(const lh_recorder &rec, const double *v, int n) { k_a<<<1, 32>>>(rec, v, n); }
'''
B_CU = r'''
#include "loghisto_b200_device.cuh"
__global__ void k_b(lh_recorder rec, const long long *v, int n) {
    extern __shared__ unsigned char smem[];
    lh::BlockHistogram bh(rec, smem);
    bh.init(2);
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { lh::record_ns(rec, 1, v[i]); bh.add((double)v[i]); }
    bh.flush();
}
void launch_a(const lh_recorder &rec, const double *v, int n);
int main() {
    lh_recorder rec = {};
    launch_a(rec, nullptr, 0);
    k_b<<<1, 32, rec.block_smem_bytes>>>(rec, nullptr, 0);
    return 0;
}
'''


@needs_nvcc
def test_device_header_links_from_two_translation_units_with_rdc(tmp_path):
    """Every function of the header has internal or inline linkage: two TUs that both include it link with -rdc=true."""
    (tmp_path / "a.cu").write_text(A_CU)
    (tmp_path / "b.cu").write_text(B_CU)
    exe = str(tmp_path / "two_tu")
    res = subprocess.run([NVCC] + ARCH + ["-std=c++17", "-rdc=true", "-I", INC, str(tmp_path / "a.cu"), str(tmp_path / "b.cu"),
                          "-o", exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    # and without relocatable device code
    res = subprocess.run([NVCC] + ARCH + ["-std=c++17", "-I", INC, str(tmp_path / "a.cu"), str(tmp_path / "b.cu"),
                          "-o", exe + "_whole"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


@needs_nvcc
def test_client_kernels_do_not_spill(tmp_path):
    res = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-shared", "-I", INC,
                          os.path.join(ROOT, "tests", "device_record_client.cu"), "-o", str(tmp_path / "client.so")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    log = res.stdout + res.stderr
    entries = re.findall(r"Compiling entry function '([^']+)'", log)
    assert len(entries) == 5, entries          # record, record_subset, record_ns, count, block
    spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", log)]
    assert spills and not any(spills), log
    frames = [int(x) for x in re.findall(r"(\d+) bytes stack frame", log)]
    assert not any(frames), log


def test_recorder_abi_is_bound():
    """record_begin / record_end are part of the ctypes surface (the header-vs-binding check of test_abi covers
    their presence); the Engine exposes them with a context manager."""
    from loghisto_b200 import _lib, engine
    assert "lh_record_begin" in _lib.SIGNATURES and "lh_record_end" in _lib.SIGNATURES
    for name in ("record_begin", "record_end", "recording"):
        assert callable(getattr(engine.Engine, name))
