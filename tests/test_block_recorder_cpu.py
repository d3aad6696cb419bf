"""CPU-side checks of lh::BlockRecorder (include/loghisto_b200_device.cuh): it links from two translation units with
-rdc=true, the client kernels of tests/block_recorder_client.cu do not spill, and smem_bytes() sizes the table as the
header documents, evaluated on the host."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")

A_CU = r'''
#include "loghisto_b200_device.cuh"
__global__ void k_a(lh_recorder rec, const double *v, int n) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, 1024);
    br.init();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { br.record(i & 7, v[i]); lh::record(rec, 0, v[i]); }
    br.flush();
}
void launch_a(const lh_recorder &rec, const double *v, int n) {
    k_a<<<1, 32, lh::BlockRecorder::smem_bytes(1024)>>>(rec, v, n);
}
'''
B_CU = r'''
#include "loghisto_b200_device.cuh"
__global__ void k_b(lh_recorder rec, const long long *v, int n) {
    extern __shared__ __align__(16) unsigned char smem[];
    lh::BlockRecorder br(rec, smem, 64);
    br.init();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    lh::TimerToken t = lh::start_timer(3);
    if (i < n) { br.record_ns(1, v[i]); br.stop(t); }
    br.flush();
}
void launch_a(const lh_recorder &rec, const double *v, int n);
int main() {
    lh_recorder rec = {};
    launch_a(rec, nullptr, 0);
    k_b<<<1, 32, lh::BlockRecorder::smem_bytes(64)>>>(rec, nullptr, 0);
    return 0;
}
'''


def test_block_recorder_links_from_two_translation_units_with_rdc(tmp_path):
    (tmp_path / "a.cu").write_text(A_CU)
    (tmp_path / "b.cu").write_text(B_CU)
    exe = str(tmp_path / "two_tu")
    for extra, out in ((["-rdc=true"], exe), ([], exe + "_whole")):
        res = subprocess.run([NVCC] + ARCH + ["-std=c++17"] + extra + ["-I", INC, str(tmp_path / "a.cu"),
                              str(tmp_path / "b.cu"), "-o", out], capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr


def test_block_recorder_client_kernels_do_not_spill(tmp_path):
    res = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-shared", "-I", INC,
                          os.path.join(ROOT, "tests", "block_recorder_client.cu"), "-o", str(tmp_path / "client.so")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    log = res.stdout + res.stderr
    entries = re.findall(r"Compiling entry function '([^']+)'", log)
    assert len(entries) == 4, entries          # record, record_subset, record_ns, stop
    spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", log)]
    assert spills and not any(spills), log
    frames = [int(x) for x in re.findall(r"(\d+) bytes stack frame", log)]
    assert not any(frames), log


ASKED = [0, 1, 16, 31, 32, 33, 63, 64, 65, 100, 1000, 1024, 1025, 4095, 4096, 8191, 8192, 16383, 16384, 65535, 65536]

SIZES_CU = r'''
#include <stdio.h>
#include "loghisto_b200_device.cuh"
static_assert(lh::BlockRecorder::smem_bytes(4096) == 49152, "smem_bytes is a constant expression");
int main() {
    const unsigned asked[] = {%s};
    for (unsigned e : asked) printf("%%u %%u %%u\n", e, lh::BlockRecorder::table_entries(e), lh::BlockRecorder::smem_bytes(e));
    return 0;
}
'''


def test_smem_bytes_on_the_host(tmp_path):
    """12 B per slot, the entry count rounded down to a power of two, nothing below 32."""
    src = tmp_path / "sizes.cu"
    src.write_text(SIZES_CU % ", ".join(str(e) for e in ASKED))
    exe = str(tmp_path / "sizes")
    res = subprocess.run([NVCC] + ARCH + ["-std=c++17", "-I", INC, str(src), "-o", exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {int(a): (int(b), int(c)) for a, b, c in (line.split() for line in out if line)}
    assert sorted(got) == sorted(ASKED)
    for e in ASKED:
        slots = 0 if e < 32 else 1 << (e.bit_length() - 1)
        assert got[e] == (slots, 12 * slots), e
