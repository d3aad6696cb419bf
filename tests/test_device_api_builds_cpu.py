"""The device API header as callers compile it, and the device-API build matrix as built (no GPU needed).

include/loghisto_b200_device.cuh is compiled by other people's nvcc commands.  It promises to build without warnings
from any translation unit, with or without -rdc=true, for sm_70 and later.  The first test compiles a translation unit
that uses every device function under C++14, 17 and 20 for compute_70 PTX, sm_80, sm_90 and sm_90a with every warning
an error, and device-links two such units with -rdc=true.

build_device_client() builds tests/device_matrix_client.cu under each flag set of build.DEVICE_MATRIX, and
tests/test_gpu_device_api_builds.py runs each against the oracle.  A flag that silently did nothing would leave that
comparison proving nothing, so the other tests read the built libraries with cuobjdump and check that each variant is
what its name says."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from loghisto_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
WERROR = ["--Werror", "all-warnings", "-Xcompiler", "-Wall,-Wextra,-Werror"]

needs_nvcc = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not installed")
needs_cuobjdump = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")

# Every function of the device API, from one kernel.  `name` keeps the kernels of two units apart.
USER_TU = r"""
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "loghisto_b200.h"
#include "loghisto_b200_device.cuh"

__global__ void every_call_%(name)s(lh_recorder rec, lh_board b, lh_raw_board raw, const double *v, long long *out,
                                    double *g64, float *g32, __half *g16, __nv_bfloat16 *gb16, int64_t *gi64,
                                    int32_t *gi32, uint64_t *gu64) {
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t id = threadIdx.x;
    lh::record(rec, id, v[id]);
    lh::record_ns(rec, id, out[id]);
    lh::count(rec, id, 3);
    const lh::TimerToken t = lh::start_timer(id);
    out[id] = lh::stop(rec, t);
    lh::BlockHistogram bh(rec, smem);
    bh.init(id);
    bh.add(v[id]);
    bh.flush();
    lh::BlockRecorder br(rec, smem, 64);
    br.init();
    br.record(id, v[id]);
    br.record_ns(id, out[id]);
    out[id] += br.stop(lh::start_timer(id));
    br.flush();
    lh::HistogramStats hs;
    lh::CounterStats cs;
    int32_t key;
    double val;
    uint64_t rank, total, cnt;
    out[id] += (long long)(lh::read_histogram(b, id, &hs) + lh::read_counter(b, id, &cs));
    out[id] += (long long)lh::raw_percentile(raw, id, 0.5, &key, &val);
    out[id] += (long long)lh::raw_rank(raw, id, v[id], &rank, &total);
    out[id] += (long long)lh::raw_bucket_count(raw, id, key, &cnt);
    lh::set_gauge(g64, val);
    lh::set_gauge(g32, (float)val);
    lh::set_gauge(g16, __float2half((float)val));
    lh::set_gauge(gb16, __float2bfloat16((float)val));
    lh::set_gauge(gi64, (int64_t)rank);
    lh::set_gauge(gi32, (int32_t)key);
    lh::set_gauge(gu64, cnt);
}
"""

TARGETS = {
    "compute_70": ["-gencode", "arch=compute_70,code=compute_70", "-Wno-deprecated-gpu-targets"],
    "sm_80": ["-gencode", "arch=compute_80,code=sm_80"],
    "sm_90": ["-gencode", "arch=compute_90,code=sm_90"],
    "sm_90a": ["-gencode", "arch=compute_90a,code=sm_90a"],
}
STDS = ("c++14", "c++17", "c++20")


def run(cmd):
    res = subprocess.run(cmd, capture_output=True, text=True)
    return res.returncode, res.stdout + res.stderr


@needs_nvcc
def test_header_compiles_warning_free_for_every_standard_and_target(tmp_path):
    """C++14, 17 and 20 x {compute_70 PTX, sm_80, sm_90, sm_90a}, every warning an error, then two units of the same
    kind built with -rdc=true and device-linked into one shared library."""
    src = tmp_path / "user.cu"
    src.write_text(USER_TU % {"name": "a"})
    jobs = {(std, tgt): [NVCC] + flags + WERROR + ["-std=" + std, "-Xcompiler", "-fPIC", "-I", INCLUDE, "-c", "-o",
                                                   str(tmp_path / ("%s_%s.o" % (std, tgt))), str(src)]
            for std in STDS for tgt, flags in TARGETS.items()}
    src_b = tmp_path / "user_b.cu"
    src_b.write_text(USER_TU % {"name": "b"})
    rdc = ["-gencode", "arch=compute_90a,code=sm_90a", "-rdc=true", "-std=c++17", "-Xcompiler", "-fPIC"] + WERROR
    objs = [str(tmp_path / "rdc_a.o"), str(tmp_path / "rdc_b.o")]
    jobs[("rdc", "a")] = [NVCC] + rdc + ["-I", INCLUDE, "-c", "-o", objs[0], str(src)]
    jobs[("rdc", "b")] = [NVCC] + rdc + ["-I", INCLUDE, "-c", "-o", objs[1], str(src_b)]
    with ThreadPoolExecutor(max_workers=8) as pool:
        results = dict(zip(jobs, pool.map(run, jobs.values())))
    for what, (rc, log) in results.items():
        assert rc == 0 and not log.strip(), (what, log)
    lib = str(tmp_path / "librdc.so")
    rc, log = run([NVCC] + rdc + ["-shared", "-o", lib] + objs)
    assert rc == 0 and not log.strip(), log
    rc, sass = run([CUOBJDUMP, "-sass", lib])
    assert rc == 0, sass
    names = functions(sass)
    assert any("every_call_a" in f for f in names) and any("every_call_b" in f for f in names), names
    assert sum(f == "_ZN2lh11exact_key16Edd" for f in names) == 1, names


def functions(sass: str) -> list:
    return re.findall(r"Function : (\S+)", sass)


def sass_by_function(sass: str) -> dict:
    """{function name: its SASS text} of cuobjdump -sass output."""
    out, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            out[name].append(line)
    return {k: "\n".join(v) for k, v in out.items()}


@pytest.fixture(scope="module")
def matrix():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not installed")
    return build.build_device_matrix()


def dump(lib, *flags):
    rc, out = run([CUOBJDUMP] + list(flags) + [lib])
    return out


def list_files(lib):
    """(ELF names, PTX names) embedded in a library."""
    out = dump(lib, "-lelf", "-lptx")
    return re.findall(r"ELF file\s+\d+: (\S+)", out), re.findall(r"PTX file\s+\d+: (\S+)", out)


@needs_cuobjdump
def test_matrix_variants_hold_the_code_their_names_say(matrix):
    """ref, fastmath, debug, maxrreg and rdc carry sm_90a SASS and no PTX; ptx90 and ptx70 carry PTX for their virtual
    architecture and no SASS, so the driver JITs them at load."""
    assert sorted(matrix) == sorted(build.DEVICE_MATRIX)
    for v in ("ref", "fastmath", "debug", "maxrreg", "rdc"):
        elf, ptx = list_files(matrix[v])
        assert elf and all(e.endswith(".sm_90a.cubin") for e in elf) and not ptx, (v, elf, ptx)
    for v, arch in (("ptx90", "sm_90"), ("ptx70", "sm_70")):
        elf, ptx = list_files(matrix[v])
        assert not elf and ptx == ["libdevice_matrix_client.1.%s.ptx" % arch], (v, elf, ptx)
        text = dump(matrix[v], "-ptx")
        assert re.search(r"^\.target %s\s*$" % arch, text, re.M), v
        assert "k_estimate" in text and "k_block_recorder" in text, v


FTZ_OPS = re.compile(r"\b(FADD|FMUL|FFMA|FSETP)\S*\.FTZ\b")


@needs_cuobjdump
def test_fastmath_flushes_the_estimate_and_ref_does_not(matrix):
    """--use_fast_math turns the FP32 ops of lh::fast_candidate into their flush-to-zero forms; the library's flags do
    not.  (The estimate is certified under the library's flags; the GPU test checks that the ftz forms give the same
    outputs for every cell.)"""
    for v, want in (("fastmath", True), ("ref", False)):
        fns = sass_by_function(dump(matrix[v], "-sass"))
        est = [t for f, t in fns.items() if "k_estimateEN2lh4Prec" in f]
        assert len(est) == 1, (v, list(fns))
        ops = FTZ_OPS.findall(est[0])
        if want:
            assert {"FADD", "FFMA", "FMUL", "FSETP"} <= set(ops), (v, ops)
        else:
            assert not ops, (v, ops)


@needs_cuobjdump
def test_debug_carries_device_debug_info(matrix, tmp_path):
    """-G: the cubin has DWARF sections; ref has none."""
    for v, want in (("debug", True), ("ref", False)):
        d = tmp_path / v
        d.mkdir()
        res = subprocess.run([CUOBJDUMP, "-xelf", "all", matrix[v]], cwd=d, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        cubins = [p.read_bytes() for p in d.iterdir() if p.suffix == ".cubin"]
        assert cubins, v
        assert any(b".debug_info\0" in c for c in cubins) == want, v


@needs_cuobjdump
def test_maxrreg_kernels_use_at_most_32_registers(matrix):
    """-maxrregcount=32 reached every kernel (ref has kernels above 32, so the flag changed code)."""
    for v, cap_ok in (("maxrreg", True), ("ref", False)):
        regs = [int(r) for r in re.findall(r"REG:(\d+)", dump(matrix[v], "-res-usage"))]
        assert len(regs) >= 13, (v, regs)
        assert (max(regs) <= 32) == cap_ok, (v, regs)


@needs_cuobjdump
def test_rdc_links_both_units_with_one_exact_key16(matrix):
    """The -rdc=true variant holds the kernels of both translation units (k_record_part2 from the second, the rest
    from the first) and one out-of-line lh::exact_key16, which both reach through lh::key16_of."""
    names = functions(dump(matrix["rdc"], "-sass"))
    units = {re.search(r"device_matrix_client_cu_([0-9a-f]+)__", f).group(1) for f in names if "__nv_static_" in f}
    assert len(units) == 2, names
    assert any("k_record_part2" in f for f in names) and any("k_estimateEN2lh4Prec" in f for f in names), names
    assert sum(f == "_ZN2lh11exact_key16Edd" for f in names) == 1, names
    assert "-rdc=true" in open(os.path.join(os.path.dirname(matrix["rdc"]), "commands.txt")).read()
