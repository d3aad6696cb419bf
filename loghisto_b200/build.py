"""Builds libloghisto_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache, no torch extension)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libloghisto_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O2",
    "--fmad=true",           # FP32 fast path may contract; the exact path uses __d*_rn intrinsics only
    "-Xptxas", "-v",
    "-shared",
]


HOST_LIB = os.path.join(HERE, "libloghisto_host.so")
HOST_SRC = os.path.join(HERE, "host", "metric_system.cc")
HOST_SRCS = [HOST_SRC, os.path.join(HERE, "host", "print_benchmark.cc")]


def needs_build_host() -> bool:
    if not os.path.exists(HOST_LIB):
        return True
    deps = HOST_SRCS + [os.path.join(HERE, "host", "metric_system.h"), os.path.join(ROOT, "include", "loghisto_b200.h"), LIB]
    return _newest([d for d in deps if os.path.exists(d)]) > os.path.getmtime(HOST_LIB)


def build_host(force: bool = False) -> str:
    """C++ mirror of MetricSystem (host glue above the C ABI); links against libloghisto_b200.so."""
    build()
    if not force and not needs_build_host():
        return HOST_LIB
    gxx = shutil.which("g++") or "g++"
    cmd = [gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall", "-Wextra",
           "-I", os.path.join(ROOT, "include"), "-o", HOST_LIB] + HOST_SRCS + [
           "-L", HERE, "-lloghisto_b200", "-Wl,-rpath,$ORIGIN", "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("g++ failed building libloghisto_host.so")
    return HOST_LIB


def sources():
    return [os.path.join(CSRC, "lh_api.cu")]


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "loghisto_b200.h"), DEVICE_HEADER]
    return _newest(deps) > os.path.getmtime(LIB)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libloghisto_b200.so (there is no CPU fallback)")
    cmd = [nvcc] + NVCC_FLAGS + ["-I", os.path.join(ROOT, "include"), "-o", LIB] + sources()
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed building libloghisto_b200.so")
    if verbose:
        print(log)
    return LIB


CLIENT_SRC = os.path.join(ROOT, "tests", "device_record_client.cu")
CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_record_client.so")
DEVICE_HEADER = os.path.join(ROOT, "include", "loghisto_b200_device.cuh")


NAMED_CLIENT_SRC = os.path.join(ROOT, "tests", "named_record_client.cu")
NAMED_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libnamed_record_client.so")

BLOCK_CLIENT_SRC = os.path.join(ROOT, "tests", "block_recorder_client.cu")
BLOCK_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libblock_recorder_client.so")

TIMER_CLIENT_SRC = os.path.join(ROOT, "tests", "gpu_timer_client.cu")
TIMER_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libgpu_timer_client.so")

GRAPH_CLIENT_SRC = os.path.join(ROOT, "tests", "graph_record_client.cu")
GRAPH_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libgraph_record_client.so")

BOARD_CLIENT_SRC = os.path.join(ROOT, "tests", "board_read_client.cu")
BOARD_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libboard_read_client.so")

GAUGE_CLIENT_SRC = os.path.join(ROOT, "tests", "gauge_write_client.cu")
GAUGE_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libgauge_write_client.so")

RAW_CLIENT_SRC = os.path.join(ROOT, "tests", "raw_read_client.cu")
RAW_CLIENT_LIB = os.path.join(ROOT, "tests", "_build", "libraw_read_client.so")

# One client of the device API built the ways callers build it (tests/device_matrix_client.cu; tests/
# test_gpu_device_api_builds.py runs every variant against the oracle).  Each variant adds -std=c++17 -Xcompiler -fPIC
# -shared -I include; "rdc" compiles the client as two translation units (-DLHM_PART=1 / 2) and device-links them.
MATRIX_SRC = os.path.join(ROOT, "tests", "device_matrix_client.cu")
MATRIX_DIR = os.path.join(ROOT, "tests", "_build", "device_matrix")
MATRIX_LIB_NAME = "libdevice_matrix_client.so"
_SM90A = ["-gencode", "arch=compute_90a,code=sm_90a"]
_MATRIX_REF = _SM90A + ["-O3", "--fmad=true"]          # the library's device flags
DEVICE_MATRIX = {
    "ref": _MATRIX_REF,
    "fastmath": _MATRIX_REF + ["--use_fast_math"],
    "debug": _SM90A + ["-G"],
    "maxrreg": _MATRIX_REF + ["-maxrregcount=32"],
    "rdc": _MATRIX_REF + ["-rdc=true"],
    "ptx90": ["-gencode", "arch=compute_90,code=compute_90"],
    "ptx70": ["-gencode", "arch=compute_70,code=compute_70", "-Wno-deprecated-gpu-targets"],
}


def matrix_lib(variant: str) -> str:
    return os.path.join(MATRIX_DIR, variant, MATRIX_LIB_NAME)


def _matrix_commands(nvcc: str, variant: str) -> list:
    """The nvcc commands that build one variant, in order."""
    flags = DEVICE_MATRIX[variant] + ["-std=c++17", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include")]
    out = matrix_lib(variant)
    if variant != "rdc":
        return [[nvcc] + flags + ["-shared", "-o", out, MATRIX_SRC]]
    objs = [os.path.join(MATRIX_DIR, variant, "part%d.o" % k) for k in (1, 2)]
    return ([[nvcc] + flags + ["-DLHM_PART=%d" % k, "-c", "-o", o, MATRIX_SRC] for k, o in zip((1, 2), objs)]
            + [[nvcc] + flags + ["-shared", "-o", out] + objs])


def _build_matrix_variant(nvcc: str, variant: str, force: bool):
    """Builds one variant unless its library is newer than the sources and was built by the same commands (kept beside
    it in commands.txt).  Returns None, or the failing command and its output."""
    lib = matrix_lib(variant)
    stamp = os.path.join(os.path.dirname(lib), "commands.txt")
    cmds = _matrix_commands(nvcc, variant)
    text = "\n".join(" ".join(c) for c in cmds) + "\n"
    deps = [MATRIX_SRC, DEVICE_HEADER, os.path.join(ROOT, "include", "loghisto_b200.h")]
    if not force and os.path.exists(lib) and os.path.exists(stamp) and _newest(deps) <= os.path.getmtime(lib):
        with open(stamp) as f:
            if f.read() == text:
                return None
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    if os.path.exists(stamp):
        os.remove(stamp)
    for c in cmds:
        res = subprocess.run(c, capture_output=True, text=True)
        if res.returncode != 0:
            return " ".join(c) + "\n" + res.stdout + res.stderr
    with open(stamp, "w") as f:
        f.write(text)
    return None


def build_device_matrix(force: bool = False) -> dict:
    """Every variant of DEVICE_MATRIX, built side by side; returns {variant: library path}."""
    from concurrent.futures import ThreadPoolExecutor
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build the device-API build matrix")
    with ThreadPoolExecutor(max_workers=len(DEVICE_MATRIX)) as pool:
        errors = list(pool.map(lambda v: _build_matrix_variant(nvcc, v, force), DEVICE_MATRIX))
    for e in errors:
        if e:
            sys.stderr.write(e)
            raise RuntimeError("nvcc failed building the device-API build matrix")
    return {v: matrix_lib(v) for v in DEVICE_MATRIX}


def build_device_client(force: bool = False) -> str:
    """CUDA clients of the device API (tests/device_record_client.cu, tests/named_record_client.cu,
    tests/block_recorder_client.cu, tests/gpu_timer_client.cu, tests/graph_record_client.cu,
    tests/board_read_client.cu, tests/gauge_write_client.cu, tests/raw_read_client.cu): separate shared libraries that
    record into a context from their own kernels, give the GPU timers spans to measure, read device subscriptions,
    write device gauges, or query raw device subscriptions, knowing the library only through the public headers.
    Then the device-API build matrix (build_device_matrix).  Returns the path of the first."""
    for src, lib in ((CLIENT_SRC, CLIENT_LIB), (NAMED_CLIENT_SRC, NAMED_CLIENT_LIB), (BLOCK_CLIENT_SRC, BLOCK_CLIENT_LIB),
                     (TIMER_CLIENT_SRC, TIMER_CLIENT_LIB), (GRAPH_CLIENT_SRC, GRAPH_CLIENT_LIB),
                     (BOARD_CLIENT_SRC, BOARD_CLIENT_LIB), (GAUGE_CLIENT_SRC, GAUGE_CLIENT_LIB),
                     (RAW_CLIENT_SRC, RAW_CLIENT_LIB)):
        deps = [src, DEVICE_HEADER, os.path.join(ROOT, "include", "loghisto_b200.h")]
        if not force and os.path.exists(lib) and _newest(deps) <= os.path.getmtime(lib):
            continue
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        if not os.path.exists(nvcc):
            raise RuntimeError("nvcc not found: cannot build the device-record clients")
        os.makedirs(os.path.dirname(lib), exist_ok=True)
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
               "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-o", lib, src]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError("nvcc failed building " + lib)
    build_device_matrix(force)
    return CLIENT_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_host(force="--force" in sys.argv))
    print(build_device_client(force="--force" in sys.argv))
