"""CPU-side checks of the drop-in boundary: the library builds, loads, exports every symbol the header
declares, and refuses to run without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "loghisto_b200.h")).read()
    return sorted(set(re.findall(r"^LH_API [^;(]*?\b(lh_[a-z0-9_]+)\(", src, flags=re.M)))


def test_library_builds_and_exports_every_declared_symbol():
    from loghisto_b200 import _lib, build
    build.build()
    lib = ctypes.CDLL(build.LIB)
    syms = header_symbols()
    assert len(syms) >= 40
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/loghisto_b200.h but not exported"
    # the ctypes binding covers exactly the declared surface
    assert sorted(_lib.SIGNATURES) == syms


def test_abi_version_and_strerror():
    from loghisto_b200 import _lib
    lib = _lib.load()
    assert lib.lh_abi_version() == 2
    assert lib.lh_strerror(0) == b"ok"
    assert b"no CPU fallback" in lib.lh_strerror(_lib.LH_ERR_NO_DEVICE)
    assert lib.lh_k1_variant_count() >= 4


def test_struct_layouts_match_header(tmp_path):
    """sizeof / offsetof of every struct of the header, as a C compiler sees them, against the ctypes mirror."""
    import subprocess
    from loghisto_b200 import _lib
    structs = {"lh_config": _lib.lh_config, "lh_staging": _lib.lh_staging, "lh_device_view": _lib.lh_device_view,
               "lh_sparse": _lib.lh_sparse, "lh_stats": _lib.lh_stats, "lh_comm_stats": _lib.lh_comm_stats,
               "lh_certify_form": _lib.lh_certify_form}
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "loghisto_b200.h"', 'int main(void) {']
    for name, cls in structs.items():
        src.append('printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        for f, _ in cls._fields_:
            src.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, f, name, f))
    src.append('printf("lh_peer_handle %zu\\n", sizeof(lh_peer_handle)); return 0; }')
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(c)], check=True)
    want = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for name, cls in structs.items():
        assert ctypes.sizeof(cls) == int(want[name]), name
        for f, _ in cls._fields_:
            assert getattr(cls, f).offset == int(want["%s.%s" % (name, f)]), (name, f)
    assert int(want["lh_peer_handle"]) == _lib.LH_PEER_HANDLE_BYTES


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import loghisto_b200 as lh
    with pytest.raises(lh.LhError) as e:
        lh.Engine()
    assert e.value.status == -4


def test_create_rejects_bad_config():
    from loghisto_b200 import _lib
    lib = _lib.load()
    h = ctypes.c_void_p()
    cfg = _lib.lh_config(ctypes.sizeof(_lib.lh_config), 0, 0, 1, 0, 0, 0)
    assert lib.lh_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.LH_ERR_INVALID
    cfg = _lib.lh_config(8, 0, 1, 1, 0, 0, 0)
    assert lib.lh_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.LH_ERR_INVALID
    assert lib.lh_destroy(None) == 0


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "loghisto_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"liblh_oracle|from oracle|import oracle|oracle[./]", text), \
                    f"{f} reaches into oracle/"


def test_plain_c_client(tmp_path):
    """The header compiles as C11 and the library links from a C program (no C++ runtime needed by the caller)."""
    import subprocess
    from loghisto_b200 import build
    build.build()
    exe = str(tmp_path / "c_abi_client")
    libdir = os.path.dirname(build.LIB)
    cmd = ["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_client.c"), "-o", exe, "-L", libdir, "-lloghisto_b200", "-Wl,-rpath," + libdir]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    run = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stdout + run.stderr
