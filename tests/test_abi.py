"""The C-ABI shared library: builds for sm_90a, loads, exports exactly what include/dplonk.h
declares, and fails loudly (no CPU fallback) without a GPU.  No compute calls here."""
import ctypes
import os
import re
import shutil

import pytest

import distributed_plonk_b200 as dp
from distributed_plonk_b200 import _binding, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "dplonk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dp_[a-z0-9_]+)\s*\(", src)))


def test_binding_covers_header():
    assert header_functions() == sorted(_binding.EXPORTS)


@pytest.fixture(scope="module")
def real_lib():
    if build.is_stale():
        if not shutil.which("nvcc") and not os.path.exists("/usr/local/cuda/bin/nvcc"):
            pytest.skip("no nvcc and no prebuilt library")
        build.build()
    return dp.load()


def test_library_exports_every_declared_symbol(real_lib):
    raw = ctypes.CDLL(dp.library_path())
    for name in header_functions():
        assert hasattr(raw, name), f"{name} declared in dplonk.h but not exported"
    assert b"sm_90a" in real_lib.dp_version()


def test_sass_is_sm90a_and_uses_tma(real_lib):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    import subprocess
    out = subprocess.run([cuobjdump, "-sass", "-fun", "_ZN2dp15ntt_tile_kernelILi3EEEvNS_7NttPassE", dp.library_path()],
                         capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "UBLKCP" in out            # cp.async.bulk (TMA) staging of the twiddle tile
    assert "LDGSTS" in out            # cp.async: the tile is copied global -> shared without passing through registers
    assert "IMAD.WIDE.U32" in out     # fused 32x32->64 multiply-accumulate chains


def test_fails_loudly_without_gpu(real_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(dp.DpError) as e:
        dp.Context(real_lib, 0, 0, 1)
    assert e.value.code == _binding.DP_E_CUDA


def test_header_is_plain_c_and_struct_layouts_match_the_binding(tmp_path):
    """include/dplonk.h compiles as C11 (-Wall -Werror -pedantic: the boundary a cgo / Rust `extern "C"`
    binding sees), and the structs mirrored in _binding.py have the same size and field offsets"""
    import subprocess
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    src = tmp_path / "abi.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "dplonk.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(dp_quotient_args), offsetof(dp_quotient_args, sigmas),\n'
        "         offsetof(dp_quotient_args, wires), offsetof(dp_quotient_args, perm), offsetof(dp_quotient_args, k),\n"
        "         offsetof(dp_quotient_args, gamma), sizeof(dp_fft_workload), offsetof(dp_fft_workload, col_end));\n"
        "  int (*f)(dp_ctx *, uint64_t, uint64_t, uint64_t, const void *, size_t) = dp_msm_submit; (void)f;\n"
        "  return 0;\n}\n")
    exe = tmp_path / "abi"
    lib = dp.library_path()
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{os.path.join(ROOT, 'include')}", str(src), "-o", str(exe),
                           f"-L{os.path.dirname(lib)}", f"-l:{os.path.basename(lib)}", f"-Wl,-rpath,{os.path.dirname(lib)}",
                           "-Wl,--unresolved-symbols=ignore-in-shared-libs"])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    Q, W = _binding.QuotientArgs, _binding.FftWorkload
    assert got == [ctypes.sizeof(Q), Q.sigmas.offset, Q.wires.offset, Q.perm.offset, Q.k.offset, Q.gamma.offset,
                   ctypes.sizeof(W), W.col_end.offset]
