"""CPU: the bf16 GEMM epilogues on a plain row-major output (QKV, GeGLU and the bf16 weight gradients) stage their tile in
shared memory and write it with TMA bulk stores (gemm_bf16_tma_out_kernel), and the direct-store kernel keeps its symbol.

Written as per-thread global stores, a 128 x 256 bf16 tile takes 64 32-bit stores per thread, each warp instruction touching
8 rows, and the tensor cores wait for all of them.  Results stay the same and only time is lost, so this test disassembles
the built library: the staged kernels must store their output with UTMASTG and no 16- or 32-bit STG."""
import os
import re
import shutil
import subprocess

import pytest

from one_peace_b200 import _lib

EPI_STORE_BF16, EPI_GEGLU_BF16, EPI_RESID_F32, EPI_GELU_BF16 = 0, 1, 2, 4   # csrc/gemm.h
TMA_OUT = "_ZN3opb24gemm_bf16_tma_out_kernelILi{}EEEv14CUtensorMap_stS1_S1_NS_12GemmEpilogueENS_8GemmGeomE"
DIRECT = "_ZN3opb16gemm_bf16_kernelILi{}EEEv14CUtensorMap_stS1_NS_12GemmEpilogueENS_8GemmGeomE"


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        exe = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return exe if os.path.exists(exe) else None


def sass_of(kernel):
    exe = cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    lib = _lib.LIB_PATH
    assert os.path.exists(lib), f"{lib} not built; {_lib.build_hint()}"
    # the library holds one cubin per source file; cuobjdump warns about each one without the kernel
    sass = subprocess.run([exe, "-sass", "-fun", kernel, lib], capture_output=True, text=True, check=True).stdout
    assert kernel in sass, f"{kernel} not found in the library"
    return sass


def narrow_global_stores(sass):
    """global stores of 16 or 32 bits (a bf16 element or pair); STG.E.64 / .128 are wider"""
    return [m.group(0) for m in re.finditer(r"\bSTG(\.[A-Z0-9_]+)*", sass)
            if not re.search(r"\.(64|128)\b", m.group(0))]


def test_narrow_global_stores_classifies_widths():
    sass = "\n".join([
        "/*0010*/ @!P2 STG.E desc[UR24][R180.64], R183 ;",
        "/*0020*/ STG.E.U16 desc[UR24][R2.64], R4 ;",
        "/*0030*/ STG.E.64 desc[UR24][R178.64], R172 ;",
        "/*0040*/ STG.E.128 desc[UR24][R2.64], R4 ;",
        "/*0050*/ UTMASTG.2D [UR8], [UR6] ;",
    ])
    assert narrow_global_stores(sass) == ["STG.E", "STG.E.U16"]


@pytest.mark.parametrize("epi", [EPI_STORE_BF16, EPI_GELU_BF16, EPI_GEGLU_BF16])
def test_staged_bf16_epilogues_store_with_tma(epi):
    sass = sass_of(TMA_OUT.format(epi))
    assert "UTMASTG" in sass, "no TMA store in the staged-output kernel"
    assert "STSM" in sass, "the tile is not written to shared memory with stmatrix"
    # GeGLU still writes its (sum, sum of squares) records as float2
    assert narrow_global_stores(sass) == [], "the staged-output kernel stores bf16 values to global memory itself"


def test_direct_store_kernel_keeps_its_symbol():
    sass = sass_of(DIRECT.format(EPI_RESID_F32))
    assert "UTMASTG" not in sass
