"""CPU: the residual GEMM epilogue (EPI_RESID_F32: out_proj and fc2 of every encoder layer) reads the residual in batches
ahead of its stores.

`out` and `resid` may alias (the stack updates the residual stream in place), so the compiler may not move a residual load
above an earlier output store.  Written as one load per column group inside the store loop, the epilogue makes a dependent
global round trip per column group, 64 per tile and thread, while the tensor cores idle.  Nothing else catches that
regression: results stay the same and only time is lost.  This test disassembles the built library and counts how many
residual loads come before each output store."""
import os
import re
import shutil
import subprocess

import pytest

from one_peace_b200 import _lib

EPI_RESID_F32 = 2   # csrc/gemm.h
KERNEL = f"_ZN3opb16gemm_bf16_kernelILi{EPI_RESID_F32}EEEv14CUtensorMap_stS1_NS_12GemmEpilogueENS_8GemmGeomE"


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        exe = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return exe if os.path.exists(exe) else None


def load_runs(sass):
    """Lengths of the runs of 8-byte global loads (the float2 residual reads) that end at a global store."""
    runs, pending = [], 0
    for line in sass.splitlines():
        m = re.search(r"\b(LDG|STG)(\.[A-Z0-9_]+)*", line)
        if m is None:
            continue
        if m.group(1) == "LDG":
            pending += m.group(0).startswith("LDG.E.64")
        elif pending:
            runs.append(pending)
            pending = 0
    return runs


def test_load_runs_counts_loads_before_each_store():
    sass = "\n".join([
        "/*0010*/ @!P2 LDG.E.64 R180, desc[UR24][R180.64] ;",
        "/*0020*/ @!P2 STG.E desc[UR24][R180.64], R183 ;",
        "/*0030*/ STG.E.64 desc[UR24][R178.64], R172 ;",
        "/*0040*/ LDG.E.64 R4, desc[UR24][R4.64] ;",
        "/*0050*/ LDG.E.64 R6, desc[UR24][R6.64] ;",
        "/*0060*/ LDG.E R8, desc[UR24][R8.64] ;",
        "/*0070*/ FADD R9, R4, R6 ;",
        "/*0080*/ STG.E.64 desc[UR24][R2.64], R4 ;",
    ])
    assert load_runs(sass) == [1, 2]


def test_residual_epilogue_loads_ahead_of_stores():
    exe = cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    lib = _lib.LIB_PATH
    assert os.path.exists(lib), f"{lib} not built; {_lib.build_hint()}"
    # the library holds one cubin per source file; cuobjdump warns about each one without the kernel
    sass = subprocess.run([exe, "-sass", "-fun", KERNEL, lib], capture_output=True, text=True, check=True).stdout
    assert KERNEL in sass, "gemm_bf16_kernel<EPI_RESID_F32> not found in the library"
    runs = load_runs(sass)
    # each epilogue copy reads 2 fragment rows x 32 column groups; loaded one group per store pair that is 64 runs of 1
    assert sum(runs) >= 64, runs
    assert sum(runs) >= 8 * len(runs), f"residual loads are not batched ahead of the stores: runs {runs}"
