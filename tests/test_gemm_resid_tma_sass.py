"""CPU: the residual GEMM epilogue on plain aligned operands (gemm_bf16_resid_tma_kernel: out_proj and fc2 of every encoder
layer) moves its residual, fp32 output and bf16 copy only with TMA.

Loaded and stored from registers, a 128 x 256 residual tile is 128 KB read and 192 KB written with 8-byte accesses, and
the tensor cores wait for all of them.  Results stay the same and only time is lost, so this test disassembles the built
library: the ring kernel must load with UTMALDG and store with UTMASTG, with no 8-byte global loads beyond the epilogue-operand
stager's and no global store other than the 8-byte statistics records."""
import re

from test_gemm_tma_store_sass import EPI_GEGLU_BF16, EPI_RESID_F32, TMA_OUT, sass_of

RING = ("_ZN3opb26gemm_bf16_resid_tma_kernelILi{}EEEv14CUtensorMap_stS1_S1_S1_S1_NS_12GemmEpilogueENS_8GemmGeomE"
        .format(EPI_RESID_F32))


def global_accesses(sass, op):
    """the LDG or STG instructions of `sass`, with their modifiers"""
    return [m.group(0) for m in re.finditer(rf"\b{op}(\.[A-Z0-9_]+)*", sass)]


def test_global_accesses_lists_modifiers():
    sass = "\n".join([
        "/*0010*/ @!P2 LDG.E.64 R180, desc[UR24][R180.64] ;",
        "/*0020*/ @!P0 STG.E.64 desc[UR18][R2.64], R4 ;",
        "/*0030*/ LDG.E R8, desc[UR24][R8.64] ;",
        "/*0040*/ UTMASTG.2D [UR8], [UR6] ;",
    ])
    assert global_accesses(sass, "LDG") == ["LDG.E.64", "LDG.E"]
    assert global_accesses(sass, "STG") == ["STG.E.64"]


def test_ring_kernel_moves_the_residual_tile_with_tma():
    sass = sass_of(RING)
    assert "UTMALDG" in sass and "UTMASTG" in sass
    # The only 8-byte global loads left are the stager warps' reads of the LayerNorm records, the same ones the GeGLU
    # staged-output kernel makes (its epilogue reads nothing else from global memory).  The direct-store kernel has about
    # 130 more: the residual fragments.
    wide = [op for op in global_accesses(sass, "LDG") if re.search(r"\.(64|128)\b", op)]
    geglu = [op for op in global_accesses(sass_of(TMA_OUT.format(EPI_GEGLU_BF16)), "LDG") if re.search(r"\.(64|128)\b", op)]
    assert len(wide) <= len(geglu), f"{len(wide)} 8-byte global loads against {len(geglu)}: residual read from global memory"
    # the only global stores left are the (sum, sum of squares) records of the two fragment rows
    stores = global_accesses(sass, "STG")
    assert stores and all(op == "STG.E.64" for op in stores), stores
    assert len(stores) <= 4, f"{len(stores)} global stores: results stored from registers"
