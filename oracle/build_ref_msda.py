"""TEST INFRASTRUCTURE.  Builds the reference's own multi-scale deformable attention extension
(one_peace_vision/seg/ops/src, ``MultiScaleDeformableAttention``) for sm_90a into oracle/_ref/, so the GPU tests and
scripts/bench_msda.py can compare against the reference's compiled op.  It needs the reference source tree; __graft_entry__
.build() calls it where that tree exists and otherwise leaves oracle/_ref/ as it is.

    python oracle/build_ref_msda.py

The sources are copied to a temporary directory and built there with torch.utils.cpp_extension, TORCH_CUDA_ARCH_LIST=9.0a
and the nvcc defines of the reference's setup.py.  One fix is made in the copy: the two AT_DISPATCH_FLOATING_TYPES calls
take ``value.type()``, which current torch no longer accepts, and get ``value.scalar_type()``.  Only the built
MultiScaleDeformableAttention*.so is kept.
"""
import glob
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_stub  # noqa: E402

OPS = os.path.join(ref_stub.REF_ROOT, "one_peace_vision", "seg", "ops")
OUT = os.path.join(HERE, "_ref")
NAME = "MultiScaleDeformableAttention"


def built_path():
    """The built extension under oracle/_ref/, or None."""
    hits = sorted(glob.glob(os.path.join(OUT, NAME + "*.so")))
    return hits[0] if hits else None


def reference_available():
    return os.path.isdir(os.path.join(OPS, "src"))


def build(force=False):
    if built_path() and not force:
        return built_path()
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    from torch.utils import cpp_extension
    with open(os.path.join(OPS, "setup.py")) as f:
        defines = re.findall(r"'(-D[A-Za-z0-9_]+(?:=[^']*)?)'", f.read())
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "src")
        shutil.copytree(os.path.join(OPS, "src"), src)
        cu = os.path.join(src, "cuda", "ms_deform_attn_cuda.cu")
        with open(cu) as f:
            text = f.read()
        fixed, n = re.subn(r"AT_DISPATCH_FLOATING_TYPES\(value\.type\(\)", "AT_DISPATCH_FLOATING_TYPES(value.scalar_type()",
                           text)
        if n != 2:
            raise RuntimeError(f"expected 2 dispatch calls to fix in {cu}, found {n}")
        with open(cu, "w") as f:
            f.write(fixed)
        sources = glob.glob(os.path.join(src, "*.cpp")) + glob.glob(os.path.join(src, "cpu", "*.cpp")) + \
            glob.glob(os.path.join(src, "cuda", "*.cu"))
        bdir = os.path.join(tmp, "build")
        os.makedirs(bdir)
        cpp_extension.load(name=NAME, sources=sources, extra_include_paths=[src], extra_cflags=["-DWITH_CUDA"],
                           extra_cuda_cflags=["-DWITH_CUDA"] + defines, build_directory=bdir, with_cuda=True,
                           is_python_module=False, verbose=False)
        so = glob.glob(os.path.join(bdir, NAME + "*.so"))
        if len(so) != 1:
            raise RuntimeError(f"no {NAME} library in {bdir}")
        os.makedirs(OUT, exist_ok=True)
        dst = os.path.join(OUT, os.path.basename(so[0]))
        shutil.copy2(so[0], dst)
    return dst


if __name__ == "__main__":
    if not reference_available():
        sys.exit(f"reference sources not found under {OPS}")
    print(build(force="--force" in sys.argv))
