"""Compiles the reference's Gaussian rasterizer (Inria's `diff-gaussian-rasterization`, as vendored by the
reference under third_party/PhysGaussian/gaussian-splatting/submodules/) for sm_90a into oracle/_ref/, where the
GPU tests load it by file as the device rasterizer's oracle.

The reference checkout is $PIXIE_REFERENCE, or a `reference` directory beside this repository. When neither
holds the rasterizer's sources, nothing is done and an artefact already in oracle/_ref/ is kept: the sources are
not part of this repository, only the binary built from them travels with the tree.

The sources build unchanged except for `-include cstdint`: rasterizer_impl.h uses std::uintptr_t without that
header, which current host compilers reject.
"""
from __future__ import annotations

import glob
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
NAME = "diff_gaussian_rasterization_ref"
OUT = os.path.join(HERE, "_ref", "gs_rasterizer")
SUBDIR = os.path.join("third_party", "PhysGaussian", "gaussian-splatting", "submodules", "diff-gaussian-rasterization")


def artefact() -> str | None:
    """Path of the built extension module, or None when it has not been built."""
    hits = sorted(glob.glob(os.path.join(OUT, NAME + "*.so")))
    return hits[0] if hits else None


def source_dir() -> str | None:
    ref = os.environ.get("PIXIE_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")
    src = os.path.join(ref, SUBDIR)
    return src if os.path.isfile(os.path.join(src, "rasterize_points.cu")) else None


def build() -> str | None:
    src = source_dir()
    if src is None:
        return artefact()
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    from torch.utils import cpp_extension
    os.makedirs(OUT, exist_ok=True)
    sources = [os.path.join(src, p) for p in ("cuda_rasterizer/rasterizer_impl.cu", "cuda_rasterizer/forward.cu",
                                              "cuda_rasterizer/backward.cu", "rasterize_points.cu", "ext.cpp")]
    glm = os.path.join(src, "third_party", "glm")
    cpp_extension.load(NAME, sources, extra_cflags=["-O3", "-include", "cstdint"],
                       extra_cuda_cflags=["-O3", "-include", "cstdint", "-I" + glm],
                       build_directory=OUT, verbose=False)
    return artefact()


if __name__ == "__main__":
    path = build()
    print(f"[oracle] reference rasterizer: {path or 'not built (reference sources absent)'}")
    sys.exit(0)
