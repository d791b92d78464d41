"""The C-ABI library loads and exports every symbol include/neuman_b200.h declares (no compute
calls: there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "neuman_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nm_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_path():
    syms = header_symbols()
    for needed in ("nm_ctx_create", "nm_net_pack", "nm_mlp_forward", "nm_mlp_forward_rays", "nm_raygen", "nm_near_far",
                   "nm_ray_to_samples", "nm_sample_pdf", "nm_importance_samples", "nm_raw2outputs", "nm_merge_samples",
                   "nm_mesh_set", "nm_warp_to_canonical", "nm_render_vanilla", "nm_render_smpl_nerf", "nm_render_hybrid"):
        assert needed in syms


def test_library_exports_every_declared_symbol():
    from neuman_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "run `python -m neuman_b200.build` (or __graft_entry__.build())"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in header_symbols():
        assert hasattr(lib, s), f"{s} declared in include/neuman_b200.h but not exported"
    # and the ctypes binding covers exactly the header
    assert sorted(_lib.SIGNATURES) == header_symbols()
    assert b"sm_90a" in _lib.load().nm_version()


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import neuman_b200 as nb
    with pytest.raises(Exception):
        nb._lib.Context(0)
    coarse, _ = nb.build_nerf(nb.default_opt(use_cuda=False))
    with pytest.raises(RuntimeError):
        coarse(torch.zeros(4, 3), torch.zeros(4, 3))       # CPU tensors: no fallback
    with pytest.raises(RuntimeError):
        nb.raw2outputs(torch.zeros(2, 3, 4), torch.zeros(2, 3), torch.zeros(2, 3))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "neuman_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, fn)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, fn


def test_product_reads_only_known_environment_variables():
    """No code path of the product is picked by an environment variable.  The ones it reads: the fp32 CUDA-core MLP
    mode (NEUMAN_MLP_MODE, a supported mode), the policy for range errors (NEUMAN_RANGE_POLICY, reports, selects no
    code) and the compiler the build uses (NVCC).  A read whose variable name is not a literal counts as unknown."""
    allowed = {"NEUMAN_MLP_MODE", "NEUMAN_RANGE_POLICY", "NVCC"}
    read = re.compile(r"""(?:getenv\(|os\.environ(?:\.get\(|\[)?)\s*(?:["']([A-Za-z0-9_]*)["'])?""")
    pkg = os.path.join(ROOT, "neuman_b200")
    csrc = os.path.join(pkg, "csrc")
    files = [os.path.join(csrc, f) for f in os.listdir(csrc)] + [os.path.join(pkg, f) for f in os.listdir(pkg) if f.endswith(".py")]
    found = [(os.path.basename(f), m.group(1)) for f in sorted(files) for m in read.finditer(open(f).read())]
    assert {name for _, name in found} >= {"NEUMAN_MLP_MODE", "NEUMAN_RANGE_POLICY"}, found      # the scan sees the known reads
    assert [(f, name) for f, name in found if name not in allowed] == []
