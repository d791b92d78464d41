"""TEST INFRASTRUCTURE ONLY -- imports the *unmodified* reference (apple/ml-neuman) from the tree named by
$NEUMAN_REFERENCE, so that golden vectors can be generated from it (tools/make_golden*.py).  Nothing in the test suite,
bench.py or the library needs it.

The reference imports eight third-party packages that are NOT used on the hot path (SURVEY.md §8c): igl, pytorch3d,
open3d, matplotlib, imageio, lpips, tensorboardX, skimage.  They are replaced by empty stub modules.  `igl` is special:
three of its functions ARE on the hot path (utils/ray_utils.py:53,55,70); the stub routes them to the float64
brute-force restatement in oracle/mesh_oracle.py ("parity unpinned" for that one stage -- libigl 2.2.1 itself is not
available, environment.yml:13).
"""
import importlib
import os
import sys
import types



REF_ROOT = os.environ.get("NEUMAN_REFERENCE", "")


def available():
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "utils"))


class _Anything:
    """Attribute sink: any attribute access / call returns another sink."""
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Anything()


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    def fallback(attr):                      # module-level fallback (PEP 562); dunders stay missing (inspect probes __file__)
        if attr.startswith("__"):
            raise AttributeError(attr)
        return _Anything
    m.__getattr__ = fallback
    sys.modules[name] = m
    return m


def install_stubs():
    import torch                        # noqa: F401  (torch inspects sys.modules while importing: load it before the stubs exist)
    from oracle import mesh_oracle
    if "igl" not in sys.modules or not hasattr(sys.modules["igl"], "_neuman_stub"):
        _stub("igl",
              _neuman_stub=True,
              point_mesh_squared_distance=mesh_oracle.point_mesh_squared_distance,
              barycentric_coordinates_tri=mesh_oracle.barycentric_coordinates_tri,
              signed_distance=mesh_oracle.signed_distance)
    for name in ["pytorch3d", "pytorch3d.structures", "pytorch3d.renderer", "pytorch3d.renderer.mesh",
                 "pytorch3d.renderer.mesh.shader", "pytorch3d.io", "pytorch3d.ops",
                 "open3d", "matplotlib", "matplotlib.pyplot", "matplotlib.cm", "imageio", "lpips",
                 "tensorboardX", "skimage", "skimage.metrics", "skimage.io", "tqdm_stub"]:
        if name not in sys.modules:
            _stub(name)
    # make "from a.b import c" work for dotted stubs
    for name in list(sys.modules):
        if "." in name and isinstance(sys.modules[name], types.ModuleType):
            parent, child = name.rsplit(".", 1)
            if parent in sys.modules and not hasattr(sys.modules[parent], "_neuman_stub"):
                try:
                    setattr(sys.modules[parent], child, sys.modules[name])
                except Exception:
                    pass


def load():
    """Returns a namespace with the reference's hot-path modules imported."""
    if not available():
        raise RuntimeError(f"reference tree not found (set NEUMAN_REFERENCE): {REF_ROOT!r}")
    install_stubs()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    ns = types.SimpleNamespace()
    ns.vanilla = importlib.import_module("models.vanilla")
    ns.smpl = importlib.import_module("models.smpl")
    ns.ray_utils = importlib.import_module("utils.ray_utils")
    ns.render_utils = importlib.import_module("utils.render_utils")
    ns.human_nerf = importlib.import_module("models.human_nerf")
    ns.constant = importlib.import_module("utils.constant")
    ns.pinhole_camera = importlib.import_module("cameras.pinhole_camera")
    ns.camera_pose = importlib.import_module("cameras.camera_pose")
    ns.captures = importlib.import_module("cameras.captures")
    return ns
