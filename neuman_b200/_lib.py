"""ctypes binding of libneuman_b200.so (the C ABI declared in include/neuman_b200.h).

The library is mandatory: importing the product path without the built extension raises -- there is
no CPU / eager fallback anywhere in neuman_b200.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libneuman_b200.so")

NM_PE_POSENC, NM_PE_ROTATE = 0, 1
NM_MLP_TC_F16, NM_MLP_SIMT_F32 = 0, 1
NM_MAX_NET_SLOTS, NM_MAX_ACTORS = 16, 8


class NmNerfDesc(C.Structure):
    _fields_ = [("pts_w", C.c_void_p * 8), ("pts_b", C.c_void_p * 8),
                ("feature_w", C.c_void_p), ("feature_b", C.c_void_p),
                ("alpha_w", C.c_void_p), ("alpha_b", C.c_void_p),
                ("views_w", C.c_void_p), ("views_b", C.c_void_p),
                ("rgb_w", C.c_void_p), ("rgb_b", C.c_void_p),
                ("pos_pe_kind", C.c_int32), ("dir_pe_kind", C.c_int32),
                ("pos_min_freq", C.c_float), ("pos_max_freq", C.c_float), ("pos_n_freqs", C.c_int32),
                ("dir_min_freq", C.c_float), ("dir_max_freq", C.c_float), ("dir_n_freqs", C.c_int32)]


class NmNerfNoviewDesc(C.Structure):
    _fields_ = [("pts_w", C.c_void_p * 8), ("pts_b", C.c_void_p * 8),
                ("output_w", C.c_void_p), ("output_b", C.c_void_p),
                ("pos_pe_kind", C.c_int32),
                ("pos_min_freq", C.c_float), ("pos_max_freq", C.c_float), ("pos_n_freqs", C.c_int32)]


class NmCamera(C.Structure):
    _fields_ = [("K", C.c_double * 9), ("c2w", C.c_double * 16), ("H", C.c_int32), ("W", C.c_int32)]


class NmRenderOpts(C.Structure):
    _fields_ = [("samples_per_ray", C.c_int32), ("importance_samples_per_ray", C.c_int32),
                ("white_bkg", C.c_int32), ("mlp_mode", C.c_int32), ("rays_per_batch", C.c_int32),
                ("render_can", C.c_int32), ("near_bkg", C.c_float), ("far_bkg", C.c_float),
                ("geo_threshold", C.c_float), ("interval_comp", C.c_float)]


class NmSmplModel(C.Structure):
    _fields_ = [("v_template", C.c_void_p), ("shapedirs", C.c_void_p), ("J_regressor", C.c_void_p),
                ("weights", C.c_void_p), ("parents", C.POINTER(C.c_int32)),
                ("n_verts", C.c_int32), ("n_joints", C.c_int32), ("n_betas", C.c_int32)]


_P = C.c_void_p
_I32, _I64, _F = C.c_int32, C.c_int64, C.c_float

# name -> (restype, argtypes); every symbol include/neuman_b200.h declares
SIGNATURES = {
    "nm_ctx_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "nm_ctx_destroy": (C.c_int, [_P]),
    "nm_last_error": (C.c_char_p, [_P]),
    "nm_version": (C.c_char_p, []),
    "nm_launch_count": (_I64, [_P]),
    "nm_net_pack": (C.c_int, [_P, C.c_int, C.POINTER(NmNerfDesc), _P]),
    "nm_net_pack_noview": (C.c_int, [_P, C.c_int, C.POINTER(NmNerfNoviewDesc), _P]),
    "nm_net_pack_nerft": (C.c_int, [_P, C.c_int, C.POINTER(NmNerfDesc), _P]),
    "nm_mlp_forward": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _I64, _I32, _P, _P]),
    "nm_mlp_forward_train": (C.c_int, [_P, C.c_int, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P]),
    "nm_encode_f16": (C.c_int, [_P, C.c_int, _I32, _P, _I64, _I64, _P, _P]),
    "nm_mlp_backward": (C.c_int, [_P, C.c_int, _P, _P, _I64, _P, _P, _P, _P, _P, _P]),
    "nm_pe_backward": (C.c_int, [_P, C.c_int, _I32, _P, _I64, _P, _I32, _P, _I64, _P, _P]),
    "nm_dw_gemm": (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _P, _P, _P]),
    "nm_mlp_forward_rays": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, _I64, _I32, _P, _P]),
    "nm_raygen": (C.c_int, [_P, C.POINTER(NmCamera), C.c_int, _I64, _I64, _P, _P, _P, _P]),
    "nm_near_far": (C.c_int, [_P, _P, _P, _I64, _P, _I32, _F, _P, _P, _P]),
    "nm_near_far_mesh": (C.c_int, [_P, C.c_int, _P, _P, _I64, _F, _P, _P, _P]),
    "nm_ray_to_samples": (C.c_int, [_P, _P, _P, _P, _P, _F, _F, _I64, _I32, _I32, _P, _P, _P, _P, _P]),
    "nm_sample_pdf": (C.c_int, [_P, _P, _P, _I64, _I32, _I32, _P, _P, _P]),
    "nm_importance_samples": (C.c_int, [_P, _P, _P, _P, _P, _I64, _I32, _I32, _I32, _P, _P, _P, _P]),
    "nm_raw2outputs": (C.c_int, [_P, _P, _P, _P, _I64, _I32, _P, _F, _I32, _P, _P, _P, _P, _P, _P]),
    "nm_raw2outputs_backward": (C.c_int, [_P, _P, _P, _P, _I64, _I32, _P, _F, _I32, _P, _P, _P, _P, _P, _P]),
    "nm_merge_samples": (C.c_int, [_P, _I32, C.POINTER(_P), C.POINTER(_P), C.POINTER(_I32), _I64, _P, _P, _P]),
    "nm_mesh_set": (C.c_int, [_P, C.c_int, _P, _I32, _P, _I32, _P, _I32, _I32, _P]),
    "nm_signed_distance": (C.c_int, [_P, C.c_int, _P, _I64, _P, _P, _P, _P]),
    "nm_warp_to_canonical": (C.c_int, [_P, C.c_int, _P, _I64, _I32, _P, _P, _P, _P, _P]),
    "nm_smpl_vertex_transforms": (C.c_int, [_P, C.POINTER(NmSmplModel), _P, _P, _I32, _P, _P, _P]),
    "nm_smpl_scene_transforms": (C.c_int, [_P, C.POINTER(NmSmplModel), _P, _P, _P, C.POINTER(C.c_double), C.c_double,
                                           _P, _P, _P]),
    "nm_warp_diff_forward": (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _P, _P]),
    "nm_warp_diff_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _P, _I32, _P, _P, _P]),
    "nm_human_canonicalize": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I64, _I32, _P, _P, _P]),
    "nm_human_canonicalize_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _I32, _I32, _P, _P, _P, _P]),
    "nm_smpl_scene_forward_train": (C.c_int, [_P, C.POINTER(NmSmplModel), _P, _P, _P, _P, _F, _P, _P, _P]),
    "nm_smpl_scene_backward": (C.c_int, [_P, C.POINTER(NmSmplModel), _P, _P, _P, _P, _F, _P, _P, _P, _P, _P, _P]),
    "nm_render_vanilla": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(NmCamera), C.POINTER(NmRenderOpts), _I64, _I64, _P,
                                    _P, _P, _I32, _P]),
    "nm_render_vanilla_t": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(NmCamera), C.POINTER(NmRenderOpts), _F, _I64, _I64,
                                      _P, _P, _P, _I32, _P]),
    "nm_render_smpl_nerf": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(NmCamera), C.POINTER(NmRenderOpts), _I64, _I64, _P,
                                      _P, _P, _P, _I32, _P]),
    "nm_render_hybrid": (C.c_int, [_P, C.c_int, C.c_int, _I32, C.POINTER(_I32), C.POINTER(_I32), _I32,
                                   C.POINTER(NmCamera), C.POINTER(NmRenderOpts), _I64, _I64, _P, _P, _P, _P, _I32, _P]),
    "nm_assemble_frame": (C.c_int, [_P, _P, _I32, _I64, _I32, _P, _P, _P, _P, _P]),
    "nm_profile_enable": (C.c_int, [_P, _I32]),
    "nm_profile_read": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(_I64), C.POINTER(_I64)]),
    "nm_last_render_stats": (C.c_int, [_P, C.POINTER(_I64), C.POINTER(_I64)]),
    "nm_range_status": (C.c_int, [_P, _I32, _P]),
}

_lib = None
_lock = threading.Lock()


def load():
    """dlopen the library and bind every declared symbol (raises if the build is missing)."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m neuman_b200.build` "
                "(nvcc, sm_90a). neuman_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)            # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


class NmError(RuntimeError):
    pass


class Context:
    """One nm_ctx per (process, device)."""
    _by_device = {}

    def __init__(self, device):
        self.lib = load()
        self.device = int(device)
        h = _P()
        rc = self.lib.nm_ctx_create(self.device, C.byref(h))
        if rc != 0:
            raise NmError(f"nm_ctx_create(device={device}) failed with {rc} (is a CUDA device present?)")
        self.h = h
        self.slots = {}          # key -> slot
        self.slot_keys = [None] * NM_MAX_NET_SLOTS
        self.slot_clock = 0
        self.slot_used = [0] * NM_MAX_NET_SLOTS
        self.finalized_uids = set()   # modules with a weakref.finalize hook registered for this ctx

    @classmethod
    def get(cls, device):
        d = int(device)
        if d not in cls._by_device:
            cls._by_device[d] = cls(d)
        return cls._by_device[d]

    def stream(self):
        """The caller's current torch stream on THIS ctx's device (not the thread's current device)."""
        import torch
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def check(self, rc):
        if rc != 0:
            raise NmError(f"libneuman_b200 error {rc}: {self.lib.nm_last_error(self.h).decode()}")

    def range_check(self, clear=True):
        """Raises NmError (NM_ERR_RANGE) if a tensor-core MLP launch saturated an fp16 operand since the last check.
        Synchronises on the current stream."""
        self.check(self.lib.nm_range_status(self.h, int(bool(clear)), self.stream()))

    def launch_count(self):
        return int(self.lib.nm_launch_count(self.h))

    def profile(self, on):
        self.check(self.lib.nm_profile_enable(self.h, int(bool(on))))

    def profile_read(self):
        ms, nl, ne = C.c_double(), _I64(), _I64()
        self.check(self.lib.nm_profile_read(self.h, C.byref(ms), C.byref(nl), C.byref(ne)))
        return {"mlp_ms": ms.value, "mlp_launches": nl.value, "mlp_evals": ne.value}

    def render_stats(self):
        a, b = _I64(), _I64()
        self.check(self.lib.nm_last_render_stats(self.h, C.byref(a), C.byref(b)))
        return {"mlp_evals": a.value, "hit_rays": b.value}
