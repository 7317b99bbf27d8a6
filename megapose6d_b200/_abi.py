"""ctypes binding of libmpx.so (C ABI declared in include/mpx.h).

The product path has no CPU fallback: if the library is missing or a call fails, this module raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_size_t, c_uint32, c_void_p
from pathlib import Path
from typing import Optional

import torch

_LIB_PATH = Path(__file__).resolve().parent / "csrc" / "libmpx.so"
_lib: Optional[ctypes.CDLL] = None
ABI_VERSION = 5  # MPX_ABI_VERSION of include/mpx.h this binding was written against


class MpxError(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def _declare(lib: ctypes.CDLL) -> None:
    vp = c_void_p
    lib.mpx_abi_version.restype = c_int
    lib.mpx_act_dtype.restype = c_int
    lib.mpx_last_error.restype = c_char_p
    lib.mpx_meshdb_create.argtypes = [c_int, vp, vp, vp, vp, vp, vp, POINTER(vp)]
    lib.mpx_meshdb_destroy.argtypes = [vp]
    lib.mpx_meshdb_set_textures.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.mpx_raster_workspace_bytes.argtypes = [c_int, c_int]
    lib.mpx_raster_workspace_bytes.restype = c_size_t
    lib.mpx_raster_render.argtypes = [vp, vp, vp, vp, c_int, c_int, c_int, c_uint32, vp, vp, vp, vp, c_size_t, vp]
    lib.mpx_raster_render_fused.argtypes = [vp, vp, vp, vp, c_int, c_int, c_int, c_int, c_uint32, vp, c_int,
                                            c_int, c_int, vp, vp, c_size_t, vp]
    lib.mpx_raster_render_scene.argtypes = [vp, c_int, c_int, vp, vp, vp, vp, vp, c_int, c_int, c_uint32, vp, vp, vp,
                                            vp, vp, c_size_t, vp]
    lib.mpx_render_crop_fused.argtypes = [vp, vp, vp, vp, c_int, c_int, c_int, c_uint32, vp, c_int, c_int, c_int, vp,
                                          vp, c_int, vp, c_int, c_int, vp, vp, c_size_t, vp]
    lib.mpx_pose_init_autodepth.argtypes = [vp, c_int, vp, vp, vp, vp, c_int, vp, vp]
    lib.mpx_normalize_T.argtypes = [vp, c_int, vp, vp]
    lib.mpx_crop_geometry.argtypes = [vp, c_int, vp, vp, vp, vp, c_int, c_float, c_int, c_int, c_int, c_int,
                                      vp, vp, vp, vp]
    lib.mpx_multiview_cameras.argtypes = [vp, vp, c_int, vp, c_int, vp, vp]
    lib.mpx_pose_update.argtypes = [vp, vp, vp, vp, c_int, vp, vp]
    lib.mpx_topk_per_group.argtypes = [vp, c_int, c_int, c_int, vp, vp]
    lib.mpx_image_to_nhwc4.argtypes = [vp, c_int, c_int, c_int, c_int, vp, vp]
    lib.mpx_roi_align.argtypes = [vp, c_int, c_int, c_int, vp, vp, c_int, c_int, c_int, c_int, vp, vp]
    lib.mpx_roi_align_fused.argtypes = [vp, c_int, c_int, c_int, vp, vp, c_int, c_int, c_int, c_int, vp, c_int,
                                        vp, c_int, vp]
    lib.mpx_net_input_bytes.argtypes = [c_int, c_int, c_int, c_int]
    lib.mpx_net_input_bytes.restype = c_size_t
    lib.mpx_conv2d.argtypes = [vp, c_int, c_int, c_int, c_int, vp, vp, c_int, c_int, c_int, c_int, c_int,
                                    c_int, c_int, c_int, c_int, vp, vp, c_int, c_int, vp]
    lib.mpx_conv2d_splitk.argtypes = [vp, c_int, c_int, c_int, c_int, vp, vp, c_int, c_int, c_int, c_int, c_int,
                                           c_int, c_int, c_int, c_int, vp, vp, c_int, c_int, vp]
    lib.mpx_maxpool3x3s2.argtypes = [vp, c_int, c_int, c_int, c_int, vp, vp]
    lib.mpx_avgpool_linear.argtypes = [vp, c_int, c_int, c_int, vp, vp, c_int, vp, vp]
    lib.mpx_net_create.argtypes = [c_int, c_int, POINTER(vp), POINTER(vp), c_int, vp, vp, POINTER(vp)]
    lib.mpx_net_create_preact.argtypes = [c_int, c_int, POINTER(ctypes.c_int32), POINTER(vp), POINTER(vp), c_int, POINTER(vp), c_int,
                                          vp, vp, POINTER(vp)]
    lib.mpx_net_destroy.argtypes = [vp]
    lib.mpx_net_workspace_bytes.argtypes = [vp, c_int, c_int, c_int]
    lib.mpx_net_workspace_bytes.restype = c_size_t
    lib.mpx_net_forward.argtypes = [vp, vp, c_int, c_int, c_int, vp, vp, c_size_t, vp]
    lib.mpx_fpn_create.argtypes = [POINTER(vp), POINTER(vp), c_int, c_int, POINTER(vp)]
    lib.mpx_fpn_destroy.argtypes = [vp]
    lib.mpx_fpn_workspace_bytes.argtypes = [c_int, c_int, c_int]
    lib.mpx_fpn_workspace_bytes.restype = c_size_t
    lib.mpx_fpn_forward.argtypes = [vp, vp, c_int, c_int, c_int, POINTER(vp), POINTER(vp), POINTER(vp), vp, c_size_t, vp]
    lib.mpx_mask_paste.argtypes = [vp, vp, vp, c_int, c_int, c_int, c_int, POINTER(ctypes.c_int32), POINTER(ctypes.c_int32),
                                   vp, POINTER(vp), vp]
    i32p = POINTER(ctypes.c_int32)
    lib.mpx_roi_heads_create.argtypes = [POINTER(vp), POINTER(vp), c_int, c_int, c_int, POINTER(vp)]
    lib.mpx_roi_heads_destroy.argtypes = [vp]
    lib.mpx_roi_heads_workspace_bytes.argtypes = [vp, c_int, c_int, c_int]
    lib.mpx_roi_heads_workspace_bytes.restype = c_size_t
    lib.mpx_roi_pool.argtypes = [POINTER(vp), c_int, c_int, c_int, POINTER(c_float), c_int, c_int, c_int, vp, i32p, c_int,
                                 vp, vp, vp]
    lib.mpx_roi_box_forward.argtypes = [vp, POINTER(vp), c_int, c_int, c_int, POINTER(c_float), c_int, c_int, c_int, vp,
                                        i32p, vp, vp, vp, c_size_t, vp]
    lib.mpx_roi_mask_forward.argtypes = [vp, POINTER(vp), c_int, c_int, c_int, POINTER(c_float), c_int, c_int, c_int, c_int,
                                         vp, i32p, vp, vp, c_size_t, vp]
    lib.mpx_bop_vsd.argtypes = [c_int, c_int, c_int, vp, c_int, vp, vp, vp, c_int, vp, c_int, vp, vp, vp, vp, vp, c_int,
                                c_float, vp, vp, vp]
    lib.mpx_bop_point_errors.argtypes = [c_int, c_int, c_int, vp, vp, ctypes.c_longlong, vp, vp, ctypes.c_longlong, vp, vp,
                                         vp, vp, vp, vp, vp]
    lib.mpx_bop_gt_info.argtypes = [c_int, c_int, c_int, vp, c_int, vp, vp, vp, vp, c_float, vp, vp, vp, vp, vp]
    lib.mpx_bop_cus.argtypes = [c_int, c_int, c_int, vp, c_int, vp, c_int, vp, vp, vp, vp, vp]
    lib.mpx_bop_pose_errors.argtypes = [c_int, c_int, vp, vp, ctypes.c_longlong, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.mpx_teaser_points.argtypes = [c_int, c_int, c_int, vp, vp, c_int, vp, vp, c_int, c_float, vp, vp, vp, vp, vp, vp]
    lib.mpx_teaser_fps_workspace_bytes.argtypes = [c_int, c_int]
    lib.mpx_teaser_fps_workspace_bytes.restype = c_size_t
    lib.mpx_teaser_fps.argtypes = [c_int, c_int, vp, vp, vp, c_int, vp, vp, vp, vp, c_size_t, vp]
    lib.mpx_teaser_graph.argtypes = [c_int, c_int, vp, vp, vp, ctypes.c_double, vp, vp]
    lib.mpx_teaser_clique_workspace_bytes.argtypes = [c_int, c_int]
    lib.mpx_teaser_clique_workspace_bytes.restype = c_size_t
    lib.mpx_teaser_max_clique.argtypes = [c_int, c_int, vp, vp, ctypes.c_longlong, vp, vp, vp, vp, vp, c_size_t, vp]
    lib.mpx_teaser_solve.argtypes = [c_int, c_int, vp, vp, vp, vp, vp, ctypes.c_double, ctypes.c_double, c_int,
                                     ctypes.c_double, c_int, vp, vp, vp, vp, vp, vp]
    lib.mpx_launch_count.restype = ctypes.c_longlong
    lib.mpx_profile_enable.argtypes = [c_int]
    lib.mpx_set_sm_limit.argtypes = [c_int]
    lib.mpx_profile_summary.argtypes = [POINTER(ctypes.c_double), POINTER(ctypes.c_double),
                                        POINTER(ctypes.c_longlong)]
    for name in EXPORTS:
        getattr(lib, name)  # every declared symbol must be exported
    # diagnostic overrides of the kernel-selection bits (see include/mpx.h)
    if os.environ.get("MPX_CONV_MODE"):
        lib.mpx_conv_set_mode(int(os.environ["MPX_CONV_MODE"]))
    if os.environ.get("MPX_RASTER_MODE"):
        lib.mpx_raster_set_mode(int(os.environ["MPX_RASTER_MODE"]))


EXPORTS = [
    "mpx_abi_version", "mpx_act_dtype", "mpx_last_error", "mpx_launch_count", "mpx_set_sm_limit", "mpx_sm_count", "mpx_profile_enable", "mpx_profile_summary",
    "mpx_meshdb_create", "mpx_meshdb_destroy", "mpx_meshdb_set_textures",
    "mpx_raster_workspace_bytes", "mpx_raster_set_mode", "mpx_raster_render", "mpx_raster_render_fused", "mpx_raster_render_scene", "mpx_render_crop_fused",
    "mpx_pose_init_autodepth", "mpx_normalize_T", "mpx_crop_geometry", "mpx_multiview_cameras",
    "mpx_pose_update", "mpx_topk_per_group", "mpx_image_to_nhwc4", "mpx_roi_align", "mpx_roi_align_fused",
    "mpx_net_input_bytes", "mpx_conv2d", "mpx_conv2d_splitk", "mpx_conv_set_mode", "mpx_maxpool3x3s2", "mpx_avgpool_linear",
    "mpx_net_create", "mpx_net_create_preact", "mpx_net_destroy", "mpx_net_set_graphs", "mpx_net_workspace_bytes", "mpx_net_forward",
    "mpx_fpn_create", "mpx_fpn_destroy", "mpx_fpn_workspace_bytes", "mpx_fpn_forward", "mpx_mask_paste",
    "mpx_roi_heads_create", "mpx_roi_heads_destroy", "mpx_roi_heads_workspace_bytes", "mpx_roi_pool", "mpx_roi_box_forward",
    "mpx_roi_mask_forward",
    "mpx_bop_vsd", "mpx_bop_point_errors", "mpx_bop_gt_info", "mpx_bop_cus", "mpx_bop_pose_errors",
    "mpx_teaser_points", "mpx_teaser_fps_workspace_bytes", "mpx_teaser_fps", "mpx_teaser_graph",
    "mpx_teaser_clique_workspace_bytes", "mpx_teaser_max_clique", "mpx_teaser_solve",
]


def lib() -> ctypes.CDLL:
    """Load libmpx.so (once). Raises MpxError when the extension has not been built."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise MpxError(
                f"{_LIB_PATH} is missing: build it with `python -m megapose6d_b200.build` "
                "(there is no CPU fallback for the CUDA path)"
            )
        handle = ctypes.CDLL(str(_LIB_PATH))
        _declare(handle)
        if handle.mpx_abi_version() != ABI_VERSION:
            raise MpxError(f"{_LIB_PATH} has ABI version {handle.mpx_abi_version()}, this package needs {ABI_VERSION}: "
                           "rebuild it with `python -m megapose6d_b200.build --force`")
        _lib = handle
    return _lib


def act_dtype() -> torch.dtype:
    """torch dtype of the library's 16-bit weights / activations / network input (include/mpx.h: mpx_act_dtype)."""
    return torch.float16 if lib().mpx_act_dtype() == 0 else torch.bfloat16


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().mpx_last_error()
        raise MpxError(f"libmpx error {rc}: {msg.decode() if msg else '?'}")


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise MpxError("libmpx needs CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise MpxError("libmpx needs contiguous tensors")
    return t.data_ptr()


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream
