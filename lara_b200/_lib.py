"""ctypes binding of ``libsurfel_b200.so`` (the C ABI in include/surfel_rasterizer.h).

There is no fallback path: if the shared library is missing or does not export
the expected ABI the import of :mod:`lara_b200` still succeeds (so that LaRa's
CPU-only plumbing can import ``diff_surfel_rasterization``), but the first use of
the rasterizer raises ``RuntimeError`` loudly.

Every entry that enqueues work is called through :func:`launch`, which passes torch's current stream.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_void_p
from typing import Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsurfel_b200.so")
ABI_VERSION = 13
CAM_FLOATS, CAM_VIEW, CAM_CAMPOS, CAM_BG = 24, 0, 16, 19      # include/surfel_rasterizer.h SRF_CAM_*


class MsSsimAddr(Structure):
    """srf_ms_ssim_addr: element (b, c, y, x) at b sb + c sc + y sy + (x // wv) sv + (x % wv) sx."""
    _fields_ = [("sb", c_int64), ("sc", c_int64), ("sy", c_int64), ("sx", c_int64), ("sv", c_int64), ("wv", c_int64)]


class PfImageAddr(Structure):
    """srf_pf_image_addr: element strides (ss, sv, sc, sy, sx) of img_ref [S,Vs,3,H,W]."""
    _fields_ = [("ss", c_int64), ("sv", c_int64), ("sc", c_int64), ("sy", c_int64), ("sx", c_int64)]


_A = POINTER(MsSsimAddr)
_I3 = POINTER(c_int)            # host int[3]
_P5 = POINTER(c_void_p)         # host void*[5]
MESH_CAM_FLOATS = 24            # include/surfel_mesh.h SRF_MESH_CAM_FLOATS

# name -> (restype, argtypes); mirrors include/surfel_rasterizer.h one to one
_P = c_void_p
SIGNATURES = {
    "srf_abi_version": (c_int, []),
    "srf_last_error": (c_char_p, []),
    "srf_views_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, c_size_t, c_int, POINTER(c_size_t)]),
    "srf_state_layout": (c_int, [c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t), POINTER(c_size_t)]),
    "srf_views_forward_render": (c_int, [
        _P, c_int, c_int, c_int, c_int,     # stream, V, P, H, W
        c_size_t, _P, _P,                   # capacity, geom_state, tile_state
        _P, _P, _P,                         # entries, point_list, image_state
        _P, _P, _P,                         # cams, out_color, out_others
        c_int,                              # for_backward
    ]),
    "srf_views_subset_workspace_bytes": (c_int, [c_int, POINTER(c_size_t)]),
    "srf_scenes_forward": (c_int, [
        _P, c_int, c_int, c_int, c_int, c_int,  # stream, S, Vs, P, D, M
        _P, _P, _P,                         # means3D, shs, colors_precomp
        _P, _P, _P,                         # opacities, scales, rotations
        _P, _P, _P,                         # transMat_precomp, cams, tan_fov (host float [S,2])
        c_int, c_int, c_int, c_size_t,      # H, W, prefiltered, capacity
        _P, _P, _P, _P, _P, _P,             # radii, geom_state, tile_state, entries, point_list, image_state
        _P, _P, _P, _P,                     # out_color, out_others, num_rendered_host, count_event
        c_int, c_int,                       # raw_activations, for_backward
    ]),
    "srf_scenes_subset_forward": (c_int, [
        _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int,  # stream, S, Vs, P, n, n_max, D, M
        _P, _P, _P, _P, _P, _P,             # idx, offsets, means3D, shs, colors_precomp, cams
        c_int, c_int, c_size_t,             # H, W, capacity
        _P, _P, _P, _P, c_size_t, c_int,    # coarse radii, geom_state, tile_state, point_list, capacity, for_backward
        _P, _P, _P, _P, _P,                 # radii, geom_state, tile_state, point_list, image_state
        _P, _P, _P, c_int,                  # out_color, out_others, workspace, for_backward
    ]),
    "srf_scenes_backward": (c_int, [
        _P, c_int, c_int, c_int, _P, c_int, c_int,   # stream, S, Vs, P, offsets, D, M
        c_int, c_int, c_size_t, _P,              # H, W, capacity, cams
        _P, _P, c_int,                           # means3D, shs, colors_were_precomputed
        _P, _P, c_int,                           # scales, rotations, transmat_was_precomputed
        _P, _P,                                  # tan_fov (host float [S,2]), radii
        _P, _P, _P, _P,                          # geom_state, tile_state, point_list, image_state
        _P, _P,                                  # dL_dout_color, dL_dout_others
        _P, c_int,                               # scratch, accumulate
        _P, _P, _P, _P,                          # dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors
        _P, _P, _P, _P,                          # dL_dopacity, dL_dscales, dL_drotations, dL_dtransMat
        c_int, c_int,                            # raw_activations, deterministic
    ]),
    "srf_views_backward_deterministic_scratch_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "srf_views_epilogue_forward": (c_int, [_P, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_views_epilogue_backward": (c_int, [_P, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_loss_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_loss_deterministic_workspace_bytes": (c_int, [c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_loss_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_float, c_float, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_loss_passes_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_loss_passes_deterministic_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_loss_passes_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_float, c_float, c_float,
                                         _P, _P, _P, _P, _P, _P, _P,   # image, image_fine, target, rn, dn, acc, upstream
                                         _P, _P, _P, _P, _P]),         # g_image, g_image_fine, g_rn, g_dn, g_dist
    "srf_decoder_layout_forward": (c_int, [_P, c_size_t, c_int, c_int, c_int, c_float, c_float, c_float, _P, _P, _P, _P, _P, _P, _P]),
    "srf_decoder_layout_backward": (c_int, [_P, c_size_t, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P]),
    "srf_point_feats_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "srf_point_feats_backward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                         _P]),
    "srf_point_feats_deterministic_workspace_bytes": (c_int, [c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_point_feats_scenes_forward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int,  # stream .. n, H, W
                                               _P, _P, _P, _P, _P,        # offsets (host), rows, centers, w2cs, ixts
                                               _P, POINTER(PfImageAddr),  # img_ref and its strides (host)
                                               _P, _P, _P, _P]),          # image, acc, depth, feats
    "srf_point_feats_scenes_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                                _P, _P, _P, _P, _P,
                                                _P, POINTER(PfImageAddr),
                                                _P, _P, _P, _P,           # image, acc, depth, g_feats
                                                _P, _P, _P, _P, _P]),     # g_centers, g_image, g_acc, g_depth, workspace
    "srf_point_feats_scenes_deterministic_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_ms_ssim_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_ms_ssim_workspace_layout": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t),
                                             POINTER(c_int)]),
    "srf_ms_ssim_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _A, _P, _A, c_float, c_int, _P, _P]),
    "srf_ms_ssim_backward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _A, _P, _A, c_float, c_int, _P, _P, _P, _A]),
    "srf_ms_ssim_passes_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_ms_ssim_passes_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _A, _P, _A, c_float, _P, _P]),
    "srf_ms_ssim_passes_backward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _A, _P, _A, c_float, _P, _P, _P,
                                            _P, _A, c_int]),
    "srf_ssim_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_ssim_forward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _A, _P, _A, c_float, c_int, c_int, _P, _P]),
    "srf_ssim_backward": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _A, _P, _A, c_float, c_int, c_int, _P, _P, _P,
                                  _A]),
    "srf_mark_visible": (c_int, [_P, c_int, _P, _P, _P, _P]),
    # include/surfel_mesh.h
    "srf_tsdf_integrate": (c_int, [_P, _I3, _I3, c_float, c_float, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P,
                                   c_float]),
    "srf_mesh_workspace_bytes": (c_int, [_I3, POINTER(c_size_t)]),
    "srf_mesh_count": (c_int, [_P, _I3, _P, _P, _P, _P]),
    "srf_mesh_emit": (c_int, [_P, _I3, _I3, c_float, _P, _P, _P, c_int, c_int, _P, _P, _P]),
    "srf_mesh_filter_workspace_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "srf_mesh_filter_count": (c_int, [_P, c_int, c_int, _P, _P, POINTER(c_double), c_int, _P, _P]),
    "srf_mesh_filter_emit": (c_int, [_P, c_int, c_int, _P, _P, _P, _P, c_int, c_int, _P, _P, _P]),
    # include/surfel_fine_head.h
    "srf_fine_head_forward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int,   # stream, n, V, D, sh_dim, K, N
                                      _P, _P, _P, _P,                               # volume_feat, idx, point_feats, shs
                                      _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,       # norm w, b, wq, wk, wv, wo, w1, b1, w2, b2
                                      _P]),                                         # sh_out
    "srf_fine_head_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_fine_head_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int,  # stream, n, V, D, sh_dim, K, N
                                       _P, _P, _P,                                    # volume_feat, idx, point_feats
                                       _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,        # the ten parameters
                                       _P, _P,                                        # dL_dsh, workspace
                                       _P, _P, _P,                                    # dL_dvolume_feat, _dpoint_feats, _dshs
                                       _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),      # the ten parameter gradients
    # include/surfel_coarse_head.h
    "srf_coarse_head_forward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int,      # stream, rows, N, D, K, sh_dim
                                        c_float, c_float, c_float,                  # opacity / scaling shift, half_cell
                                        _P, _P, _P, _P, _P, _P, _P, _P,             # feats, group_centers, w0 .. b2
                                        _P, _P, _P, _P, _P]),                       # the five outputs
    "srf_coarse_head_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_coarse_head_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_float,   # stream .. sh_dim, half_cell
                                         _P, _P, _P, _P, _P, _P, _P, _P,            # feats, group_centers, w0 .. b2
                                         _P, _P, _P, _P, _P, _P,                    # the five upstreams, workspace
                                         _P, _P, _P, _P, _P, _P, _P]),              # dL_dfeats, the six gradients
    # include/surfel_feat_volume.h
    "srf_feat_volume_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_feat_volume_forward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int,   # stream, B, V, C, h, w, R, E
                                        c_int, c_int, c_int, c_int,                  # Vmax, H_img, W_img, n_group
                                        _P, _P, _P, _P, _P,                          # img_feats, rays, w2c, ixt, grid
                                        _P, _P, _P, _P, _P,                          # norm w, b, mlp w, b, view_embed
                                        _P, _P]),                                    # workspace, out
    "srf_feat_volume_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_int,
                                         _P, _P, _P, _P, _P,
                                         _P, _P, _P, _P,                             # norm w, b, mlp w, b
                                         _P, _P,                                     # dL_dout, workspace
                                         _P, _P, _P, _P, _P, _P]),                   # the six gradients
    # include/surfel_vol_transformer.h
    "srf_group_attn_forward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int,   # stream, B, R, g, S, C, H
                                       _P, _P, _P, _P]),                             # q, k, v, o
    "srf_group_attn_backward": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int,
                                        _P, _P, _P, _P,                              # q, k, v, dL_do
                                        _P, _P, _P]),                                # dL_dq, dL_dk, dL_dv
    "srf_add_layernorm_forward": (c_int, [_P, c_int, c_int, c_float,                 # stream, rows, C, eps
                                          _P, _P, _P, _P, _P, _P]),                  # a, b, gamma, beta, y, n
    "srf_add_layernorm_workspace_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "srf_add_layernorm_backward": (c_int, [_P, c_int, c_int, c_float,
                                           _P, _P, _P, _P, _P,                       # y, gamma, dL_dn, dL_dy, workspace
                                           _P, _P, _P]),                             # dL_da, d_gamma, d_beta
    # include/surfel_eval.h
    "srf_eval_workspace_bytes": (c_int, [POINTER(c_size_t)]),
    "srf_eval_metrics": (c_int, [_P, c_int, c_int, c_int, c_int, c_int,   # stream, V, H, W, v0, v1
                                 _P, _A, _P, _A,                          # image, target
                                 _P, _A, _P, _A, _P, _A,                  # depth, depth_gt, mask
                                 c_int, POINTER(c_double), _P, _P]),      # n_thresholds, thresholds, workspace, out
    "srf_video_frames": (c_int, [_P, c_int, c_int, c_int,                 # stream, N, H, W
                                 _P, _A, _P, _A, _P, _A,                  # image, normal, alpha
                                 _P, _P]),                                # rgb, nrm
    # include/surfel_batch.h
    "srf_batch_assemble": (c_int, [_P, c_int, c_int, c_int, c_int,      # stream, B, N, H, W
                                   _P, _P, _P,                           # rgba, normal, bg
                                   _P, _P, _P, _P,                       # i2w, i2w_down, origin, nrm_rot
                                   _P, _P, _P, _P, _P]),                 # tar_rgb, tar_msk, tar_nrm, tar_rays, tar_rays_down
    "srf_batch_cameras": (c_int, [_P, c_int, _P, _P, _P]),                 # stream, n, c2w, bg, cams
    # include/surfel_finetune.h
    "srf_gaussian_adam_step": (c_int, [_P, c_int, c_int, _P5, _P5, _P,  # stream, n, M, params, grads, moments
                                       POINTER(c_double), c_double, c_double, c_double,   # lr (host [6]), beta1, beta2, eps
                                       c_double, c_double, c_int]),     # bias_correction1, _2_sqrt, zero_grads
    # include/surfel_image_encoder.h
    "srf_vit_patchify": (c_int, [_P, c_int, c_int, c_int,                 # stream, N, H, W
                                 c_int64, c_int64, c_int64, c_int64,      # sn, sc, sy, sx
                                 _P, _P]),                                # image, patches
    "srf_vit_tokens_forward": (c_int, [_P, c_int, c_int, c_int, c_float,  # stream, N, L, C, eps
                                       _P, _P, _P, _P, _P, _P, _P,        # patch_out, bias, cls, pos0, pos_r, gamma, beta
                                       _P, _P]),                          # x, n1
    "srf_vit_tokens_workspace_bytes": (c_int, [c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_vit_tokens_backward": (c_int, [_P, c_int, c_int, c_int, c_float,
                                        _P, _P, _P, _P, _P,               # x, gamma, dL_dn1, dL_dx, workspace
                                        _P, _P, _P, _P, _P, _P]),         # dL_dtokens, d_bias, d_cls, d_pos_r, d_gamma, d_beta
    "srf_vit_layernorm_forward": (c_int, [_P, c_int, c_int, c_float,      # stream, rows, C, eps
                                          _P, _P, _P, _P, _P, _P]),       # a, b, gamma, beta, y, n
    "srf_vit_layernorm_workspace_bytes": (c_int, [c_int, c_int, POINTER(c_size_t)]),
    "srf_vit_layernorm_backward": (c_int, [_P, c_int, c_int, c_float,
                                           _P, _P, _P, _P, _P,            # y, gamma, dL_dn, dL_dy, workspace
                                           _P, _P, _P]),                  # dL_da, d_gamma, d_beta
    "srf_vit_final_norm_forward": (c_int, [_P, c_int, c_int, c_int, c_float,   # stream, N, L, C, eps
                                           _P, _P, _P, _P, _P, _P]),      # a, b, gamma, beta, y, maps
    "srf_vit_final_norm_workspace_bytes": (c_int, [c_int, c_int, c_int, POINTER(c_size_t)]),
    "srf_vit_final_norm_backward": (c_int, [_P, c_int, c_int, c_int, c_float,
                                            _P, _P, _P, _P,               # y, gamma, dL_dmaps, workspace
                                            _P, _P, _P]),                 # dL_da, d_gamma, d_beta
    "srf_profile_begin": (c_int, []),
    "srf_profile_end": (c_int, [POINTER(c_float), POINTER(c_int), c_int]),
}

_lib = None


class SurfelLibraryError(RuntimeError):
    pass


def load(path: str | None = None):
    """Load (once) and return the ctypes handle; raises if the library is unusable."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.isfile(p):
        raise SurfelLibraryError(
            f"{p} not found: the CUDA extension is not built. Run `python -m lara_b200.build` "
            "(or __graft_entry__.build()). There is no CPU or PyTorch fallback for the rasterizer.")
    lib = ctypes.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as ex:
            raise SurfelLibraryError(f"{p} does not export {name}; rebuild the extension") from ex
        fn.restype = res
        fn.argtypes = args
    if lib.srf_abi_version() != ABI_VERSION:
        raise SurfelLibraryError(f"{p}: ABI version {lib.srf_abi_version()} != expected {ABI_VERSION}")
    if path is None:
        _lib = lib
    return lib


def check(status: int, lib=None) -> None:
    if status != 0:
        l = lib or _lib
        msg = l.srf_last_error().decode("utf-8", "replace") if l is not None else "unknown error"
        raise RuntimeError(msg)


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _contig(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return None if t is None else t.contiguous()


def _dev_index(device: torch.device) -> int:
    return device.index if device.index is not None else torch.cuda.current_device()


def _raw_stream(device: torch.device) -> int:
    return torch._C._cuda_getCurrentRawStream(_dev_index(device))


class _DeviceGuard:
    """`with torch.cuda.device(d)` only when d is not already current (the common case)."""

    def __init__(self, device: torch.device):
        self.idx = device.index
        self.ctx = None

    def __enter__(self):
        if self.idx is not None and self.idx != torch.cuda.current_device():
            self.ctx = torch.cuda.device(self.idx)
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)
        return False


def launch(name: str, device: torch.device, *args) -> None:
    """Call the enqueuing entry ``name`` with torch's current stream of ``device`` as its first argument and ``args``
    after it, ``device`` current during the call.  The stream is read now, so work is enqueued on whatever stream is
    current when this runs.  A non-zero status raises ``RuntimeError`` with the library's message."""
    lib = load()
    with _DeviceGuard(device):
        check(getattr(lib, name)(_raw_stream(device), *args), lib)


def views_sizes(lib, V: int, P: int, H: int, W: int, capacity: int, for_backward: bool = True):
    """(geom, tile, image, entries, point_list, backward scratch) bytes for V back-to-back per-view workspaces; with
    ``for_backward=False`` those of a forward-only forward (image and scratch 0, a list-only point_list)."""
    b = (c_size_t * 6)()
    check(lib.srf_views_workspace_bytes(V, P, H, W, capacity, 1 if for_backward else 0, b), lib)
    return tuple(int(x) for x in b)


def _size_query(fn, *args) -> int:
    b = c_size_t()
    check(fn(*args, ctypes.byref(b)))
    return int(b.value)


def det_backward_scratch_bytes(lib, V: int, P: int) -> int:
    """Scratch of srf_scenes_backward(..., deterministic=1) for V views of P Gaussians."""
    return _size_query(lib.srf_views_backward_deterministic_scratch_bytes, V, P)


def tan_fov_array(tan_fov) -> ctypes.Array:
    """The host float [S,2] tan_fov of the srf_scenes_* entries from a sequence of (tan_fovx, tan_fovy)."""
    return (c_float * (2 * len(tan_fov)))(*(float(v) for xy in tan_fov for v in xy))


def subset_workspace_bytes(lib, P: int) -> int:
    """Workspace of srf_scenes_subset_forward for a coarse forward of P Gaussians over all its scenes."""
    return _size_query(lib.srf_views_subset_workspace_bytes, P)


def ms_ssim_workspace_bytes(lib, B: int, C: int, H: int, W: int) -> int:
    return _size_query(lib.srf_ms_ssim_workspace_bytes, B, C, H, W)


def ssim_workspace_bytes(lib, B: int, C: int, H: int, W: int) -> int:
    return _size_query(lib.srf_ssim_workspace_bytes, B, C, H, W)


def eval_workspace_bytes(lib) -> int:
    return _size_query(lib.srf_eval_workspace_bytes)


def det_point_feats_workspace_bytes(lib, V: int, H: int, W: int) -> int:
    return _size_query(lib.srf_point_feats_deterministic_workspace_bytes, V, H, W)


def det_point_feats_scenes_workspace_bytes(lib, S: int, Vs: int, H: int, W: int) -> int:
    return _size_query(lib.srf_point_feats_scenes_deterministic_workspace_bytes, S, Vs, H, W)


def det_loss_workspace_bytes(lib, V: int, H: int, W: int) -> int:
    return _size_query(lib.srf_loss_deterministic_workspace_bytes, V, H, W)


def det_loss_passes_workspace_bytes(lib, V: int, H: int, W: int, with_fine: bool) -> int:
    return _size_query(lib.srf_loss_passes_deterministic_workspace_bytes, V, H, W, 1 if with_fine else 0)


def ms_ssim_passes_workspace_bytes(lib, B: int, C: int, H: int, W: int, with_fine: bool) -> int:
    return _size_query(lib.srf_ms_ssim_passes_workspace_bytes, B, C, H, W, 1 if with_fine else 0)


def use_deterministic(requested: Optional[bool], enabled: bool, warn_only: bool) -> bool:
    """Whether an op takes its deterministic path: ``requested`` when given, else torch's switch
    (``torch.use_deterministic_algorithms``).  Warn-only mode counts as on: a deterministic implementation exists, so
    there is nothing to warn about."""
    if requested is not None:
        return bool(requested)
    return bool(enabled or warn_only)


def deterministic(requested: Optional[bool] = None) -> bool:
    """:func:`use_deterministic` with torch's current setting, read when the op runs."""
    return use_deterministic(requested, torch.are_deterministic_algorithms_enabled(),
                             torch.is_deterministic_algorithms_warn_only_enabled())


def fine_head_workspace_bytes(lib, n: int, V: int, D: int, sh_dim: int, gather: bool) -> int:
    """Workspace of srf_fine_head_backward on the current device."""
    return _size_query(lib.srf_fine_head_workspace_bytes, n, V, D, sh_dim, 1 if gather else 0)


def coarse_head_workspace_bytes(lib, rows: int, D: int, K: int, sh_dim: int) -> int:
    """Workspace of srf_coarse_head_backward on the current device."""
    return _size_query(lib.srf_coarse_head_workspace_bytes, rows, D, K, sh_dim)


def feat_volume_workspace_bytes(lib, B: int, V: int, C: int, h: int, w: int, R: int, E: int) -> int:
    """Workspace of srf_feat_volume_forward / _backward."""
    return _size_query(lib.srf_feat_volume_workspace_bytes, B, V, C, h, w, R, E)


def add_layernorm_workspace_bytes(lib, rows: int, C: int) -> int:
    """Workspace of srf_add_layernorm_backward."""
    return _size_query(lib.srf_add_layernorm_workspace_bytes, rows, C)


def layernorm_workspace_bytes(lib, entry: str, rows: int, C: int) -> int:
    """Workspace of ``{entry}_backward``, ``entry`` srf_add_layernorm or srf_vit_layernorm."""
    return _size_query(getattr(lib, entry + "_workspace_bytes"), rows, C)


def vit_tokens_workspace_bytes(lib, N: int, L: int, C: int) -> int:
    """Workspace of srf_vit_tokens_backward."""
    return _size_query(lib.srf_vit_tokens_workspace_bytes, N, L, C)


def vit_final_norm_workspace_bytes(lib, N: int, L: int, C: int) -> int:
    """Workspace of srf_vit_final_norm_backward."""
    return _size_query(lib.srf_vit_final_norm_workspace_bytes, N, L, C)


def int3(v) -> ctypes.Array:
    """A host int[3] (the mesh entries' n0 / dims)."""
    return (c_int * 3)(*(int(x) for x in v))


def mesh_workspace_bytes(lib, dims) -> int:
    return _size_query(lib.srf_mesh_workspace_bytes, int3(dims))


def mesh_filter_workspace_bytes(lib, Nv: int, Nt: int) -> int:
    """Workspace of srf_mesh_filter_count / _emit for a mesh of Nv vertices and Nt triangles."""
    return _size_query(lib.srf_mesh_filter_workspace_bytes, Nv, Nt)


def layout(lib, P: int, H: int, W: int):
    g = (c_size_t * 3)()
    t = (c_size_t * 5)()
    i = (c_size_t * 2)()
    check(lib.srf_state_layout(P, H, W, g, t, i), lib)
    return list(g), list(t), list(i)


def ms_ssim_layout(lib, B: int, C: int, H: int, W: int) -> dict:
    """srf_ms_ssim_workspace_layout: the workspace's byte offsets ("pyr", "gpyr", "part", "mean", "val", "coef",
    "total"), the per-level element indices ("pyr_l", "gpyr_l", "part_l") and geometry ("h", "w", "px", "py", "ntx",
    "nty"), each a list over the 5 levels."""
    r, lv, d = (c_size_t * 7)(), (c_size_t * 15)(), (c_int * 30)()
    check(lib.srf_ms_ssim_workspace_layout(B, C, H, W, r, lv, d), lib)
    out = dict(zip(("pyr", "gpyr", "part", "mean", "val", "coef", "total"), (int(x) for x in r)))
    for i, k in enumerate(("pyr_l", "gpyr_l", "part_l")):
        out[k] = [int(x) for x in lv[5 * i:5 * i + 5]]
    for i, k in enumerate(("h", "w", "px", "py", "ntx", "nty")):
        out[k] = [int(x) for x in d[5 * i:5 * i + 5]]
    return out


KERNEL_NAMES = ["preprocess_fwd", "tile_scan", "scatter", "sort_small", "sort_big", "render_fwd",
                "render_bwd", "preprocess_bwd"]


def profile_begin(lib=None) -> None:
    l = lib or load()
    check(l.srf_profile_begin(), l)


def profile_end(lib=None):
    """Returns {kernel name: (total ms, launches)} for the launches since profile_begin()."""
    l = lib or load()
    n = len(KERNEL_NAMES)
    ms = (c_float * n)()
    cnt = (c_int * n)()
    check(l.srf_profile_end(ms, cnt, n), l)
    return {KERNEL_NAMES[i]: (float(ms[i]), int(cnt[i])) for i in range(n)}
