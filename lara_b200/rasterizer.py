"""Host-side mirror of the reference's Python surface for the rasterizer hot path.

Same names, argument meaning and error behaviour as
``third_party/diff-surfel-rasterization/diff_surfel_rasterization/__init__.py``
(GaussianRasterizationSettings :158-170, GaussianRasterizer :172-222,
rasterize_gaussians :21-42, _RasterizeGaussians :44-156), so that
``lightning/renderer_2dgs.py`` runs unchanged.  Underneath it calls the C ABI in
``include/surfel_rasterizer.h`` through ctypes; torch only provides device memory
and the current CUDA stream.

Differences from the reference that a caller can observe (all documented in
DESIGN.md): work is enqueued on torch's *current* stream instead of the legacy
default stream; omitted optional inputs are passed as NULL instead of
``torch.Tensor([]).cuda()`` (which costs a synchronous H2D copy each);
``grad_colors_precomp`` / ``grad_cov3Ds_precomp`` are returned only when the
corresponding input was given (autograd discards them otherwise).
"""
from __future__ import annotations

import os
import threading
import warnings
from typing import List, NamedTuple, Optional, Sequence

import torch
import torch.nn as nn

from . import _lib
from ._lib import _DeviceGuard, _dev_index, _ptr
from ._lib import _raw_stream  # noqa: F401  (still importable from here: callers of the raw entries use it)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


# ---------------------------------------------------------------------------------
# small host-side helpers
# ---------------------------------------------------------------------------------

_size_cache: dict = {}            # (V, P, H, W, capacity, for_backward) -> workspace sizes
_cam_pads: dict = {}              # device -> zero padding of a camera record
_capacity_hwm: dict = {}          # device index -> largest num_rendered seen (instances per view)
_lock = threading.Lock()          # autograd calls backward() from another host thread


def _opt(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """The reference passes empty tensors for "not given"; normalise to None."""
    if t is None or t.numel() == 0:
        return None
    return t


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        raise RuntimeError(f"expected scalar type Float but found {t.dtype} for {name}")
    return t.contiguous()


def _views_sizes(lib, V: int, P: int, H: int, W: int, capacity: int, for_backward: bool = True):
    """srf_views_workspace_bytes: the six sizes, those of a forward-only forward with for_backward=False."""
    key = (V, P, H, W, capacity, for_backward)
    v = _size_cache.get(key)
    if v is None:
        v = _lib.views_sizes(lib, V, P, H, W, capacity, for_backward)
        if len(_size_cache) > 64:
            _size_cache.clear()
        _size_cache[key] = v
    return v


def _blob(nbytes: int, device) -> torch.Tensor:
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


def initial_capacity(P: int, device: torch.device) -> int:
    """Optimistic per-view instance capacity for the binning buffers of a forward call."""
    hwm = _capacity_hwm.get(_dev_index(device), 0)
    return max(int(hwm * 1.25) + 1024, 8 * P, 1 << 16)


def _note_rendered(R: int, device: torch.device) -> None:
    idx = _dev_index(device)
    with _lock:
        if R > _capacity_hwm.get(idx, 0):
            _capacity_hwm[idx] = R


# ---------------------------------------------------------------------------------
# num_rendered read-back.  The reference blocks the host on a cudaMemcpy in the middle of every
# forward (rasterizer_impl.cu:282).  Here the count travels to a pinned slot asynchronously and is
# only *needed* by the host to verify the optimistic instance capacity, so the wait is deferred:
# a forward returns without touching the event; the count is resolved the first time somebody asks
# for it (ForwardState.num_rendered / ctx.num_rendered), when the backward of that forward starts, or
# -- without blocking -- at the next forward on the device once its event has completed.  If the
# capacity turns out to have been too small (first call of a much larger scene), stage 2 is re-run in
# place with larger buffers and a RuntimeWarning says that results consumed in between were stale.
# raster_settings.debug=True (the reference's "synchronise and check" switch) or
# SRF_SYNC_NUM_RENDERED=1 restore the eager wait inside the forward.
# ---------------------------------------------------------------------------------

_SLOT_WORDS = 32
_readback_pool: dict = {}         # device index -> list of free (pinned int32[_SLOT_WORDS], event)
_pending: dict = {}               # device index -> list of unresolved _Pending


def _take_readback(device: torch.device, words: int):
    idx = _dev_index(device)
    with _lock:
        free = _readback_pool.setdefault(idx, [])
        for k, (slot, ev) in enumerate(free):
            if slot.numel() >= words:
                return free.pop(k)
    slot = torch.zeros(max(words, _SLOT_WORDS), dtype=torch.int32).pin_memory()
    # Spinning wait (cudaEventSynchronize without cudaEventBlockingSync).  Whoever resolves a count waits at most for the
    # tile scan of that forward, and the thread has nothing else to do meanwhile.  A sleeping wait costs a wake-up: with several
    # ranks on one machine some rank wakes late every step, its GPU runs dry and all ranks wait for it at the
    # all-reduce.  SRF_BLOCKING_EVENT_WAIT=1 restores the sleeping wait.
    ev = torch.cuda.Event(blocking=os.environ.get("SRF_BLOCKING_EVENT_WAIT", "0") == "1")
    ev.record()          # materialises the cudaEvent_t so that the C entry point can record it between its two stages
    return slot, ev


def _give_readback(device: torch.device, rb) -> None:
    with _lock:
        _readback_pool.setdefault(_dev_index(device), []).append(rb)


def _eager_sync(debug: bool) -> bool:
    return bool(debug) or os.environ.get("SRF_SYNC_NUM_RENDERED", "0") == "1"


class _Pending:
    """An enqueued forward whose instance counts have not been read back yet."""

    def __init__(self, device, rb, nviews: int, capacity: int, rerun):
        self.device, self.rb, self.V, self.capacity, self.rerun = device, rb, nviews, capacity, rerun
        self.counts: Optional[List[int]] = None
        self.lock = threading.Lock()

    def ready(self) -> bool:
        return self.counts is not None or self.rb[1].query()

    def resolve(self, stale_ok: bool = False) -> List[int]:
        with self.lock:
            if self.counts is not None:
                return self.counts
            slot, ev = self.rb
            ev.synchronize()
            counts = [int(x) & 0xFFFFFFFF for x in slot[:self.V].tolist()]
            _give_readback(self.device, self.rb)
            self.rb = None
            R = max(counts) if counts else 0
            _note_rendered(R, self.device)
            if R > self.capacity:
                self.rerun(int(R * 1.25) + 1024)
                if not stale_ok:
                    warnings.warn(
                        f"surfel rasterizer: {R} instances exceeded the optimistic capacity {self.capacity}; the forward "
                        "was re-run in place, but work enqueued between the two runs read incomplete images. Set "
                        "raster_settings.debug=True or SRF_SYNC_NUM_RENDERED=1 to verify the capacity inside every forward.",
                        RuntimeWarning, stacklevel=3)
            self.rerun = None
            self.counts = counts
        with _lock:
            lst = _pending.get(_dev_index(self.device))
            if lst and self in lst:
                lst.remove(self)
        return counts


def _drain_ready(device: torch.device) -> None:
    """Resolve, without blocking, the pending forwards of this device whose read-back has landed."""
    with _lock:
        lst = list(_pending.get(_dev_index(device), ()))
    for p in lst:
        if p.ready():
            p.resolve()


class LazyCount:
    """int-like view of a forward's num_rendered that waits for the read-back only when asked."""

    def __init__(self, pending: "_Pending", view: int = 0):
        self._p, self._v = pending, view

    def __int__(self):
        return self._p.resolve()[self._v]

    __index__ = __int__

    def __eq__(self, o):
        return int(self) == o

    def __hash__(self):
        return hash(int(self))

    def __repr__(self):
        return str(int(self))


class ForwardState:
    """What a forward leaves behind for the backward (the reference's three blobs): V per-view workspaces back to
    back, and the [V, SRF_CAM_FLOATS] camera records the forward ran on.  A forward-only state
    (``for_backward=False``) keeps no image state and no point list: it cannot feed a backward."""
    __slots__ = ("geom", "tile", "image", "point_list", "capacity", "nviews", "cams", "for_backward", "_pending",
                 "_counts")

    def __init__(self, geom, tile, image, point_list, capacity, num_rendered=0, nviews: int = 1, pending=None,
                 cams=None, for_backward: bool = True):
        self.geom, self.tile, self.image, self.point_list = geom, tile, image, point_list
        self.capacity, self.nviews, self.cams, self.for_backward = capacity, nviews, cams, for_backward
        self._pending = pending
        self._counts = None if pending is not None else ([int(num_rendered)] * nviews
                                                         if not isinstance(num_rendered, (list, tuple)) else list(num_rendered))

    def resolve(self) -> List[int]:
        if self._counts is None:
            self._counts = self._pending.resolve()
            self._pending = None
        return self._counts

    @property
    def num_rendered(self):
        c = self.resolve()
        return c[0] if self.nviews == 1 else list(c)


def pack_cameras(settings_list: Sequence[GaussianRasterizationSettings], device) -> torch.Tensor:
    """[V, SRF_CAM_FLOATS] device tensor of per-view camera records (viewmatrix | campos | bg | pad) built
    from per-view settings with ONE cat kernel (the tensors are already on the device, as LaRa's MiniCam
    produces them, lightning/utils.py:33-48; the zero padding is made once per device)."""
    parts = []
    pad = _cam_pad(device)
    for rs in settings_list:
        parts += [rs.viewmatrix.reshape(16), rs.campos.reshape(3), rs.bg.reshape(3), pad]
    return torch.cat(parts).view(len(settings_list), _lib.CAM_FLOATS)


def _cam_pad(device) -> torch.Tensor:
    pad = _cam_pads.get(device)
    if pad is None:
        device = torch.device(device)
        if device.type == "cuda":
            device = torch.device("cuda", _dev_index(device))
        pad = _cam_pads.get(device)
        if pad is None:
            pad = torch.zeros(_lib.CAM_FLOATS - 22, dtype=torch.float32, device=device)
            if device.type == "cuda":
                torch.cuda.synchronize(device)      # filled before a record on any stream reads it
            _cam_pads[device] = pad
    return pad


def forward_raw(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp,
                raster_settings: GaussianRasterizationSettings, raw_activations: bool = False, *,
                for_backward: bool = True):
    """Enqueue one forward on the current stream of the tensors' device: :func:`forward_views_raw` with V = 1 on the
    settings' camera record, which the returned state keeps for :func:`backward_raw`.

    Returns (color[3,H,W], allmap[8,H,W], radii[P], ForwardState).  Inputs must already be
    normalised (None for absent, fp32, contiguous, CUDA).  ``for_backward=False``: the forward-only path, as in
    :func:`forward_views_raw`.
    """
    rs = raster_settings
    with _DeviceGuard(means3D.device):
        return _forward(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp,
                        pack_cameras([rs], means3D.device), [(rs.tanfovx, rs.tanfovy)], int(rs.image_height),
                        int(rs.image_width), rs.sh_degree, rs.prefiltered, rs.debug, raw_activations, single=True,
                        for_backward=for_backward)


def forward_views_raw(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp,
                      cams: torch.Tensor, tanfovx: float, tanfovy: float, H: int, W: int, sh_degree: int,
                      prefiltered: bool = False, debug: bool = False, raw_activations: bool = False, *,
                      for_backward: bool = True, keep_list: bool = False):
    """All V views of one Gaussian set in ONE launch set (srf_scenes_forward with S = 1): every kernel carries a view
    dimension.  `cams` is the [V, 24] device tensor of camera records (pack_cameras).
    Returns (color [V,3,H,W], allmap [V,8,H,W], radii [V,P], ForwardState with V back-to-back workspaces).
    ``for_backward=False``: the forward-only forward (srf_scenes_forward with for_backward = 0), bit-identical outputs
    without the blend's contribution record and image state; the returned state cannot feed :func:`backward_views_raw`.
    ``keep_list``: a forward-only state keeps its point list too (the tile lists a subset render filters)."""
    with _DeviceGuard(means3D.device):
        if cams.dtype != torch.float32 or not cams.is_cuda or cams.shape[1] != _lib.CAM_FLOATS or not cams.is_contiguous():
            raise RuntimeError(f"cams must be a contiguous float32 CUDA tensor [V,{_lib.CAM_FLOATS}]")
        return _forward(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp, cams,
                        [(tanfovx, tanfovy)], H, W, sh_degree, prefiltered, debug, raw_activations, single=False,
                        for_backward=for_backward, keep_list=keep_list)


def forward_batch_raw(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp,
                      cams: torch.Tensor, tan_fov: Sequence, H: int, W: int, sh_degree: int, prefiltered: bool = False,
                      debug: bool = False, raw_activations: bool = False, *, for_backward: bool = True,
                      keep_list: bool = False):
    """S scenes of Vs views each in ONE launch set (srf_scenes_forward): Gaussian inputs [S,P,...], `cams` the
    [S*Vs, 24] camera records (scene s's views are records s*Vs .. s*Vs+Vs-1), `tan_fov` S pairs (tan_fovx, tan_fovy).
    Returns (color [S*Vs,3,H,W], allmap [S*Vs,8,H,W], radii [S*Vs,P], ForwardState of S*Vs views), each view's values
    those of :func:`forward_views_raw` on its scene alone; the state feeds :func:`backward_batch_raw`."""
    with _DeviceGuard(means3D.device):
        if cams.dtype != torch.float32 or not cams.is_cuda or cams.shape[1] != _lib.CAM_FLOATS or not cams.is_contiguous():
            raise RuntimeError(f"cams must be a contiguous float32 CUDA tensor [S*Vs,{_lib.CAM_FLOATS}]")
        return _forward(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp, cams, tan_fov,
                        H, W, sh_degree, prefiltered, debug, raw_activations, single=False, for_backward=for_backward,
                        keep_list=keep_list)


def _forward(means3D, shs, colors_precomp, opacities, scales, rotations, transMat_precomp, cams, tan_fov,
             H, W, sh_degree, prefiltered, debug, raw_activations, single, for_backward, keep_list=False):
    """srf_scenes_forward on the current stream: stage 1 (preprocess + tile scan + async count read-back) and stage 2
    (binning + blend) with an optimistic capacity, then an event for whoever eventually asks for the instance counts.
    `tan_fov`: (tan_fovx, tan_fovy) of each of the S scenes, whose Gaussian inputs are [S,P,...] ([P,...] for one).
    `single`: one view, with the outputs in the reference's one-view shapes.  `for_backward` False: the forward-only
    forward and its smaller workspaces, no image state and, unless `keep_list`, no point list kept."""
    lib = _lib.load()
    device = means3D.device
    V, P = int(cams.shape[0]), int(means3D.shape[-2])
    M = int(shs.shape[-2]) if shs is not None else 0
    # The outputs are separate tensors in the caller's shapes: outputs of an autograd.Function that are views (of a
    # common base, or one view of a stacked buffer) cannot be modified in place by the caller.
    lead = () if single else (V,)
    color = torch.empty(lead + (3, H, W), dtype=torch.float32, device=device)
    allmap = torch.empty(lead + (8, H, W), dtype=torch.float32, device=device)
    radii = torch.empty(lead + (P,), dtype=torch.int32, device=device)
    capacity = initial_capacity(P, device)
    geom_b, tile_b, image_b, ent_b, pl_b = _views_sizes(lib, V, P, H, W, capacity, for_backward)[:5]
    # the state workspaces share one byte blob (sub-blobs stay 256-byte aligned: the sizes are multiples of 256)
    blob = _blob(geom_b + tile_b + image_b, device)
    geom, tile = blob[:geom_b], blob[geom_b:geom_b + tile_b]
    image = blob[geom_b + tile_b:] if for_backward else None
    if P == 0:
        # reference: zero-filled outputs, nothing rendered (rasterize_points.cu:92-94,105)
        color.zero_(); allmap.zero_(); tile.zero_()
        if not for_backward:
            pl = torch.empty((0,), dtype=torch.int32, device=device) if keep_list else None
            return color, allmap, radii, ForwardState(geom, tile, None, pl, 0, 0, nviews=V, cams=cams,
                                                      for_backward=False)
        image.zero_()
        pl = torch.empty((0,), dtype=torch.int32, device=device)
        return color, allmap, radii, ForwardState(geom, tile, image, pl, 0, 0, nviews=V, cams=cams)

    _drain_ready(device)
    rb = _take_readback(device, V)
    slot, ev = rb
    point_list = _blob(pl_b, device)
    # Stage 2 is enqueued before the counts are known on the host, so the GPU never idles behind the read-back; an
    # overflow (rare) re-runs stage 2.  The event sits between the stages: whoever resolves the counts later waits for
    # the tile scan, never for the blend.
    # the forward-only point list and entries are scratch of this call: they go back to the caching allocator when
    # it returns, stream-ordered behind the kernels that use them
    S = len(tan_fov)
    _lib.launch("srf_scenes_forward", device, S, V // S, P, int(sh_degree), M, _ptr(means3D), _ptr(shs),
                _ptr(colors_precomp), _ptr(opacities), _ptr(scales), _ptr(rotations), _ptr(transMat_precomp),
                cams.data_ptr(), _lib.tan_fov_array(tan_fov), H, W, 1 if prefiltered else 0, capacity,
                radii.data_ptr(), geom.data_ptr(), tile.data_ptr(), _blob(ent_b, device).data_ptr(), point_list.data_ptr(),
                _ptr(image), color.data_ptr(), allmap.data_ptr(), slot.data_ptr(), ev.cuda_event,
                1 if raw_activations else 0, 1 if for_backward else 0)
    state = ForwardState(geom, tile, image, point_list if for_backward or keep_list else None, capacity, nviews=V,
                         cams=cams, for_backward=for_backward)

    def rerun(new_capacity: int):
        # enqueued on whatever stream is current: a deferred re-run happens on the caller's stream
        e_b, p_b = _views_sizes(lib, V, P, H, W, new_capacity, for_backward)[3:5]
        pl2 = _blob(p_b, device)
        _lib.launch("srf_views_forward_render", device, V, P, H, W, new_capacity, geom.data_ptr(), tile.data_ptr(),
                    _blob(e_b, device).data_ptr(), pl2.data_ptr(), _ptr(image), cams.data_ptr(), color.data_ptr(),
                    allmap.data_ptr(), 1 if for_backward else 0)
        state.capacity = new_capacity
        if for_backward or keep_list:
            state.point_list = pl2

    pend = _Pending(device, rb, V, capacity, rerun)
    state._pending, state._counts = pend, None
    if _eager_sync(debug):
        pend.resolve(stale_ok=True)      # nothing has consumed the outputs yet
        state.resolve()
    else:
        with _lock:
            _pending.setdefault(_dev_index(device), []).append(pend)
    if debug:
        torch.cuda.synchronize(device)
    return color, allmap, radii, state


def _grad_outputs(P, M, device, shs, colors_precomp, transMat_precomp, out, accumulate, need_means2D):
    """Gradient tensors the caller did not supply: one small allocation each (cheaper on the host than slicing views out
    of a flat buffer; the caching allocator hands out 512-byte aligned blocks, so the kernel's vector stores are fine)."""
    new = torch.zeros if accumulate else torch.empty
    g = {"means3D": out.get("means3D"), "means2D": out.get("means2D"), "sh": out.get("sh"),
         "colors_precomp": out.get("colors_precomp"), "opacities": out.get("opacities"), "scales": out.get("scales"),
         "rotations": out.get("rotations"), "cov3Ds_precomp": out.get("cov3Ds_precomp")}
    if g["means3D"] is None:
        g["means3D"] = new((P, 3), dtype=torch.float32, device=device)
    if need_means2D and g["means2D"] is None:
        g["means2D"] = new((P, 3), dtype=torch.float32, device=device)
    if shs is not None and g["sh"] is None:
        g["sh"] = new((P, M, 3), dtype=torch.float32, device=device)
    if colors_precomp is not None and g["colors_precomp"] is None:
        g["colors_precomp"] = new((P, 3), dtype=torch.float32, device=device)
    if g["opacities"] is None:
        g["opacities"] = new((P, 1), dtype=torch.float32, device=device)
    if g["scales"] is None:
        g["scales"] = new((P, 2), dtype=torch.float32, device=device)
    if g["rotations"] is None:
        g["rotations"] = new((P, 4), dtype=torch.float32, device=device)
    if transMat_precomp is not None and g["cov3Ds_precomp"] is None:
        g["cov3Ds_precomp"] = new((P, 9), dtype=torch.float32, device=device)
    if not need_means2D:
        g["means2D"] = out.get("means2D")
    if shs is None:
        g["sh"] = None
    return g


def backward_raw(state: ForwardState, radii, means3D, shs, colors_precomp, scales, rotations,
                 transMat_precomp, raster_settings, grad_color, grad_allmap, *,
                 out: Optional[dict] = None, accumulate: bool = False, need_means2D: bool = True,
                 raw_activations: bool = False, deterministic: Optional[bool] = None):
    """Enqueue the backward of :func:`forward_raw`: :func:`backward_views_raw` with V = 1 on the camera record the
    forward kept in ``state``; returns a dict of gradient tensors.

    ``out`` may supply pre-allocated (possibly strided-into-a-flat-buffer but contiguous)
    tensors for 'means3D','sh','opacities','scales','rotations'; with ``accumulate`` the
    kernel adds into them (view-sharded accumulation).
    ``deterministic``: bit-reproducible gradients (fixed-point sums of the blend backward, DESIGN §3.13; the call then
    waits for the GPU); ``None`` follows ``torch.use_deterministic_algorithms``.
    """
    rs = raster_settings
    return backward_views_raw(state, radii, means3D, shs, colors_precomp, scales, rotations, transMat_precomp,
                              state.cams, rs.tanfovx, rs.tanfovy, int(rs.image_height), int(rs.image_width),
                              rs.sh_degree, grad_color, grad_allmap, out=out, accumulate=accumulate,
                              need_means2D=need_means2D, raw_activations=raw_activations, debug=rs.debug,
                              deterministic=deterministic)


def backward_views_raw(state: ForwardState, radii, means3D, shs, colors_precomp, scales, rotations, transMat_precomp,
                       cams: torch.Tensor, tanfovx: float, tanfovy: float, H: int, W: int, sh_degree: int,
                       grad_color, grad_allmap, *, out: Optional[dict] = None, accumulate: bool = False,
                       need_means2D: bool = False, raw_activations: bool = False, debug: bool = False,
                       deterministic: Optional[bool] = None):
    """Backward of forward_views_raw: grad_color [V,3,H,W], grad_allmap [V,8,H,W]; the per-Gaussian backward
    sums the V views in registers and writes (accumulate: adds into) every parameter-gradient row once.
    ``deterministic`` as in :func:`backward_raw`."""
    return _backward(state, radii, means3D, shs, colors_precomp, scales, rotations, transMat_precomp, cams,
                     [(tanfovx, tanfovy)], H, W, sh_degree, grad_color, grad_allmap, None, None, out, accumulate,
                     need_means2D, raw_activations, debug, deterministic)


def backward_batch_raw(state: ForwardState, radii, means3D, shs, scales, rotations, cams: torch.Tensor, tan_fov: Sequence,
                       H: int, W: int, sh_degree: int, grad_color, grad_allmap, *, offsets: Optional[torch.Tensor] = None,
                       P: Optional[int] = None, raw_activations: bool = False, debug: bool = False,
                       deterministic: Optional[bool] = None):
    """Backward of :func:`forward_batch_raw` (srf_scenes_backward): gradients shaped like the inputs, [S,P,...], each
    scene's rows the sum of its own views.  With ``offsets`` (device int64 [S+1]) the state is a subset forward's, of
    ``P`` Gaussians per view, and the inputs and gradients are the scenes' rows concatenated, [n,...].
    ``deterministic`` as in :func:`backward_raw`."""
    lead = tuple(means3D.shape[:-1])
    g = _backward(state, radii, means3D, shs, None, scales, rotations, None, cams, tan_fov, H, W, sh_degree, grad_color,
                  grad_allmap, offsets, P, None, False, False, raw_activations, debug, deterministic)
    return {k: (t.view(lead + tuple(t.shape[1:])) if t is not None else None) for k, t in g.items()}


def _backward(state: ForwardState, radii, means3D, shs, colors_precomp, scales, rotations, transMat_precomp, cams,
              tan_fov, H, W, sh_degree, grad_color, grad_allmap, offsets, P, out, accumulate, need_means2D,
              raw_activations, debug, deterministic):
    """srf_scenes_backward on the current stream for the S = len(tan_fov) scenes of ``state``: ``P`` Gaussians per view
    (None: ``means3D.shape[-2]``), ``offsets`` as in :func:`backward_batch_raw`.  Returns the gradient rows of the
    ``means3D.numel() // 3`` input rows, flat ([rows, ...]); ``out`` / ``accumulate`` as in :func:`backward_raw`."""
    if not state.for_backward:
        raise RuntimeError("backward of a forward-only render: this state comes from a forward with "
                           "for_backward=False, which keeps no contribution record or image state; run the "
                           "forward with for_backward=True to take its gradient")
    lib = _lib.load()
    device = means3D.device
    S, V = len(tan_fov), int(cams.shape[0])
    rows = means3D.numel() // 3
    if P is None:
        P = int(means3D.shape[-2])
    M = int(shs.shape[-2]) if shs is not None else 0
    g = _grad_outputs(rows, M, device, shs, colors_precomp, transMat_precomp, out or {}, accumulate, need_means2D)
    if P == 0 or rows == 0:
        return g
    state.resolve()                 # capacity verified (re-run if it overflowed) before the lists are walked again
    det = _lib.deterministic(deterministic)
    scratch_b = (_lib.det_backward_scratch_bytes(lib, V, P) if det
                 else _views_sizes(lib, V, P, H, W, state.capacity)[5])
    _lib.launch(
        "srf_scenes_backward", device, S, V // S, P, _ptr(offsets), int(sh_degree), M, H, W, state.capacity,
        cams.data_ptr(), _ptr(means3D), _ptr(shs), 1 if colors_precomp is not None else 0,
        _ptr(scales), _ptr(rotations), 1 if transMat_precomp is not None else 0, _lib.tan_fov_array(tan_fov),
        radii.data_ptr(), state.geom.data_ptr(), state.tile.data_ptr(), state.point_list.data_ptr(),
        state.image.data_ptr(), grad_color.data_ptr(), grad_allmap.data_ptr(), _blob(scratch_b, device).data_ptr(),
        1 if accumulate else 0, _ptr(g["means3D"]), _ptr(g["means2D"]), _ptr(g["sh"]), _ptr(g["colors_precomp"]),
        _ptr(g["opacities"]), _ptr(g["scales"]), _ptr(g["rotations"]), _ptr(g["cov3Ds_precomp"]),
        1 if raw_activations else 0, 1 if det else 0)
    if debug:
        torch.cuda.synchronize(device)
    return g


def _dump_snapshot(path: str, items) -> None:
    """CPU copies of the call's tensors, like the reference's cpu_deep_copy_tuple + torch.save."""
    try:
        def cpu(x):
            if isinstance(x, torch.Tensor):
                return x.detach().cpu().clone()
            if isinstance(x, tuple) and hasattr(x, "_fields"):
                return tuple(cpu(v) for v in x)
            return x
        torch.save(tuple(cpu(i) for i in items), path)
    except Exception:
        pass


def _check_settings(rs: GaussianRasterizationSettings, device) -> GaussianRasterizationSettings:
    """Device / dtype checks of the settings tensors, and `.contiguous()` exactly where the reference
    calls it (rasterize_points.cu:113-131): LaRa's MiniCam passes `w2c.transpose(0, 1)`, a
    non-contiguous view, as the view matrix (lightning/utils.py:40)."""
    fixed = {}
    for name in ("bg", "viewmatrix", "projmatrix", "campos"):
        t = getattr(rs, name)
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor")
        if t.dtype != torch.float32:
            raise RuntimeError(f"expected scalar type Float but found {t.dtype} for raster_settings.{name}")
        if not t.is_contiguous():
            fixed[name] = t.contiguous()
    return rs._replace(**fixed) if fixed else rs


def _normalise_inputs(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp):
    sh, colors_precomp = _opt(sh), _opt(colors_precomp)
    scales, rotations, cov3Ds_precomp = _opt(scales), _opt(rotations), _opt(cov3Ds_precomp)
    # shape checks of RasterizeGaussiansCUDA (rasterize_points.cu:61-71)
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    if scales is not None and (scales.ndim != 2 or scales.shape[1] != 2):
        raise RuntimeError("scales must have dimensions (num_points, 2)")
    if rotations is not None and (rotations.ndim != 2 or rotations.shape[1] != 4):
        raise RuntimeError("rotations must have dimensions (num_points, 4)")
    P = means3D.shape[0]
    means3D = _f32c(means3D, "means3D")
    opacities = _f32c(opacities, "opacity")
    if opacities.numel() != P:
        raise RuntimeError("opacity must have one entry per point")
    if sh is not None:
        sh = _f32c(sh, "sh")
        if sh.ndim != 3 or sh.shape[0] != P or sh.shape[2] != 3:
            raise RuntimeError("sh must have dimensions (num_points, M, 3)")
    if colors_precomp is not None:
        colors_precomp = _f32c(colors_precomp, "colors")
        if colors_precomp.shape != (P, 3):
            raise RuntimeError("colors must have dimensions (num_points, 3)")
    if scales is not None:
        scales = _f32c(scales, "scales")
    if rotations is not None:
        rotations = _f32c(rotations, "rotations")
    if cov3Ds_precomp is not None:
        cov3Ds_precomp = _f32c(cov3Ds_precomp, "transMat_precomp")
        if cov3Ds_precomp.numel() != P * 9:
            raise RuntimeError("transMat_precomp must have dimensions (num_points, 9)")
    if P > 0:
        if (sh is None) == (colors_precomp is None):
            raise RuntimeError("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3Ds_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3Ds_precomp is not None):
            raise RuntimeError("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    return means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp


# ---------------------------------------------------------------------------------
# the reference's public surface
# ---------------------------------------------------------------------------------

def needs_backward(*inputs) -> bool:
    """Whether a render can have a gradient: grad mode is on and a tensor input requires grad.  Decided before any
    ``autograd.Function`` runs: inside its forward grad mode is always off, and under ``torch.no_grad()``
    ``ctx.needs_input_grad`` still reports inputs that require grad.  Renders for which this is False (``no_grad``,
    ``inference_mode``, inputs that need no gradient) take the forward-only path."""
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs)


def _rasterize(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
               raw_activations, for_backward):
    """The checks of the reference's forward, then forward_raw; returns (settings, normalised inputs, color, allmap,
    radii, state)."""
    raster_settings = _check_settings(raster_settings, means3D.device)
    inputs = _normalise_inputs(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
    try:
        color, allmap, radii, state = forward_raw(*inputs, raster_settings, raw_activations=raw_activations,
                                                  for_backward=for_backward)
    except Exception:
        if raster_settings.debug:
            # same debugging aid as the reference (DSR __init__.py:83-90)
            _dump_snapshot("snapshot_fw.dump", (raster_settings, means3D, sh, colors_precomp, opacities,
                                               scales, rotations, cov3Ds_precomp))
            print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
        raise
    return raster_settings, inputs, color, allmap, radii, state


def _rasterize_any(fn, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                   raster_settings):
    """``fn.apply`` when a gradient can flow, else the forward-only path without an autograd node: the same
    (color, radii, allmap)."""
    if needs_backward(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp):
        return fn.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings)
    _, _, color, allmap, radii, _ = _rasterize(means3D, sh, colors_precomp, opacities, scales, rotations,
                                               cov3Ds_precomp, raster_settings, fn.RAW_ACTIVATIONS, False)
    return color, radii, allmap


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings):
    return _rasterize_any(_RasterizeGaussians, means3D, means2D, sh, colors_precomp, opacities, scales,
                          rotations, cov3Ds_precomp, raster_settings)


class _RasterizeGaussians(torch.autograd.Function):
    RAW_ACTIVATIONS = False     # the subclass below flips this: inputs are raw network outputs

    @classmethod
    def forward(cls, ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings):
        raster_settings, inputs, color, allmap, radii, state = _rasterize(
            means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
            cls.RAW_ACTIVATIONS, True)
        (means3D_c, sh_c, colors_c, opac_c, scales_c, rot_c, cov_c) = inputs
        ctx.raster_settings = raster_settings
        ctx.state = state
        # an int for an eager forward, else an int-like object that waits for the read-back when asked
        ctx.num_rendered = state.num_rendered if state._pending is None else LazyCount(state._pending)
        ctx.present = (sh_c is not None, colors_c is not None, scales_c is not None,
                       rot_c is not None, cov_c is not None)
        ctx.opac_shape = tuple(opacities.shape)
        ctx.raw_activations = cls.RAW_ACTIVATIONS
        dummy = means3D_c.new_empty(0)
        ctx.save_for_backward(
            colors_c if colors_c is not None else dummy, means3D_c,
            scales_c if scales_c is not None else dummy, rot_c if rot_c is not None else dummy,
            cov_c if cov_c is not None else dummy, radii, sh_c if sh_c is not None else dummy,
            state.geom, state.image, state.tile)
        ctx.mark_non_differentiable(radii)
        return color, radii, allmap

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth):
        rs = ctx.raster_settings
        (colors_c, means3D, scales, rotations, cov_c, radii, sh, geom, image, tile) = ctx.saved_tensors
        has_sh, has_col, has_sc, has_rot, has_cov = ctx.present
        state = ctx.state     # holds the index list (replaced if a deferred capacity check re-ran stage 2)
        grad_out_color = _f32c(grad_out_color, "dL_dout_color")
        grad_depth = _f32c(grad_depth, "dL_dout_others")
        try:
            g = backward_raw(state, radii, means3D,
                             sh if has_sh else None, colors_c if has_col else None,
                             scales if has_sc else None, rotations if has_rot else None,
                             cov_c if has_cov else None, rs, grad_out_color, grad_depth,
                             raw_activations=ctx.raw_activations)
        except Exception:
            if rs.debug:
                _dump_snapshot("snapshot_bw.dump", (rs, means3D, radii, sh, scales, rotations, grad_out_color, grad_depth))
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
            raise
        # order of DSR __init__.py:144-154
        if g["opacities"].shape != ctx.opac_shape:
            g["opacities"] = g["opacities"].view(ctx.opac_shape)
        return (g["means3D"], g["means2D"], g["sh"], g["colors_precomp"], g["opacities"],
                g["scales"], g["rotations"], g["cov3Ds_precomp"], None)


class _RasterizeGaussiansRaw(_RasterizeGaussians):
    """Same call, but opacities / scales / rotations are LaRa's raw network outputs (logits,
    log-scales, unnormalised quaternions): the activations of renderer_2dgs.py:183-188 and their
    vjps run inside the preprocess kernels (next-row extension, SURVEY 8f rank 1)."""
    RAW_ACTIVATIONS = True


def rasterize_gaussians_raw(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                            cov3Ds_precomp, raster_settings):
    return _rasterize_any(_RasterizeGaussiansRaw, means3D, means2D, sh, colors_precomp, opacities, scales,
                          rotations, cov3Ds_precomp, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Boolean mask of points in front of the near plane (DSR __init__.py:177-186)."""
        with torch.no_grad():
            pos = _f32c(positions, "means3D")
            rs = _check_settings(self.raster_settings, pos.device)
            P = int(pos.shape[0])
            present = torch.zeros((P,), dtype=torch.bool, device=pos.device)
            if P:
                _lib.launch("srf_mark_visible", pos.device, P, pos.data_ptr(), rs.viewmatrix.data_ptr(),
                            rs.projmatrix.data_ptr(), present.data_ptr())
        return present

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                rotations=None, cov3D_precomp=None):
        raster_settings = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales,
                                   rotations, cov3D_precomp, raster_settings)

    def forward_raw_activations(self, means3D, means2D, opacities, scales, rotations, shs=None, colors_precomp=None):
        """Extension (no reference counterpart): like ``forward`` on the scale/rotation path, but
        opacities / scales / rotations are LaRa's raw network outputs; sigmoid / exp / F.normalize
        (renderer_2dgs.py:183-188) and their vjps run inside the preprocess kernels."""
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if scales is None or rotations is None:
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        return rasterize_gaussians_raw(means3D, means2D, shs, colors_precomp, opacities, scales,
                                       rotations, None, self.raster_settings)
