"""numpy/ctypes wrapper of the CPU oracle (``oracle/surfel_oracle.c``).

TEST INFRASTRUCTURE ONLY -- importable from tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline leg; never from lara_b200/.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import POINTER, c_float, c_int, c_uint8, c_uint32, c_void_p
from typing import Dict, Optional

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle.so")


class _In(ctypes.Structure):
    _fields_ = [("P", c_int), ("D", c_int), ("M", c_int), ("H", c_int), ("W", c_int),
                ("tanfovx", c_float), ("tanfovy", c_float),
                ("bg", c_void_p), ("means3D", c_void_p), ("shs", c_void_p), ("colors_precomp", c_void_p),
                ("opacities", c_void_p), ("scales", c_void_p), ("rotations", c_void_p),
                ("viewmatrix", c_void_p), ("campos", c_void_p)]


_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "surfel_oracle.c")
    if force or not os.path.isfile(LIB) or os.path.getmtime(LIB) < os.path.getmtime(src):
        subprocess.run(["make", "-C", HERE, "-B", "liboracle.so"], check=True,
                       stdout=subprocess.DEVNULL)
    return LIB


def load():
    global _lib
    if _lib is None:
        build()
        lib = ctypes.CDLL(LIB)
        lib.oracle_forward.restype = c_void_p
        lib.oracle_forward.argtypes = [POINTER(_In)]
        lib.oracle_destroy.argtypes = [c_void_p]
        lib.oracle_backward.restype = c_int
        lib.oracle_backward.argtypes = [c_void_p] + [c_void_p] * 10
        lib.oracle_ntiles.restype = c_int
        lib.oracle_ntiles.argtypes = [c_void_p]
        lib.oracle_num_rendered.restype = c_uint32
        lib.oracle_num_rendered.argtypes = [c_void_p]
        lib.oracle_threads.restype = c_int
        for name in ("radii", "depths", "transmat", "center", "normal", "rgb", "clamped", "tiles_touched",
                     "point_list", "ranges", "accum", "n_contrib", "out_color", "out_others", "masks"):
            fn = getattr(lib, "oracle_" + name)
            fn.restype = c_void_p
            fn.argtypes = [c_void_p]
        _lib = lib
    return _lib


def _f32(a) -> Optional[np.ndarray]:
    if a is None:
        return None
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


def _view(ptr, dtype, shape):
    n = int(np.prod(shape))
    if n == 0 or not ptr:
        return np.zeros(shape, dtype=dtype)
    buf = (ctypes.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()


class OracleRun:
    """One forward of the oracle; keeps the state alive for ``backward``."""

    def __init__(self, *, means3D, opacities, scales, rotations, viewmatrix, campos, bg,
                 image_height, image_width, tanfovx, tanfovy, shs=None, colors_precomp=None, sh_degree=0):
        lib = load()
        self._keep = dict(
            means3D=_f32(means3D), opacities=_f32(opacities).reshape(-1), scales=_f32(scales),
            rotations=_f32(rotations), viewmatrix=_f32(viewmatrix).reshape(-1), campos=_f32(campos),
            bg=_f32(bg), shs=_f32(shs), colors_precomp=_f32(colors_precomp))
        k = self._keep
        self.P = int(k["means3D"].shape[0])
        self.M = int(k["shs"].shape[1]) if k["shs"] is not None else 0
        self.H, self.W = int(image_height), int(image_width)

        def p(a):
            return a.ctypes.data if a is not None else None

        arg = _In(self.P, int(sh_degree), self.M, self.H, self.W, float(tanfovx), float(tanfovy),
                  p(k["bg"]), p(k["means3D"]), p(k["shs"]), p(k["colors_precomp"]), p(k["opacities"]),
                  p(k["scales"]), p(k["rotations"]), p(k["viewmatrix"]), p(k["campos"]))
        self._h = lib.oracle_forward(ctypes.byref(arg))
        if not self._h:
            raise MemoryError("oracle_forward failed")
        h, P, H, W = self._h, self.P, self.H, self.W
        self.ntiles = lib.oracle_ntiles(h)
        self.num_rendered = int(lib.oracle_num_rendered(h))
        R = self.num_rendered
        self.radii = _view(lib.oracle_radii(h), np.int32, (P,))
        self.depths = _view(lib.oracle_depths(h), np.float32, (P,))
        self.transMat = _view(lib.oracle_transmat(h), np.float32, (P, 9))
        self.center = _view(lib.oracle_center(h), np.float32, (P, 2))
        self.normal = _view(lib.oracle_normal(h), np.float32, (P, 3))
        self.rgb = _view(lib.oracle_rgb(h), np.float32, (P, 3))
        self.clamped = _view(lib.oracle_clamped(h), np.uint8, (P, 3))
        self.tiles_touched = _view(lib.oracle_tiles_touched(h), np.uint32, (P,))
        self.point_list = _view(lib.oracle_point_list(h), np.uint32, (R,)) if P else np.zeros((0,), np.uint32)
        self.ranges = _view(lib.oracle_ranges(h), np.uint32, (self.ntiles, 2))
        self.masks = _view(lib.oracle_masks(h), np.uint32, (8, R)) if P else np.zeros((8, 0), np.uint32)
        self.accum = _view(lib.oracle_accum(h), np.float32, (3, H, W))
        self.n_contrib = _view(lib.oracle_n_contrib(h), np.uint32, (2, H, W))
        self.color = _view(lib.oracle_out_color(h), np.float32, (3, H, W))
        self.allmap = _view(lib.oracle_out_others(h), np.float32, (8, H, W))

    def backward(self, grad_color, grad_allmap) -> Dict[str, np.ndarray]:
        lib = load()
        gc, ga = _f32(grad_color), _f32(grad_allmap)
        P, M = self.P, self.M
        out = {
            "means3D": np.zeros((P, 3), np.float32), "means2D": np.zeros((P, 3), np.float32),
            "sh": np.zeros((P, M, 3), np.float32), "colors": np.zeros((P, 3), np.float32),
            "opacities": np.zeros((P, 1), np.float32), "scales": np.zeros((P, 2), np.float32),
            "rotations": np.zeros((P, 4), np.float32), "transMat": np.zeros((P, 9), np.float32),
        }
        rc = lib.oracle_backward(self._h, gc.ctypes.data, ga.ctypes.data,
                                 out["means3D"].ctypes.data, out["means2D"].ctypes.data, out["sh"].ctypes.data,
                                 out["colors"].ctypes.data, out["opacities"].ctypes.data, out["scales"].ctypes.data,
                                 out["rotations"].ctypes.data, out["transMat"].ctypes.data)
        if rc != 0:
            raise MemoryError("oracle_backward failed")
        return out

    def close(self):
        if getattr(self, "_h", None):
            load().oracle_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def run_scene(sc: dict, cam, bg, **kw) -> OracleRun:
    """Convenience: oracle forward for a lara_b200.scene scene + Camera."""
    return OracleRun(means3D=sc["means3D"], opacities=sc["opacities"], scales=sc["scales"],
                     rotations=sc["rotations"], shs=sc.get("shs"), sh_degree=sc.get("sh_degree", 0),
                     viewmatrix=cam.viewmatrix, campos=cam.campos, bg=bg,
                     image_height=cam.image_height, image_width=cam.image_width,
                     tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, **kw)


def threads() -> int:
    return int(load().oracle_threads())


# ---------------------------------------------------------------------------------------------------------------------
# Float64 replay of a forward's own decisions, with an error bound per element (surfel_oracle.c: oracle_replay, whose
# header derives the bound).  The per-Gaussian part (AABB centre, homography, quaternion, SH, fused activations, the
# densification statistic, the view loop) is vectorised here over the Gaussians with the same per-operation rules.
# ---------------------------------------------------------------------------------------------------------------------

class _ReplayIn(ctypes.Structure):
    _fields_ = [("P", c_int), ("H", c_int), ("W", c_int)] + \
        [(n, c_void_p) for n in ("T", "center", "opacity", "normal", "rgb", "ranges", "point_list", "n_contrib", "masks")] + \
        [("mask_stride", ctypes.c_longlong)] + \
        [(n, c_void_p) for n in ("tiles", "bg", "dL_dpix", "dL_dothers", "lowpass")] + [("fix_lowpass", c_int)]


class _ReplayOut(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("img", "img_e", "g", "g_e", "npairs", "nlow", "band")] + \
        [("counts", ctypes.c_int64 * 4)]


K = 2.0 ** -23          # one fp32 ulp, relative: the per-operation unit of the bound


def replay(state: dict, bg, grad_color, grad_allmap, tiles=None, lowpass=None, fix_lowpass=False) -> dict:
    """Blend forward and backward in double under the decisions of `state` (keys as lara_b200.debug.unpack_state:
    transMat, means2D, opacity, normal, rgb, ranges, point_list, n_contrib, contrib_masks).  `tiles`: bool [ntiles] of
    the tiles to replay.  `lowpass`: uint8 [num_rendered, 256] footprint choices, written, or read with fix_lowpass.
    Returns images [14,H,W] (colour, allmap, accum) and per-Gaussian partials g [P,18] (dT[9], dmean2D[2],
    dnormal[3], dopacity, dcolor[3]), each with its bound (img_e, g_e), plus pair counts."""
    lib = load()
    if not hasattr(lib, "_replay_ready"):
        lib.oracle_replay.restype = c_int
        lib.oracle_replay.argtypes = [POINTER(_ReplayIn), POINTER(_ReplayOut)]
        lib._replay_ready = True
    d = lambda a: np.ascontiguousarray(np.asarray(a), dtype=np.float64)
    u = lambda a: np.ascontiguousarray(np.asarray(a).view(np.uint32) if np.asarray(a).dtype == np.int32 else np.asarray(a),
                                       dtype=np.uint32)
    T, cen, op, nrm, rgb = (d(state[k]) for k in ("transMat", "means2D", "opacity", "normal", "rgb"))
    P = T.shape[0]
    nc = u(state["n_contrib"])
    H, W = nc.shape[1], nc.shape[2]
    ranges, plist, masks = u(state["ranges"]), u(state["point_list"]), u(state["contrib_masks"])
    keep = [T, cen, op, nrm, rgb, ranges, plist, nc, masks]
    f = lambda a: np.ascontiguousarray(np.asarray(a.detach().cpu() if hasattr(a, "detach") else a), dtype=np.float32)
    bgf, gc, ga = f(bg), f(grad_color), f(grad_allmap)
    tl = None if tiles is None else np.ascontiguousarray(tiles, dtype=np.uint8)
    keep += [bgf, gc, ga, tl, lowpass]
    p = lambda a: None if a is None else a.ctypes.data
    arg = _ReplayIn(P, H, W, p(T), p(cen), p(op), p(nrm), p(rgb), p(ranges), p(plist), p(nc), p(masks),
                    masks.shape[1], p(tl), p(bgf), p(gc), p(ga), p(lowpass), 1 if fix_lowpass else 0)
    out = dict(img=np.zeros((14, H, W)), img_e=np.zeros((14, H, W)), g=np.zeros((P, 18)), g_e=np.zeros((P, 18)),
               npairs=np.zeros(P, np.int64), nlow=np.zeros(P, np.int64), band=np.zeros(P, np.uint8))
    res = _ReplayOut(*(out[k].ctypes.data for k in ("img", "img_e", "g", "g_e", "npairs", "nlow", "band")))
    if lib.oracle_replay(ctypes.byref(arg), ctypes.byref(res)) != 0:
        raise MemoryError("oracle_replay failed")
    out.update(pairs=res.counts[0], lowpass_pairs=res.counts[1], band_pairs=res.counts[2], pixels=res.counts[3])
    return out


class EB:
    """float64 value with a bound on the error of an fp32 evaluation of the same formula: the per-operation rules of
    the replay (surfel_oracle.c), over numpy arrays.  A float operand is a constant: exact when it is an fp32 value,
    else rounded to fp32 (K/2 relative)."""
    __array_priority__ = 100

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, dtype=np.float64)

    @staticmethod
    def w(o):
        if isinstance(o, EB):
            return o
        o = np.asarray(o, dtype=np.float64)
        return EB(o, np.where(o.astype(np.float32).astype(np.float64) == o, 0.0, 0.5 * K * np.abs(o)))

    def __add__(a, b):
        b = EB.w(b)
        return EB(a.v + b.v, a.e + b.e + K * (np.abs(a.v) + np.abs(b.v)))
    __radd__ = __add__

    def __sub__(a, b):
        return a + (-EB.w(b))

    def __rsub__(a, b):
        return EB.w(b) + (-a)

    def __neg__(a):
        return EB(-a.v, a.e)

    def __mul__(a, b):
        b = EB.w(b)
        v = a.v * b.v
        return EB(v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + K * np.abs(v))
    __rmul__ = __mul__

    def __truediv__(a, b):
        b = EB.w(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = a.v / b.v
            den = np.abs(b.v) - b.e
            e = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0) + 2 * K * np.abs(v), np.inf)
        return EB(v, e)

    def __rtruediv__(a, b):
        return EB.w(b) / a

    def sqrt(a):
        v = np.sqrt(a.v)
        with np.errstate(divide="ignore", invalid="ignore"):
            return EB(v, np.where(v > 0, 0.5 * a.e / np.where(v > 0, v, 1.0), np.sqrt(a.e)) + K * v)

    def rsqrt(a):            # rsqrtf: 2 ulp
        v = 1.0 / np.sqrt(a.v)
        return EB(v, v * 0.5 * a.e / a.v + 2 * K * v)

    def exp(a):              # expf: 2 ulp
        v = np.exp(a.v)
        return EB(v, v * (np.expm1(a.e) + 2 * K))

    def where(m, a, b):
        a, b = EB.w(a), EB.w(b)
        return EB(np.where(m, a.v, b.v), np.where(m, a.e, b.e))


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435]


def _sh_basis(D, x, y, z, shv):
    """SH coefficients and d(rgb)/d(dir) (backward.cu:20-139); shv(k) -> three channel values of coefficient k."""
    coef = [SH_C0 + 0 * x] + [None] * 15
    zero = [0 * x, 0 * x, 0 * x]
    ddx, ddy, ddz = list(zero), list(zero), list(zero)
    sc = lambda s, v: [s * v[0], s * v[1], s * v[2]]
    ad = lambda a, b: [a[0] + b[0], a[1] + b[1], a[2] + b[2]]
    if D > 0:
        coef[1], coef[2], coef[3] = -SH_C1 * y, SH_C1 * z, -SH_C1 * x
        ddx, ddy, ddz = sc(-SH_C1, shv(3)), sc(-SH_C1, shv(1)), sc(SH_C1, shv(2))
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            coef[4], coef[5], coef[6] = SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2.0 * zz - xx - yy)
            coef[7], coef[8] = SH_C2[3] * xz, SH_C2[4] * (xx - yy)
            ddx = ad(ad(ad(ad(ddx, sc(SH_C2[0] * y, shv(4))), sc(SH_C2[2] * 2.0 * -x, shv(6))), sc(SH_C2[3] * z, shv(7))),
                     sc(SH_C2[4] * 2.0 * x, shv(8)))
            ddy = ad(ad(ad(ad(ddy, sc(SH_C2[0] * x, shv(4))), sc(SH_C2[1] * z, shv(5))), sc(SH_C2[2] * 2.0 * -y, shv(6))),
                     sc(SH_C2[4] * 2.0 * -y, shv(8)))
            ddz = ad(ad(ad(ddz, sc(SH_C2[1] * y, shv(5))), sc(SH_C2[2] * 2.0 * 2.0 * z, shv(6))), sc(SH_C2[3] * x, shv(7)))
            if D > 2:
                coef[9] = SH_C3[0] * y * (3.0 * xx - yy)
                coef[10] = SH_C3[1] * xy * z
                coef[11] = SH_C3[2] * y * (4.0 * zz - xx - yy)
                coef[12] = SH_C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy)
                coef[13] = SH_C3[4] * x * (4.0 * zz - xx - yy)
                coef[14] = SH_C3[5] * z * (xx - yy)
                coef[15] = SH_C3[6] * x * (xx - 3.0 * yy)
                for t in [(SH_C3[0] * 3.0 * 2.0 * xy, 9), (SH_C3[1] * yz, 10), (SH_C3[2] * -2.0 * xy, 11),
                          (SH_C3[3] * -3.0 * 2.0 * xz, 12), (SH_C3[4] * (-3.0 * xx + 4.0 * zz - yy), 13),
                          (SH_C3[5] * 2.0 * xz, 14), (SH_C3[6] * 3.0 * (xx - yy), 15)]:
                    ddx = ad(ddx, sc(t[0], shv(t[1])))
                for t in [(SH_C3[0] * 3.0 * (xx - yy), 9), (SH_C3[1] * xz, 10), (SH_C3[2] * (-3.0 * yy + 4.0 * zz - xx), 11),
                          (SH_C3[3] * -3.0 * 2.0 * yz, 12), (SH_C3[4] * -2.0 * xy, 13), (SH_C3[5] * -2.0 * yz, 14),
                          (SH_C3[6] * -3.0 * 2.0 * xy, 15)]:
                    ddy = ad(ddy, sc(t[0], shv(t[1])))
                for t in [(SH_C3[1] * xy, 10), (SH_C3[2] * 4.0 * 2.0 * yz, 11), (SH_C3[3] * 3.0 * (2.0 * zz - xx - yy), 12),
                          (SH_C3[4] * 4.0 * 2.0 * xz, 13), (SH_C3[5] * (xx - yy), 14)]:
                    ddz = ad(ddz, sc(t[0], shv(t[1])))
    return coef, ddx, ddy, ddz


def _quat(q):
    """Normalised quaternion (rsqrtf) and the rows of its rotation (auxiliary.h:188-210)."""
    s = (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]).rsqrt()
    w, x, y, z = q[0] * s, q[1] * s, q[2] * s, q[3] * s
    R0 = [1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y + w * z), 2.0 * (x * z - w * y)]
    R1 = [2.0 * (x * y - w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z + w * x)]
    R2 = [2.0 * (x * z + w * y), 2.0 * (y * z - w * x), 1.0 - 2.0 * (x * x + y * y)]
    return (w, x, y, z), R0, R1, R2


def _activate(scales, rotations, raw):
    sc = [EB(scales[:, 0]), EB(scales[:, 1])]
    q = [EB(rotations[:, k]) for k in range(4)]
    qn = None
    if raw:
        sc = [s.exp() for s in sc]
        qn = ((q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3])).sqrt()
        qn = EB.where(qn.v > 1e-12, qn, EB(np.full_like(qn.v, 1e-12)))
        q = [qk / qn for qk in q]
    return sc, q, qn


def view_vjp(rec: dict, g, g_e, params: dict, cam: dict, precomp_T=False, precomp_colors=False):
    """One view's per-Gaussian vjp (backward.cu:599-649, :533-597, :451-529, :20-139), before the activations.
    rec: the view's records (transMat [P,9], clamp_bits [P], visible [P] bool); g, g_e: replay partials [P,18].
    params: means3D, scales, rotations, shs (or None), sh_degree, raw_activations; cam: viewmatrix [16], campos, tanfovx,
    tanfovy, H, W.  Returns EB arrays keyed by output (zero where the Gaussian is not visible in the view)."""
    P = g.shape[0]
    vis = np.asarray(rec["visible"], bool)
    G = [EB(np.where(vis, g[:, k], 0.0), np.where(vis, g_e[:, k], 0.0)) for k in range(18)]
    Tr = np.where(vis[:, None], np.asarray(rec["transMat"], np.float64), 1.0)
    Tu, Tv, Tw = [EB(Tr[:, k]) for k in range(3)], [EB(Tr[:, 3 + k]) for k in range(3)], [EB(Tr[:, 6 + k]) for k in range(3)]
    vT = list(G[0:9])
    dmx, dmy = G[9], G[10]
    d = Tw[0] * Tw[0] + Tw[1] * Tw[1] - Tw[2] * Tw[2]
    inv = 1.0 / d
    f = [inv, inv, -inv]
    fTw = [f[c] * Tw[c] for c in range(3)]
    dT3 = [dmx * (f[c] * Tu[c]) + dmy * (f[c] * Tv[c]) for c in range(3)]
    dL_df = [dmx * (Tu[c] * Tw[c]) + dmy * (Tv[c] * Tw[c]) for c in range(3)]
    dL_dd = _dot(dL_df, f) * (-1.0 / d)
    dd = [2.0 * Tw[0], 2.0 * Tw[1], -2.0 * Tw[2]]
    for c in range(3):
        vT[c] = vT[c] + dmx * fTw[c]
        vT[3 + c] = vT[3 + c] + dmy * fTw[c]
        vT[6 + c] = vT[6 + c] + (dT3[c] + dL_dd * dd[c])
    tfx, tfy = float(np.float32(cam["tanfovx"])), float(np.float32(cam["tanfovy"]))
    fx, fy = EB.w(cam["W"] / (2.0 * tfx)), EB.w(cam["H"] / (2.0 * tfy))
    Wc, Hc = fx * tfx, fy * tfy
    out = {"transMat": vT, "means2D": [vT[2] * Tw[2] * Wc, vT[5] * Tw[2] * Hc],
           "opacities": G[14], "colors": G[15:18]}
    zero = EB(np.zeros(P))
    means = [zero, zero, zero]
    pm = np.asarray(params["means3D"], np.float64)
    px, py, pz = EB(pm[:, 0]), EB(pm[:, 1]), EB(pm[:, 2])
    vm = np.asarray(cam["viewmatrix"], np.float64).reshape(16)
    v = [EB.w(x) for x in vm]
    if not precomp_T:
        sc, q, _ = _activate(np.asarray(params["scales"], np.float64), np.asarray(params["rotations"], np.float64),
                             params.get("raw_activations", False))
        (w, x, y, z), R0, R1, R2 = _quat(q)
        cx, cy = fx * tfx, fy * tfy
        pview = [v[0] * px + v[4] * py + v[8] * pz + v[12], v[1] * px + v[5] * py + v[9] * pz + v[13],
                 v[2] * px + v[6] * py + v[10] * pz + v[14]]
        dM = [[fx * vT[j], fy * vT[3 + j], cx * vT[j] + cy * vT[3 + j] + vT[6 + j]] for j in range(3)]
        dRS = [[v[0] * m[0] + v[1] * m[1] + v[2] * m[2], v[4] * m[0] + v[5] * m[1] + v[6] * m[2],
                v[8] * m[0] + v[9] * m[1] + v[10] * m[2]] for m in dM]
        means = list(dRS[2])
        dn = G[11:14]
        dtn = [v[0] * dn[0] + v[1] * dn[1] + v[2] * dn[2], v[4] * dn[0] + v[5] * dn[1] + v[6] * dn[2],
               v[8] * dn[0] + v[9] * dn[1] + v[10] * dn[2]]
        tn = [v[0] * R2[0] + v[4] * R2[1] + v[8] * R2[2], v[1] * R2[0] + v[5] * R2[1] + v[9] * R2[2],
              v[2] * R2[0] + v[6] * R2[1] + v[10] * R2[2]]
        cosv = -_dot(tn, pview)
        mult = np.where(cosv.v > 0, 1.0, -1.0)
        dtn = [EB(mult * t.v, t.e) for t in dtn]
        vR0, vR1, vR2 = [sc[0] * t for t in dRS[0]], [sc[1] * t for t in dRS[1]], dtn
        out["rotations"] = [
            2.0 * (x * (vR1[2] - vR2[1]) + y * (vR2[0] - vR0[2]) + z * (vR0[1] - vR1[0])),
            2.0 * (-2.0 * x * (vR1[1] + vR2[2]) + y * (vR0[1] + vR1[0]) + z * (vR0[2] + vR2[0]) + w * (vR1[2] - vR2[1])),
            2.0 * (x * (vR0[1] + vR1[0]) - 2.0 * y * (vR0[0] + vR2[2]) + z * (vR1[2] + vR2[1]) + w * (vR2[0] - vR0[2])),
            2.0 * (x * (vR0[2] + vR2[0]) + y * (vR1[2] + vR2[1]) - 2.0 * z * (vR0[0] + vR1[1]) + w * (vR0[1] - vR1[0]))]
        out["scales"] = [_dot(dRS[0], R0), _dot(dRS[1], R1)]
        out["cosv"] = cosv
    shs = params.get("shs")
    if shs is not None and not precomp_colors:
        shs = np.asarray(shs, np.float64)
        M, D = shs.shape[1], int(params["sh_degree"])
        cb = np.asarray(rec["clamp_bits"]).astype(np.int64)
        dRGB = [EB(np.where(cb & (1 << c), 0.0, G[15 + c].v), np.where(cb & (1 << c), 0.0, G[15 + c].e)) for c in range(3)]
        cp = np.asarray(cam["campos"], np.float64)
        do = [px - cp[0], py - cp[1], pz - cp[2]]
        ln = _dot(do, do).sqrt()
        dr = [t / ln for t in do]
        coef, ddx, ddy, ddz = _sh_basis(D, dr[0], dr[1], dr[2], lambda k: [EB(shs[:, k, c]) for c in range(3)])
        ddir = [_dot(ddx, dRGB), _dot(ddy, dRGB), _dot(ddz, dRGB)]
        s2 = _dot(do, do)
        i32 = 1.0 / (s2 * s2 * s2).sqrt()
        nv = [((s2 - do[0] * do[0]) * ddir[0] - do[1] * do[0] * ddir[1] - do[2] * do[0] * ddir[2]) * i32,
              (-do[0] * do[1] * ddir[0] + (s2 - do[1] * do[1]) * ddir[1] - do[2] * do[1] * ddir[2]) * i32,
              (-do[0] * do[2] * ddir[0] - do[1] * do[2] * ddir[1] + (s2 - do[2] * do[2]) * ddir[2]) * i32]
        means = [means[c] + nv[c] for c in range(3)]
        out["sh"] = [[(coef[k] * dRGB[c]) if (k < 16 and coef[k] is not None) else zero for c in range(3)]
                     for k in range(M)]
    out["means3D"] = means
    for k, val in list(out.items()):     # nothing for a Gaussian the view culled
        out[k] = _mask(val, vis)
    return out


def _mask(val, vis):
    if isinstance(val, EB):
        return EB(np.where(vis, val.v, 0.0), np.where(vis, val.e, 0.0))
    return [_mask(x, vis) for x in val]


def _sum(a, b):
    if isinstance(a, EB):
        return a + b
    return [_sum(x, y) for x, y in zip(a, b)]


def gaussian_grads(views, params: dict, opacity_rec, precomp_T=False, out=None) -> dict:
    """Sum of view_vjp results over the views (the kernel's view loop), then the vjps of the fused activations
    (backward.cu has none; renderer_2dgs.py:183-188's sigmoid / exp / normalize), and with `out` (accumulate) the
    addition into existing outputs.  Returns {name: (value [P,...], bound [P,...])}."""
    acc = views[0]
    for vw in views[1:]:
        acc = {k: _sum(acc[k], vw[k]) for k in acc if k in vw}
    if params.get("raw_activations", False) and not precomp_T:
        sc, q, qn = _activate(np.asarray(params["scales"], np.float64), np.asarray(params["rotations"], np.float64), True)
        acc["scales"] = [acc["scales"][0] * sc[0], acc["scales"][1] * sc[1]]
        qi = [EB(np.asarray(params["rotations"], np.float64)[:, k]) for k in range(4)]
        dr = acc["rotations"]
        gx = dr[0] * qi[0] + dr[1] * qi[1] + dr[2] * qi[2] + dr[3] * qi[3]
        inv = 1.0 / qn
        big = qn.v > 1e-12
        kk = gx * inv * inv * inv
        acc["rotations"] = [EB.where(big, dr[k] * inv - qi[k] * kk, dr[k] * inv) for k in range(4)]
        y = EB(np.asarray(opacity_rec, np.float64))
        acc["opacities"] = acc["opacities"] * (1.0 - y) * y
    res = {}
    for k, val in acc.items():
        if k == "cosv":
            continue
        if isinstance(val, EB):
            val = [val]
        flat = val if isinstance(val[0], EB) else [x for row in val for x in row]
        vals = np.stack([x.v for x in flat], -1)
        errs = np.stack([x.e for x in flat], -1)
        if k == "sh":
            vals, errs = vals.reshape(vals.shape[0], -1, 3), errs.reshape(errs.shape[0], -1, 3)
        if out is not None and k in out:
            base = np.asarray(out[k], np.float64).reshape(vals.shape)
            errs = errs + K * (np.abs(vals) + np.abs(base))
            vals = vals + base
        res[k] = (vals, errs)
    return res


def preprocess64(params: dict, cam: dict, clamp_bits, mult=None):
    """The records of a forward (transMat, means2D, opacity, normal, rgb) in float64 from the parameters, with the
    forward's decisions (colour clamps, normal sign) held fixed; for finite differences of the replay's forward."""
    raw = params.get("raw_activations", False)
    pm = np.asarray(params["means3D"], np.float64)
    sc = np.asarray(params["scales"], np.float64)
    q = np.asarray(params["rotations"], np.float64)
    op = np.asarray(params["opacities"], np.float64).reshape(-1)
    if raw:
        sc, op = np.exp(sc), 1.0 / (1.0 + np.exp(-op))
        q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], -1),
                  np.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], -1),
                  np.stack([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)], -1)], 1)   # rows
    Wm = np.asarray(cam["viewmatrix"], np.float64).reshape(4, 4).T       # column-major [16] -> W[r, c]
    rot, t = Wm[:3, :3], Wm[:3, 3]
    a0, a1 = R[:, 0] * sc[:, :1], R[:, 1] * sc[:, 1:]
    M0, M1, pv = a0 @ rot.T, a1 @ rot.T, pm @ rot.T + t
    fx = cam["W"] / (2.0 * float(np.float32(cam["tanfovx"])))
    fy = cam["H"] / (2.0 * float(np.float32(cam["tanfovy"])))
    cxh, cyh = cam["W"] * 0.5, cam["H"] * 0.5
    T = np.stack([M0[:, 0] * fx + M0[:, 2] * cxh, M1[:, 0] * fx + M1[:, 2] * cxh, pv[:, 0] * fx + pv[:, 2] * cxh,
                  M0[:, 1] * fy + M0[:, 2] * cyh, M1[:, 1] * fy + M1[:, 2] * cyh, pv[:, 1] * fy + pv[:, 2] * cyh,
                  M0[:, 2], M1[:, 2], pv[:, 2]], -1)
    d = T[:, 6] ** 2 + T[:, 7] ** 2 - T[:, 8] ** 2
    cen = np.stack([(T[:, 0] * T[:, 6] + T[:, 1] * T[:, 7] - T[:, 2] * T[:, 8]) / d,
                    (T[:, 3] * T[:, 6] + T[:, 4] * T[:, 7] - T[:, 5] * T[:, 8]) / d], -1)
    tn = R[:, 2] @ rot.T
    if mult is None:
        mult = np.where(-(tn * pv).sum(1) > 0, 1.0, -1.0)
    normal = tn * mult[:, None]
    if params.get("colors_precomp") is not None:
        rgb = np.asarray(params["colors_precomp"], np.float64)
    else:
        shs = np.asarray(params["shs"], np.float64)
        dirs = pm - np.asarray(cam["campos"], np.float64)
        dirs = dirs / np.linalg.norm(dirs, axis=1, keepdims=True)
        coef, _, _, _ = _sh_basis(int(params["sh_degree"]), dirs[:, 0], dirs[:, 1], dirs[:, 2],
                                  lambda k: [shs[:, k, c] for c in range(3)])
        rgb = sum(np.asarray(coef[k])[:, None] * shs[:, k] for k in range(min(shs.shape[1], 16)) if coef[k] is not None)
        rgb = rgb + 0.5
        cb = np.asarray(clamp_bits).astype(np.int64)
        rgb = np.where((cb[:, None] >> np.arange(3)) & 1, 0.0, rgb)
    return {"transMat": T, "means2D": cen, "opacity": op, "normal": normal, "rgb": rgb}, mult
