"""Synthetic scenes and cameras for parity tests and benchmarks (SURVEY.md section 8d).

Everything is generated on the CPU from a seeded ``torch.Generator`` so that the same
bits reach the candidate, the reference build and the CPU oracle.

  * ``scene(P, seed)``  mirrors LaRa's Gaussian statistics at initialisation
    (lightning/network.py:291,340-349): positions U(-0.5,0.5)^3, log-normal scales
    around ``0.0052 * (524288/P)^(1/3)`` (so the overdraw stays LaRa-like as P varies),
    random unit quaternions (w,x,y,z), sigmoid(N(-2.1792, 1.5^2)) opacities, degree-1 SH.
  * ``cameras(V, H, W, seed)`` places V OpenCV cameras on a sphere of radius 1.905
    looking at the origin (tools/gen_video_path.py:11-25) and builds the matrices the
    way ``MiniCam`` does (lightning/utils.py:22-48): viewmatrix = inverse(c2w)^T,
    projmatrix = viewmatrix @ P^T, campos = -c2w[:3,3].
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional

import torch


class Camera(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    viewmatrix: torch.Tensor   # [4,4] float32 (= w2c^T)
    projmatrix: torch.Tensor   # [4,4] float32
    campos: torch.Tensor       # [3] float32
    c2w: torch.Tensor          # [4,4] float32


def scene(P: int, seed: int = 0, sh_degree: int = 1) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device="cpu").manual_seed(seed)
    M = (sh_degree + 1) ** 2
    means3D = torch.rand((P, 3), generator=g, dtype=torch.float32) - 0.5
    s0 = 0.0052 * (524288.0 / max(P, 1)) ** (1.0 / 3.0)
    scales = torch.exp(torch.randn((P, 2), generator=g, dtype=torch.float32) * 0.3 + math.log(s0))
    rotations = torch.nn.functional.normalize(torch.randn((P, 4), generator=g, dtype=torch.float32), dim=-1)
    opacities = torch.sigmoid(torch.randn((P, 1), generator=g, dtype=torch.float32) * 1.5 - 2.1792)
    shs = torch.randn((P, M, 3), generator=g, dtype=torch.float32) * 0.5
    return {
        "means3D": means3D.contiguous(), "scales": scales.contiguous(),
        "rotations": rotations.contiguous(), "opacities": opacities.contiguous(),
        "shs": shs.contiguous(), "sh_degree": sh_degree,
    }


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    """lightning/utils.py:5-19 (getProjectionMatrix)."""
    P = torch.zeros(4, 4, dtype=torch.float32)
    P[0, 0] = 1.0 / math.tan(fovx / 2)
    P[1, 1] = 1.0 / math.tan(fovy / 2)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def look_at_c2w(azimuth: float, elevation: float, radius: float) -> torch.Tensor:
    """OpenCV camera (x right, y down, z forward) on a sphere, looking at the origin."""
    ce, se = math.cos(elevation), math.sin(elevation)
    pos = torch.tensor([radius * ce * math.cos(azimuth), radius * ce * math.sin(azimuth), radius * se],
                       dtype=torch.float64)
    fwd = -pos / pos.norm()
    up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    right = torch.linalg.cross(fwd, up)
    right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    c2w = torch.eye(4, dtype=torch.float64)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, pos
    return c2w.to(torch.float32)


def camera_from_c2w(c2w: torch.Tensor, H: int, W: int, fovx: float, fovy: float,
                    znear: float = 0.5, zfar: float = 2.5) -> Camera:
    """MiniCam's matrices (lightning/utils.py:33-48)."""
    w2c = torch.inverse(c2w)
    view = w2c.transpose(0, 1).contiguous()
    proj = projection_matrix(znear, zfar, fovx, fovy).transpose(0, 1)
    full = (view @ proj).float().contiguous()
    campos = (-c2w[:3, 3]).contiguous()   # sic: LaRa passes -c2w[:3,3] as the camera centre
    return Camera(H, W, math.tan(fovx * 0.5), math.tan(fovy * 0.5), view, full, campos, c2w)


def cameras(V: int, H: int, W: int, seed: int = 0, fov: float = 0.75, radius: float = 1.905) -> List[Camera]:
    g = torch.Generator(device="cpu").manual_seed(1000 + seed)
    elev = (torch.rand((V,), generator=g, dtype=torch.float64) * 60.0 - 30.0) * math.pi / 180.0
    cams = []
    for v in range(V):
        az = 2.0 * math.pi * v / max(V, 1)
        cams.append(camera_from_c2w(look_at_c2w(az, float(elev[v]), radius), H, W, fov, fov))
    return cams


def upstream_grads(H: int, W: int, seed: int = 0, lara_like: bool = False):
    """dL/dcolor [3,H,W] and dL/dallmap [8,H,W] (SURVEY 8d "Upstream grads")."""
    g = torch.Generator(device="cpu").manual_seed(2000 + seed)
    n = float(H * W)
    gc = torch.randn((3, H, W), generator=g, dtype=torch.float32) / n
    ga = torch.randn((8, H, W), generator=g, dtype=torch.float32) / n
    if lara_like:
        ga[5].zero_()
        ga[7].zero_()
    return gc.contiguous(), ga.contiguous()


def settings_for(cam: Camera, bg: torch.Tensor, sh_degree: int, device, settings_cls, debug: bool = False):
    """Build a GaussianRasterizationSettings (any implementation's NamedTuple) on `device`."""
    return settings_cls(
        image_height=int(cam.image_height), image_width=int(cam.image_width),
        tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg.to(device),
        scale_modifier=1.0, viewmatrix=cam.viewmatrix.to(device), projmatrix=cam.projmatrix.to(device),
        sh_degree=sh_degree, campos=cam.campos.to(device), prefiltered=False, debug=debug)


class PathCamera:
    """A camera with the attributes and ``get_rays`` of LaRa's ``tools/camera.MiniCam`` (tools/camera.py:21-56), which
    ``MeshExtractor`` and ``Renderer.render_views`` read; ``c2w`` in OpenCV axes.  ``fov`` is the horizontal field of
    view and, unless ``fovy`` is given, the vertical one too."""

    def __init__(self, c2w: torch.Tensor, H: int, W: int, fov: float, znear: float = 0.5, zfar: float = 2.5,
                 fovy: Optional[float] = None):
        fovy = fov if fovy is None else fovy
        cam = camera_from_c2w(c2w, H, W, fov, fovy, znear, zfar)
        self.image_width, self.image_height, self.FoVx, self.FoVy = W, H, fov, fovy
        self.world_view_transform = cam.viewmatrix
        self.full_proj_transform = cam.projmatrix
        self.camera_center = cam.campos
        self.c2w = c2w

    def to_device(self, device):
        self.world_view_transform = self.world_view_transform.to(device)
        self.full_proj_transform = self.full_proj_transform.to(device)
        self.camera_center = self.camera_center.to(device)

    def get_rays(self) -> torch.Tensor:
        """[1,H,W,6] origins | directions through pixel centres, as LaRa's build_rays (dataLoader/utils.py:21-34)."""
        H, W = self.image_height, self.image_width
        f = 0.5 * W / math.tan(0.5 * self.FoVx), 0.5 * H / math.tan(0.5 * self.FoVy)
        y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
        d = torch.stack(((x + 0.5 - W / 2) / f[0], (y + 0.5 - H / 2) / f[1], torch.ones_like(x)), -1)
        d = d @ self.c2w[:3, :3].to(torch.float64).T
        o = self.c2w[:3, 3].to(torch.float64).expand(H, W, 3)
        return torch.cat((o, d), -1).to(torch.float32)[None]


def mesh_path(n: int = 16, H: int = 512, W: int = 512, fov: float = 0.75, radius: float = 1.905,
              elevations=(0.0, -30.0, 30.0)):
    """LaRa's mesh camera path (tools/gen_video_path.py:117-129): n azimuths at each elevation (degrees), looking at
    the origin from ``radius``; 48 cameras by default."""
    return [PathCamera(look_at_c2w(2.0 * math.pi * a / n, math.radians(e), radius), H, W, fov)
            for e in elevations for a in range(n)]
