"""Device mesh filter (filter_mesh_device, DESIGN §3.15) against the host filter (lara_b200.mesh.filter_mesh) and the
float64 restatement (oracle.mesh64.filter_mesh), array for array: random fields with many clusters, ties, crops at the
float64 bound, NaN vertices, non-manifold and degenerate triangles, a large fan, invalid indices; LaRa's mesh path;
bit-reproducibility; a non-default stream; and MeshExtractor's OBJ against one written from the host filter."""
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_mesh import _fuse, _sphere_surfels, lara_path  # noqa: F401  (lara_path is a fixture)

pytestmark = pytest.mark.gpu


def _f32(v, t, c):
    return (np.ascontiguousarray(v, np.float32), np.ascontiguousarray(t, np.int32).reshape(-1, 3),
            np.ascontiguousarray(c, np.float32))


def _dev(mesh, dev):
    return tuple(torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in mesh)


def _clusters(mesh_dev, aabb=None, keep=10):
    """The four totals of srf_mesh_filter_count: kept Nv, kept Nt, clusters after the crop, invalid triangles."""
    from lara_b200 import _lib
    v, t, _ = mesh_dev
    Nv, Nt = int(v.shape[0]), int(t.shape[0])
    box = None if aabb is None else (ctypes.c_double * 6)(*np.asarray(aabb, np.float64).reshape(6).tolist())
    ws = torch.empty(_lib.mesh_filter_workspace_bytes(_lib.load(), Nv, Nt), dtype=torch.uint8, device=v.device)
    totals = torch.empty(4, dtype=torch.int32, device=v.device)
    _lib.launch("srf_mesh_filter_count", v.device, Nv, Nt, v.data_ptr(), t.data_ptr(), box, keep, ws.data_ptr(),
                totals.data_ptr())
    return [int(x) for x in totals.cpu()]


def _check(mesh, dev, aabb=None, keep=10, oracle=True):
    """filter_mesh_device equals filter_mesh (and the restatement) on the float32 mesh; returns the device result on
    the host and the totals."""
    from lara_b200 import mesh as MS
    from oracle import mesh64
    md = _dev(mesh, dev)
    got = [x.cpu().numpy() for x in MS.filter_mesh_device(md, aabb, keep)]
    assert got[0].dtype == np.float32 and got[1].dtype == np.int32 and got[2].dtype == np.float32
    refs = [MS.filter_mesh(mesh, aabb, keep)]
    if oracle:
        refs.append(mesh64.filter_mesh(*mesh, aabb, keep))
    for ref in refs:
        for x, y in zip(got, ref):
            assert np.asarray(y).reshape(-1, 3).shape == x.shape
            assert np.array_equal(x, np.asarray(y).reshape(-1, 3), equal_nan=True)
    totals = _clusters(md, aabb, keep)
    assert totals[:2] == [len(got[0]), len(got[1])] and totals[3] == 0
    return got, totals


def _field(n, p, seed):
    from oracle import mesh64
    rng = np.random.default_rng(seed)
    f = np.ones((n, n, n))
    f[1:-1, 1:-1, 1:-1] = np.where(rng.random((n - 2,) * 3) < p, -1.0, 1.0)
    return _f32(*mesh64.extract((0, 0, 0), (n, n, n), 0.05, f, np.ones_like(f), rng.random((3, n, n, n)) * 255))


def test_random_field_with_ties(cuda_device):
    """The many-cluster field of tests/test_mesh.py::test_filter_matches_the_restatement."""
    from oracle import mesh64
    rng = np.random.default_rng(5)
    f = np.ones((26, 26, 26))
    f[1:-1, 1:-1, 1:-1] = np.where(rng.random((24, 24, 24)) < 0.12, -1.0, 1.0)
    mesh = _f32(*mesh64.extract((0, 0, 0), (26, 26, 26), 0.05, f, np.ones_like(f), rng.random((3, 26, 26, 26)) * 255))
    for aabb in (None, np.array([[0.2, 0.1, 0.0], [1.0, 1.2, 0.9]])):
        for keep in (1, 10, 40):
            got, totals = _check(mesh, cuda_device, aabb, keep)
            assert len(got[1]) > 0 and totals[2] > 40


def test_large_random_field(cuda_device):
    mesh = _field(64, 0.12, 7)
    assert len(mesh[1]) > 100_000
    for keep in (10, 1000):
        got, totals = _check(mesh, cuda_device, None, keep)
        print(f"[mesh filter] field 64^3: Nt {len(mesh[1])}, clusters {totals[2]}, keep {keep}: Nt {len(got[1])}")
        assert totals[2] > 1000


def _octahedron(offset):
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64) * 0.1 + offset
    t = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])
    return v, t


def _concat(parts):
    vs, ts, n = [], [], 0
    for v, t in parts:
        vs.append(v)
        ts.append(np.asarray(t) + n)
        n += len(v)
    v = np.concatenate(vs)
    c = np.random.default_rng(len(v)).random(v.shape)
    return _f32(v, np.concatenate(ts), c)


def test_twelve_equal_clusters_are_all_kept(cuda_device):
    """Twelve disjoint octahedra and three lone triangles: keep = 10 cuts at 8 triangles, so all twelve stay."""
    parts = [_octahedron(np.array([i, 0, 0], np.float64)) for i in range(12)]
    parts += [(np.array([[0, 5, 0], [0.1, 5, 0], [0, 5.1, 0]]) + i, [[0, 1, 2]]) for i in range(3)]
    got, totals = _check(_concat(parts), cuda_device, None, 10)
    assert totals[2] == 15 and len(got[1]) == 96 and len(got[0]) == 72


def test_fewer_clusters_than_keep(cuda_device):
    parts = [_octahedron(np.array([i, 0, 0], np.float64)) for i in range(3)] + [(np.eye(3) + 9, [[0, 1, 2]])]
    got, totals = _check(_concat(parts), cuda_device, None, 10)
    assert totals[2] == 4 and len(got[1]) == 25


def test_empty_and_fully_cropped(cuda_device):
    v = np.random.default_rng(0).random((5, 3))
    got, totals = _check(_f32(v, np.zeros((0, 3)), v), cuda_device, None, 10)
    assert totals == [0, 0, 0, 0] and all(len(x) == 0 for x in got)
    got, totals = _check(_f32(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3))), cuda_device, np.zeros((2, 3)), 1)
    assert all(len(x) == 0 for x in got)
    mesh = _concat([_octahedron(np.zeros(3))])
    got, totals = _check(mesh, cuda_device, np.array([[2, 2, 2], [3, 3, 3]]), 10)
    assert totals[2] == 0 and all(len(x) == 0 for x in got)


def test_crop_compares_against_the_float64_bound(cuda_device):
    """Bound x <= 0.1 (float64).  float32(0.1) lies just above it, so a triangle using it is cropped, though a bound
    rounded to float32 would keep it; its float32 predecessor is inside.  A bound equal to a float32 value keeps a
    vertex exactly on it and drops the next float32 value."""
    x = np.float32(0.1)
    below, above = np.nextafter(x, np.float32(0)), np.nextafter(x, np.float32(1))
    assert np.float64(x) > 0.1 and np.float64(below) < 0.1
    base = np.array([[0, 0, 0], [0, 0.05, 0], [0, 0, 0.05]])
    parts = [(np.vstack([base + [0, 3 * i, 0], [[xv, 3 * i, 0]]]), [[0, 1, 3], [0, 2, 3]])
             for i, xv in enumerate((x, below, above))]
    mesh = _concat(parts)
    assert mesh[0][3, 0] == x and mesh[0][7, 0] == below and mesh[0][11, 0] == above
    lo = np.full(3, -1.0)
    got, _ = _check(mesh, cuda_device, np.array([lo, [0.1, 10, 10]]), 10)
    assert {float(v) for v in got[0][:, 0]} == {0.0, float(below)}
    got, _ = _check(mesh, cuda_device, np.array([lo, [float(x), 10, 10]]), 10)
    assert float(x) in {float(v) for v in got[0][:, 0]} and float(above) not in {float(v) for v in got[0][:, 0]}


def test_nan_vertex(cuda_device):
    mesh = _concat([_octahedron(np.zeros(3)), _octahedron(np.ones(3))])
    mesh[0][2, 1] = np.nan
    got, totals = _check(mesh, cuda_device, None, 10)
    assert totals[2] == 2 and len(got[1]) == 16 and np.isnan(got[0]).sum() == 1
    got, totals = _check(mesh, cuda_device, np.array([[-1, -1, -1], [2, 2, 2]]), 10)
    assert len(got[1]) == 12 and not np.isnan(got[0]).any()


def test_edge_shared_by_three_triangles_and_a_shared_vertex(cuda_device):
    v = np.random.default_rng(3).random((9, 3))
    book = [[0, 1, 2], [1, 0, 3], [0, 1, 4]]            # edge {0, 1} in three triangles: one cluster
    bowtie = [[5, 6, 7], [5, 8, 4]]                      # only vertex 5 shared, then only vertex 4 with the book
    got, totals = _check(_f32(v, book + bowtie, v), cuda_device, None, 10)
    assert totals[2] == 3 and len(got[1]) == 5
    got, totals = _check(_f32(v, book + bowtie, v), cuda_device, None, 1)
    assert len(got[1]) == 3


def test_degenerate_triangles(cuda_device):
    """(a, a, b) has the edges {a, a} and {a, b}; (a, a, a) only {a, a}."""
    v = np.random.default_rng(4).random((8, 3))
    t = [[0, 0, 1], [1, 0, 2], [3, 3, 3], [3, 3, 4], [5, 6, 7], [7, 7, 7]]
    got, totals = _check(_f32(v, t, v), cuda_device, None, 10)
    assert totals[2] == 4
    got, totals = _check(_f32(v, t, v), cuda_device, None, 2)
    assert len(got[1]) == 4


def test_fan_of_fifty_thousand_triangles(cuda_device):
    n = 50_000
    a = np.linspace(0, 2 * np.pi, n + 1)[:-1]
    v = np.concatenate([[[0, 0, 0]], np.stack((np.cos(a), np.sin(a), np.zeros(n)), -1)])
    i = np.arange(n)
    t = np.stack((np.zeros(n, np.int64), 1 + i, 1 + (i + 1) % n), -1)
    t[n // 2] = [0, n + 1, n + 2]                        # one fan triangle apart: not edge-connected to the rest
    v = np.concatenate([v, [[5, 5, 5], [6, 5, 5]]])
    got, totals = _check(_f32(v, t, v), cuda_device, None, 1)
    assert totals[2] == 2 and len(got[1]) == n - 1


def test_unreferenced_vertices_are_dropped(cuda_device):
    v, t = _octahedron(np.zeros(3))
    v = np.concatenate([np.full((3, 3), 7.0), v[:3], np.full((2, 3), 8.0), v[3:], np.full((4, 3), 9.0)])
    t = np.where(t < 3, t + 3, t + 5)
    got, _ = _check(_f32(v, t, v), cuda_device, None, 10)
    assert len(got[0]) == 6 and not (got[0] > 5).any()


def test_out_of_range_index_raises(cuda_device):
    from lara_b200 import mesh as MS
    v, t, c = _concat([_octahedron(np.zeros(3))])
    for bad in (-1, len(v), 2**31 - 1, -2**31):
        tb = t.copy()
        tb[3, 1] = bad
        md = _dev((v, tb, c), cuda_device)
        before = [x.clone() for x in md]
        with pytest.raises(RuntimeError, match="outside"):
            MS.filter_mesh_device(md, None, 10)
        assert _clusters(md)[3] == 1
        assert all(torch.equal(x, y) for x, y in zip(before, md))


@pytest.fixture(scope="module")
def lara_mesh(lara_path):  # noqa: F811
    from lara_b200 import mesh as MS
    return MS.extract_triangle_mesh(_fuse(lara_path))


def test_laras_path_matches_the_host_filter(lara_mesh, lara_path):  # noqa: F811
    from lara_b200 import mesh as MS
    assert len(lara_mesh[1]) > 1_000_000
    host = [x.cpu().numpy() for x in lara_mesh]
    got, totals = _check(host, lara_mesh[0].device, lara_path["aabb"], 10, oracle=False)
    print(f"[mesh filter] lara path: Nv {len(host[0])}, Nt {len(host[1])}, clusters {totals[2]}, "
          f"kept Nv {len(got[0])}, Nt {len(got[1])}")
    assert 0 < len(got[1]) < len(host[1])
    # called on the device tensors directly, the same
    out = [x.cpu().numpy() for x in MS.filter_mesh_device(lara_mesh, lara_path["aabb"])]
    assert all(np.array_equal(x, y) for x, y in zip(out, got))


def test_bits_repeat_and_deterministic_and_on_a_side_stream(lara_mesh, lara_path):  # noqa: F811
    from lara_b200 import mesh as MS
    field = _dev(_field(64, 0.12, 11), lara_mesh[0].device)

    def run():
        return [list(MS.filter_mesh_device(lara_mesh, lara_path["aabb"])), list(MS.filter_mesh_device(field, None, 10))]
    a, b = run(), run()
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = run()
    finally:
        torch.use_deterministic_algorithms(was)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d = run()
    torch.cuda.current_stream().wait_stream(s)
    for other in (b, c, d):
        for x, y in zip(a, other):
            assert all(torch.equal(p, q) for p, q in zip(x, y))


def test_extract_writes_the_host_filters_obj(cuda_device, tmp_path, monkeypatch):
    """MeshExtractor.extract on the 200 k-surfel sphere of test_gpu_mesh.py: its OBJ is byte for byte the one written
    from the host filter's output on the same unfiltered mesh."""
    from lara_b200 import mesh as MS
    from lara_b200 import scene as S
    from lara_b200.renderer import Renderer
    seen = {}
    device_filter = MS.filter_mesh_device

    def spy(mesh, aabb=None, keep=10):
        seen["mesh"], seen["aabb"] = [x.clone() for x in mesh], aabb
        return device_filter(mesh, aabb, keep)
    monkeypatch.setattr(MS, "filter_mesh_device", spy)
    ex = MS.MeshExtractor(_sphere_surfels(200_000, 0.3, cuda_device), Renderer(sh_degree=0),
                          aabb=[-0.5, -0.5, -0.5, 0.5, 0.5, 0.5])
    path, ref_path = tmp_path / "device.obj", tmp_path / "host.obj"
    v, t, c = ex.extract(str(path), S.mesh_path(16, 512, 512, 0.75))
    assert not v.is_cuda and t.dtype == torch.int32 and len(t) > 10000
    hv, ht, hc = MS.filter_mesh(seen["mesh"], seen["aabb"])
    MS.write_obj(str(ref_path), hv, ht, hc)
    assert path.read_bytes() == ref_path.read_bytes()
    assert np.array_equal(v.numpy(), hv) and np.array_equal(t.numpy(), ht) and np.array_equal(c.numpy(), hc)
