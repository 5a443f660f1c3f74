"""The box around a keyframe's view that DepthmapNode(prior_view_box=True) takes the volume prior from
(node.prior_view_box; DESIGN.md 4.8).  CPU only.

  * containment: on random poses and cameras (positive and negative fy, principal points off centre and outside the
    image), every sample c + k s q of every border pixel and of random interior pixels, up to max_depth + s, has its 8
    trilinear corner voxels inside the box, and so does the camera centre -- in float64;
  * tightness: the box is at most one voxel per face larger than the corner box of a dense brute-force sampling of the
    view (the extremes of each axis lie at t = 0 or t = max_depth + s, so those two suffice);
  * input checks, and the node's.
"""
import numpy as np
import pytest

from rpg_open_remode_b200 import node
from rpg_open_remode_b200.api import PinholeCamera


def _rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _case(rng):
    """(dims, s, origin, camera, width, height, T_world_ref 3x4, max_depth)"""
    w, h = int(rng.integers(2, 700)), int(rng.integers(2, 500))
    f = rng.uniform(150.0, 900.0)
    fy = f * rng.uniform(0.8, 1.2) * (1.0 if rng.random() < 0.5 else -1.0)
    cx = rng.uniform(-0.3, 1.3) * (w - 1)
    cy = rng.uniform(-0.3, 1.3) * (h - 1)
    s = float(np.float32(rng.uniform(0.005, 0.05)))
    origin = np.float32(rng.uniform(-3.0, 3.0, 3))
    T = np.concatenate([_rotation(rng), rng.uniform(-2.0, 2.0, (3, 1))], axis=1)
    T = T.astype(np.float32).astype(np.float64)   # the pose the seeds keep, in float32
    dims = tuple(int(x) for x in rng.integers(16, 256, 3))
    return dims, s, origin, PinholeCamera(f, fy, cx, cy), w, h, T, float(rng.uniform(0.5, 4.0))


def _rays(cam, px, py, R):
    """World directions of the unit rays of pixel positions (px, py)."""
    v = np.stack([(px - cam.cx) / cam.fx, (py - cam.cy) / cam.fy, np.ones_like(px)], axis=1)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)) @ R.T


def _grid(points, s, origin):
    return (points - np.asarray(origin, np.float64)) / s


def _border(w, h, step=1.0):
    xs, ys = np.arange(0.0, w - 1.0 + 1e-9, step), np.arange(0.0, h - 1.0 + 1e-9, step)
    xs, ys = np.append(xs, w - 1.0), np.append(ys, h - 1.0)
    px = np.concatenate([xs, xs, np.zeros_like(ys), np.full_like(ys, w - 1.0)])
    py = np.concatenate([np.zeros_like(xs), np.full_like(xs, h - 1.0), ys, ys])
    return px, py


@pytest.mark.parametrize("seed", range(6))
def test_containment(seed):
    rng = np.random.default_rng(1000 + seed)
    for _ in range(40):
        dims, s, origin, cam, w, h, T, max_depth = _case(rng)
        lo, m = node.prior_view_box(dims, s, origin, cam, w, h, T, max_depth)
        assert lo.dtype == np.int64 and m.dtype == np.int64 and np.all(m > 0)
        bx, by = _border(w, h)
        px = np.concatenate([bx, rng.uniform(0.0, w - 1.0, 300)])
        py = np.concatenate([by, rng.uniform(0.0, h - 1.0, 300)])
        q = _rays(cam, px, py, T[:, :3])
        t = np.arange(0, int(np.floor((max_depth + s) / s)) + 1) * s
        pts = T[:, 3][None, None] + t[:, None, None] * q[None]
        g = np.floor(_grid(pts.reshape(-1, 3), s, origin)).astype(np.int64)
        assert np.all(g >= lo) and np.all(g + 1 <= lo + m - 1), (seed, lo, m, g.min(0), g.max(0) + 1)
        # the camera centre lies inside the box of the voxel centres, so the rays start at the camera
        gc = _grid(T[:, 3][None], s, origin)[0]
        assert np.all(gc >= lo) and np.all(gc <= lo + m - 1)


@pytest.mark.parametrize("seed", range(4))
def test_tightness(seed):
    rng = np.random.default_rng(2000 + seed)
    for _ in range(15):
        dims, s, origin, cam, w, h, T, max_depth = _case(rng)
        lo, m = node.prior_view_box(dims, s, origin, cam, w, h, T, max_depth)
        bx, by = _border(w, h, 0.25)
        gx, gy = np.meshgrid(np.arange(0.0, w, 2.0), np.arange(0.0, h, 2.0))
        px, py = np.concatenate([bx, gx.ravel()]), np.concatenate([by, gy.ravel()])
        q = _rays(cam, px, py, T[:, :3])
        pts = np.concatenate([T[:, 3][None], T[:, 3][None] + (max_depth + s) * q])
        g = _grid(pts, s, origin)
        # the samples' corner box, with 0.02 voxels of slack for the directions between the brute-force samples
        lo_bf = np.floor(g.min(0) - 0.02).astype(np.int64)
        hi_bf = np.floor(g.max(0) + 0.02).astype(np.int64) + 1
        assert np.all(lo >= lo_bf - 1) and np.all(lo + m - 1 <= hi_bf + 1), (seed, lo, m, lo_bf, hi_bf)


def test_camera_looking_along_an_axis():
    """A camera looking straight down +z: the box is the pyramid's exact extent, plus the face voxel."""
    cam = PinholeCamera(100.0, 100.0, 50.0, 50.0)
    T = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1)
    lo, m = node.prior_view_box((8, 8, 8), 0.5, (0.0, 0.0, 0.0), cam, 101, 101, T, 9.5)
    # reach 10 m; the corner rays (+-0.5, +-0.5, 1) / |.| reach x = +-10 * 0.5 / sqrt(1.5); the axis ray reaches z = 10
    r = 10.0 * 0.5 / np.sqrt(1.5) / 0.5
    assert list(lo) == [int(np.floor(-r)) - 1, int(np.floor(-r)) - 1, -1]
    assert list(lo + m - 1) == [int(np.ceil(r)) + 1, int(np.ceil(r)) + 1, 21]


def test_input_checks():
    cam = PinholeCamera(300.0, 300.0, 100.0, 80.0)
    T = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1)
    ok = dict(dims=(64, 64, 64), voxel_size=0.02, origin=(0.0, 0.0, 0.0), camera=cam, width=200, height=160,
              T_world_ref=T, max_depth=3.0)
    node.prior_view_box(**ok)
    node.prior_view_box(**dict(ok, camera=(300.0, -300.0, 100.0, 80.0)))
    bad = [dict(dims=(64, 64)), dict(dims=(64, 0, 64)), dict(dims=(64, 64.5, 64)), dict(voxel_size=0.0),
           dict(voxel_size=float("nan")), dict(origin=(0.0, float("inf"), 0.0)), dict(origin=(0.0, 0.0)),
           dict(camera=PinholeCamera(0.0, 300.0, 100.0, 80.0)), dict(camera=(300.0, 0.0, 100.0, 80.0)),
           dict(camera=(300.0, 300.0, float("nan"), 80.0)), dict(width=0), dict(height=1.5),
           dict(T_world_ref=np.full((3, 4), np.nan)), dict(max_depth=0.0), dict(max_depth=float("inf"))]
    for b in bad:
        with pytest.raises(ValueError):
            node.prior_view_box(**dict(ok, **b))


def test_node_option_needs_the_volume_prior():
    with pytest.raises(ValueError):
        node.DepthmapNode(None, prior_view_box=True)
    with pytest.raises(ValueError):
        node.DepthmapNode(None, volume=object(), prior_from_volume=0.0, prior_view_box=True)


class _Recorder:
    """A stand-in depthmap that records the calls the node makes on a new keyframe."""

    def __init__(self):
        self.calls = []

    def setReferenceImage(self, img, T_curr_world, min_depth, max_depth):
        self.calls.append(("setReferenceImage", min_depth, max_depth))
        return True

    def priorFromVolume(self, volume, f, *box):
        self.calls.append(("priorFromVolume", volume, f) + box)


def test_node_without_the_view_box_makes_todays_calls():
    """prior_view_box=False (the default) asks for the window prior exactly as a node without the option does, and
    that reaches rmd_volume_prior_seeds -- not the box entry point -- with the same arguments."""
    from rpg_open_remode_b200.api import SE3, SeedMatrix
    vol = object()
    T = SE3(np.eye(3, 4).reshape(12))
    calls = []
    for kw in ({}, {"prior_view_box": False}):
        dm = _Recorder()
        nd = node.DepthmapNode(dm, volume=vol, prior_from_volume=0.0625, **kw)
        nd.denseInputCallback(np.zeros((4, 4), np.uint8), T, 0.5, 2.0)
        calls.append(dm.calls)
    assert calls[0] == calls[1] == [("setReferenceImage", 0.5, 2.0), ("priorFromVolume", vol, 0.0625, None, None)]

    class L:
        def __init__(self):
            self.calls = []

        def rmd_volume_prior_seeds(self, *a):
            self.calls.append(("window",) + a)
            return 0

        def rmd_volume_prior_seeds_box(self, *a):
            self.calls.append(("box",) + a)
            return 0

    class V:
        handle = "volume"

    g = object.__new__(SeedMatrix)
    g._L, g._h = L(), "seeds"
    g.priorFromVolume(V(), 0.0625, None, None)
    g.priorFromVolume(V(), 0.0625)
    assert g._L.calls == [("window", "volume", "seeds", 0.0625)] * 2
    g._h = None   # nothing to destroy
