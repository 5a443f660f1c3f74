"""The ESDF box's checker (tests/volume_esdf_box_oracle.py) and the node's box policy pinned without a GPU.

  * box_records against a voxel-by-voxel lookup by the definition: ragged boxes with negative corners, boxes disjoint
    from the window, boxes inside it, one-voxel-thick boxes, stale stored copies of window voxels, and a store walk with
    evictions and restores (where it also equals StoreModel.dense_map() cut to the box);
  * the box origin against a float32 restatement of rmd_volume_shift's origin rule, exact for any int64 corner;
  * DepthmapNode's esdf_camera_margin box on bench.py's c2 poses: it holds the window and every keyframe camera's cube,
    within the size limit, while the camera itself lies outside the following window.
"""
from fractions import Fraction

import numpy as np

import volume_esdf_box_oracle as veb
import volume_esdf_oracle as veo
from test_volume_store_oracle import _model, paint
from volume_store_oracle import B

u32 = np.uint32


def _same(a, b):
    return all(np.array_equal(x.view(u32), y.view(u32)) for x, y in zip(a, b))


def _boxes(n):
    """Ragged (lo, dims) boxes in window indices around a window of dims n."""
    n = np.asarray(n)
    return [((0, 0, 0), tuple(n)), ((-5, -3, -11), tuple(n + (9, 4, 13))), ((-13, 2, -1), (7, 5, 30)),
            ((3, 2, 1), (4, 3, 2)), (tuple(n + 2), (9, 6, 5)), ((-20, -9, -17), (6, 5, 4)),
            ((1, -4, 2), (1, 17, 1)), ((-9, 0, -9), (n[0] + 18, n[1], 1))]


def test_box_records_equal_brute_force_with_stale_bricks():
    rng = np.random.default_rng(0xB0C5)
    n = (13, 10, 11)
    D = np.array([-21, 5, -3], np.int64)
    t = rng.uniform(-1, 1, n[::-1]).astype(np.float32)
    w = rng.integers(0, 3, n[::-1]).astype(np.float32)
    bricks = {}
    for _ in range(40):   # around the window, some overlapping it (stale copies with other values)
        c = tuple(int(x) for x in rng.integers((D - 24) // B, (D + np.array(n) + 24) // B + 1))
        bricks[c] = (rng.uniform(-1, 1, (B, B, B)).astype(np.float32),
                     rng.integers(1, 4, (B, B, B)).astype(np.float32))
    for lo, m in _boxes(n):
        lo_u = D + np.asarray(lo)
        got = veb.box_records(lo_u, m, D, t, w, bricks)
        assert got[0].shape == tuple(m[::-1])
        assert _same(got, veb.box_records_brute(lo_u, m, D, t, w, bricks)), (lo, m)
        assert _same(veb.box_records(lo_u, m, D, t, w), veb.box_records_brute(lo_u, m, D, t, w)), (lo, m)
    # the window's own box is the window
    assert _same(veb.box_records(D, n, D, t, w, bricks), (t, w))


def test_store_walk_box_records():
    """A walk with shifts that evict and restore: box_records of the model equals the brute-force lookup and the
    model's dense map cut to the box (zeros outside it)."""
    rng = np.random.default_rng(0xB0C6)
    dims = (19, 14, 23)
    m = _model(dims)
    seen_restore = False
    for d in [(7, -3, 5), (-7, 3, -5), (25, 0, 0), (-25, 0, 0), (-4, 9, -12), (3, -2, 8)]:
        paint(m, rng, 0.5, intensity=False)
        m.shift(d)
        seen_restore = seen_restore or m.restored > 0
        bricks = veb.model_bricks(m)
        lo_d, dt, dw = m.dense_map()
        big = ((-40, -30, -35), (dims[0] + 80, dims[1] + 60, dims[2] + 70))
        for lo, mm in _boxes(dims) + [big]:
            lo_u = m.D + np.asarray(lo)
            got = veb.box_records(lo_u, mm, m.D, m.tsdf, m.weight, bricks)
            if (lo, mm) != big:
                assert _same(got, veb.box_records_brute(lo_u, mm, m.D, m.tsdf, m.weight, bricks)), (d, lo, mm)
            # the dense map, cut to the box and padded with zeros
            want = veb.box_records(lo_u, mm, lo_d, dt, dw)
            assert _same(got, want), (d, lo, mm)
            # downloadStore()'s layout (window voxels zeroed) gives the same records
            coords, rec = m.download_store()
            got2 = veb.box_records(lo_u, mm, m.D, m.tsdf, m.weight,
                                   veb.downloaded_bricks(coords, rec[:, 0], rec[:, 1]))
            assert _same(got, got2), (d, lo, mm)
    assert seen_restore and len(m.bricks) > 0
    # a box around everything sees stored obstacles outside the window: closer than the window alone says
    lo = (-40, -30, -35)
    mm = (dims[0] + 80, dims[1] + 60, dims[2] + 70)
    bt, bw = veb.box_records(m.D + np.asarray(lo), mm, m.D, m.tsdf, m.weight, veb.model_bricks(m))
    assert (bw > 0).sum() > (m.weight > 0).sum()
    d_box, _ = veo.esdf(bt, bw, m.s)
    d_win, _ = veo.esdf(m.tsdf, m.weight, m.s)
    inner = d_box[-lo[2]:-lo[2] + dims[2], -lo[1]:-lo[1] + dims[1], -lo[0]:-lo[0] + dims[0]]
    assert np.all(np.abs(inner) <= np.abs(d_win)) and np.any(np.abs(inner) < np.abs(d_win))


def _f32_exact(x: Fraction) -> Fraction:
    """x rounded to the nearest float32, ties to even (normal range)."""
    if x == 0:
        return Fraction(0)
    sign = -1 if x < 0 else 1
    a = abs(x)
    e = 0
    while a >= 2:
        a /= 2
        e += 1
    while a < 1:
        a *= 2
        e -= 1
    q = a * 2 ** 23
    f = int(q)
    r = q - f
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and f % 2):
        f += 1
    return sign * Fraction(f) * Fraction(2) ** (e - 23)


def test_box_origin_rule():
    """o0 + (float)(D + lo) * s, each operation rounded to float32, restated with exact rationals."""
    rng = np.random.default_rng(0xB0C7)
    corners = [0, 1, -1, 7, -8, 123456, -987654, 2 ** 24 + 1, -(2 ** 31) - 3, 2 ** 40 + 12345,
               2 ** 62 + 2 ** 39 + 1, -(2 ** 63), 2 ** 63 - 1]
    corners += [int(x) for x in rng.integers(-2 ** 62, 2 ** 62, 40)]
    for s in (np.float32(0.0166), np.float32(0.05), np.float32(1.0 / 3.0)):
        for q in range(0, len(corners), 3):
            lo_u = np.array((corners + corners[:2])[q:q + 3], np.int64)
            o0 = rng.uniform(-50, 50, 3).astype(np.float32)
            got = veb.box_origin(o0, lo_u, s)
            for a in range(3):
                step = _f32_exact(_f32_exact(Fraction(int(lo_u[a]))) * Fraction(float(s)))
                want = _f32_exact(Fraction(float(o0[a])) + step)
                assert Fraction(float(got[a])) == want, (lo_u[a], o0[a], s)


def test_node_camera_box_on_c2_poses():
    """followVolume's recentring replayed on bench.py's c2 sequence, each frame taken as a finished keyframe: the box
    of esdf_camera_margin = 32 holds the 128^3 window and the cube around the camera's voxel, within the ESDF's size
    limit, and the camera lies outside the window (the gap the box closes)."""
    from rpg_open_remode_b200 import multi_gpu, node, synth
    from test_volume import _grid
    W, H, N, r = 640, 480, 200, 32
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))
    s, _, _ = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    dims = np.array((128, 128, 128), np.int64)
    o0 = np.zeros(3, np.float32)
    D = np.zeros(3, np.int64)
    origin = o0.copy()
    outside = 0
    for k in range(0, N, 5):
        T = seq.frame(k, want_depth=False).T_world_cam.reshape(3, 4).astype(np.float32).astype(np.float64)
        centre = T[:, 3] + 0.5 * (dmin + dmax) * T[:, 2]   # followVolume's shift
        off = (centre - origin.astype(np.float64)) / float(s) - 0.5 * (dims - 1.0)
        d = np.where(np.abs(off) > dims / 8.0, np.round(off), 0.0).astype(np.int64)
        D = D + d
        origin = veb.box_origin(o0, D, s)
        lo, m = node.esdf_camera_box(tuple(dims), float(s), origin, T[:, 3], r)
        c = np.round((T[:, 3] - origin.astype(np.float64)) / float(s)).astype(np.int64)
        assert np.all(lo <= 0) and np.all(lo + m >= dims), k
        assert np.all(lo <= c - r) and np.all(c + r < lo + m), k
        assert np.all(m > 0) and ((m - 1) ** 2).sum() < 2 ** 24, k
        assert lo.dtype == np.int64 and m.dtype == np.int64
        outside += bool(np.any(c < 0) or np.any(c >= dims))
    assert outside == len(range(0, N, 5))
    # the window alone when the camera lies in it
    lo, m = node.esdf_camera_box((128, 128, 128), 0.1, (0, 0, 0), (6.4, 6.4, 6.4), 8)
    assert list(lo) == [0, 0, 0] and list(m) == [128, 128, 128]
