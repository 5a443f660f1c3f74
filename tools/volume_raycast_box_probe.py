"""Device time of the box raycast and what the view-box prior gives on c2 (DESIGN.md 4.8, 6): rmd_volume_raycast_box
and rmd_volume_prior_seeds_box, i.e. the gather of the box's records (the ESDF box's kernel) and the existing raycast.

  * volume_probe.py's scene (bench.py's c2 sequence, VGA, eight keyframes' ground-truth depth fused) in a 256^3 and a
    512^3 window with the store, shifted out and back by n / 8 along x so that bricks are stored.  From frame 100's
    pose, the box raycast over that frame's view box (node.prior_view_box) against the window raycast: the median of
    REPEATS calls after WARMUP, CUDA events on the volume's stream; the split into gather and raycast kernels from a
    torch.profiler run of its own.
  * the node on c2 (a following 128^3 window with the store, the volume prior f = 1/16, 200 frames), with and without
    prior_view_box: per keyframe the view box's dims and scratch bytes (8 B per box voxel and 4 B per brick of the box
    for the brick table), the interior seeds given a prior by the box prior and by the window prior from the same
    volume and pose (the window raycast's hits within the depth range: the prior's rule), and the converged
    percentage at publish of both runs.

Prints one JSON line with the GPU's name and power limit, read before and after.  GPU box only."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import _native, multi_gpu, node, synth  # noqa: E402
from volume_esdf_probe import gpu_info  # noqa: E402
from volume_probe import REPEATS, W, H, scene_box, timed  # noqa: E402

GRIDS = (256, 512)
F_PRIOR = 1.0 / 16.0
KERNELS = (("gather", "volume_esdf_gather_kernel"), ("raycast", "volume_raycast_kernel"))


def box_bytes(lo, dims, offset):
    """Scratch of a box without intensity: 8 B per voxel and 4 B per brick of the box."""
    lo_u = np.asarray(offset, np.int64) + np.asarray(lo, np.int64)
    nb = np.floor_divide(lo_u + np.asarray(dims) - 1, 8) - np.floor_divide(lo_u, 8) + 1
    return int(8 * np.prod(np.asarray(dims, np.int64)) + 4 * np.prod(nb))


def kernel_split(torch, v, stream, fn):
    """Mean device time (ms) of each kernel of fn over REPEATS calls, from the profiler's kernel records."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(stream):
            for _ in range(REPEATS):
                fn()
        v.sync()
    ms = {tag: 0.0 for tag, _ in KERNELS}
    for e in prof.events():
        for tag, name in KERNELS:
            if name in e.name:
                ms[tag] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return {k: round(t / REPEATS, 3) for k, t in ms.items()}


def box_case(torch, stream, seq, frames, cam, lo, hi, n):
    L = _native.lib()
    s = float(np.float32((hi - lo).max() / (n - 1 - 16)))
    v = rmd.TsdfVolume((n, n, n), s, lo - 8 * s, 4 * s, 64.0, device=0, store=True)
    v.setStream(stream.cuda_stream)
    for fr in frames:
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
    d = n // 8
    v.shift((d, 0, 0))
    v.shift((-d, 0, 0))
    v.sync()
    fr = seq.frame(100)
    dmax = float(seq.frame(0).depth.max())
    T_wc = fr.T_world_cam.astype(np.float64).reshape(3, 4)
    blo, bdims = node.prior_view_box(v.dims, v.voxel_size, v.origin, cam, W, H, T_wc, dmax)
    lo64, m32 = blo.astype(np.int64), bdims.astype(np.int32)
    img = rmd.DeviceImage(W, H, "float32")
    T = np.ascontiguousarray(np.asarray(fr.T_cam_world, np.float32).reshape(12))

    def window():
        assert L.rmd_volume_raycast(v.handle, W, H, cam.fx, cam.fy, cam.cx, cam.cy, T.ctypes.data, img.data,
                                    img.pitch) == 0

    def box():
        assert L.rmd_volume_raycast_box(v.handle, lo64.ctypes.data, m32.ctypes.data, W, H, cam.fx, cam.fy, cam.cx,
                                        cam.cy, T.ctypes.data, img.data, img.pitch, None, 0, None, 0) == 0

    t_win, _ = timed(stream, torch, window)
    hits_win = int((img.getDevData() > 0).sum())
    t_box, _ = timed(stream, torch, box)
    hits_box = int((img.getDevData() > 0).sum())
    split = kernel_split(torch, v, stream, box)
    out = {"window": f"{n}^3", "view_box_dims": [int(x) for x in bdims], "view_box_lo": [int(x) for x in blo],
           "scratch_MiB": round(box_bytes(blo, bdims, v.offset) / 2 ** 20, 1),
           "stored_bricks": int(v.storeInfo()[0]), "window_raycast_ms_median": round(t_win, 3),
           "box_raycast_ms_median": round(t_box, 3), "box_kernels_ms": split,
           "hit_pixels_window": hits_win, "hit_pixels_box": hits_box}
    del v
    torch.cuda.empty_cache()
    return out


def node_case(torch, stream, view_box):
    from test_volume import _grid
    N = 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))
    s, _, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fx, fy, cx, cy = seq.camera
    cam = rmd.PinholeCamera(fx, fy, cx, cy)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    vol = rmd.TsdfVolume((128, 128, 128), s, (0.0, 0.0, 0.0), tau, 64.0, device=0, store=True)
    vol.setStream(stream.cuda_stream)
    dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
    rows, conv = [], []
    prior, set_ref, pose = dm.priorFromVolume, dm.setReferenceImage, []

    def set_reference(img, T_curr_world, mn, mx):
        pose.append(T_curr_world)
        return set_ref(img, T_curr_world, mn, mx)

    def prior_from_volume(volume, f, lo=None, dims=None):
        prior(volume, f, lo, dims)
        g = dm.seeds_
        interior = g.downloadConvergence() != rmd.ConvergenceStates.BORDER
        s2 = g.downloadSigmaSq()
        given = int((interior & (s2 != s2[interior].max())).sum())
        d = volume.raycast(cam, pose[-1], W, H)
        window = int((interior & (d > 0) & (d >= np.float32(dmin)) & (d <= np.float32(dmax))).sum())
        row = {"prior_seeds": given, "window_prior_seeds": window}
        if lo is not None:
            row.update(view_box_dims=[int(x) for x in dims], scratch_MiB=round(box_bytes(lo, dims, volume.offset)
                                                                             / 2 ** 20, 1))
        rows.append(row)

    def publisher(kind, d):
        if kind == "depthmap_and_pointcloud":
            conv.append(round(100.0 * float((d.getConvergenceMap() == rmd.ConvergenceStates.CONVERGED).mean()), 2))

    dm.setReferenceImage, dm.priorFromVolume = set_reference, prior_from_volume
    nd = node.DepthmapNode(dm, publisher=publisher, volume=vol, follow_volume=True, prior_from_volume=F_PRIOR,
                           prior_view_box=view_box)
    for k in range(N):
        fr = seq.frame(k, want_depth=False)
        nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
    vol.sync()
    return {"keyframes": rows, "converged_percent_at_publish": conv,
            "prior_seeds_total": sum(r["prior_seeds"] for r in rows),
            "window_prior_seeds_total": sum(r["window_prior_seeds"] for r in rows)}


def main():
    import torch
    if rmd.device_count() < 1 or not torch.cuda.is_available():
        raise RuntimeError("volume_raycast_box_probe.py needs an H100")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    torch.cuda.set_device(0)
    result = {"gpu": gpu_info()}
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    frames = [seq.frame(k) for k in range(0, 200, 25)]
    lo, hi = scene_box(seq, frames)
    cam = rmd.PinholeCamera(*seq.camera)
    stream = torch.cuda.Stream()
    for n in GRIDS:
        result[f"{n}^3"] = box_case(torch, stream, seq, frames, cam, lo, hi, n)
    result["node_c2_view_box"] = node_case(torch, stream, True)
    result["node_c2_window"] = node_case(torch, stream, False)
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
