"""Device time of the TSDF volume's ESDF over a box of the map (DESIGN.md 4.8, 6): rmd_volume_esdf_box, i.e. the gather
of the box's records from the window and the brick store, then the three passes.

  * volume_probe.py's scene (bench.py's c2 sequence, VGA, eight keyframes' ground-truth depth fused) in a 256^3 window
    with the store, shifted out and back by n / 8 along x so that bricks are stored, then the ESDF of a 384^3 box around
    it; the same with a 512^3 window and a 768^3 box.  Compute = the median of REPEATS runs after WARMUP, CUDA events on
    the volume's stream; the split into gather, z, y and x passes from a torch.profiler run of its own.  The window's
    own compute (rmd_volume_esdf) is timed alongside.
  * the node's esdf_camera_margin=32 on c2 (a following 128^3 window with the store, 200 frames): at each finished
    keyframe, the box compute the node ran and the window-only compute, each timed with CUDA events (median of REPEATS
    after WARMUP, the box last so that the published snapshot stays the node's).

Bytes of the gather: one 8 B record write per box voxel, one 8 B read per window voxel, and at most 8 B per voxel of
the stored bricks (a voxel outside the window and the stored bricks reads only its table entry, 4 B per brick of the
box, which the caches hold).  Prints one JSON line with the GPU's name and power limit.  GPU box only."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import multi_gpu, node, synth  # noqa: E402
from volume_esdf_probe import gpu_info  # noqa: E402
from volume_probe import HBM_BYTES_PER_S, REPEATS, W, H, scene_box, timed  # noqa: E402

CASES = ((256, 384), (512, 768))
VOXELS_PER_BRICK = 512
KERNELS = (("gather", "volume_esdf_gather_kernel"), ("z", "volume_esdf_kernel<0>"), ("y", "volume_esdf_kernel<1>"),
           ("x", "volume_esdf_kernel<2>"))


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


def box_case(torch, stream, seq, frames, cam, lo, hi, n, m):
    s = float(np.float32((hi - lo).max() / (n - 1 - 16)))
    v = rmd.TsdfVolume((n, n, n), s, lo - 8 * s, 4 * s, 64.0, device=0, store=True)
    v.setStream(stream.cuda_stream)
    for fr in frames:
        v.integrateDepth(fr.depth, cam, fr.T_cam_world)
    # out and back along x by n / 8: the bricks the window leaves are stored, then restored (and stay stored)
    d = n // 8
    v.shift((d, 0, 0))
    v.shift((-d, 0, 0))
    v.sync()
    bricks = v.storeInfo()[0]
    b = (m - n) // 2
    box = ((-b, -b, -b), (m, m, m))
    med, _ = timed(stream, torch, lambda: v.computeEsdf(*box))
    split = kernel_split(torch, v, stream, lambda: v.computeEsdf(*box))
    win, _ = timed(stream, torch, v.computeEsdf)
    vox = m ** 3
    g = split["gather"]
    gather_bytes = 8 * vox + 8 * n ** 3 + 8 * VOXELS_PER_BRICK * bricks   # writes, window reads, stored bricks at most
    out = {"window": f"{n}^3", "box": f"{m}^3", "stored_bricks": int(bricks), "box_compute_ms_median": round(med, 3),
           "kernels_ms": split, "window_compute_ms_median": round(win, 3),
           "gather_bytes": int(gather_bytes),
           "gather_GB_per_s": round(gather_bytes / (g * 1e-3) / 1e9, 1) if g > 0 else None,
           "gather_share_of_3.35TB/s": round(gather_bytes / (g * 1e-3) / HBM_BYTES_PER_S, 3) if g > 0 else None,
           "box_esdf_GiB": round(24 * vox / 2 ** 30, 2)}
    del v
    torch.cuda.empty_cache()
    return out


def node_case(torch, stream):
    from test_volume import _grid
    N = 200
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))
    s, _, tau = _grid(seq, [seq.frame(k) for k in range(0, N, 25)] + [seq.frame(N - 1)], 512)
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    vol = rmd.TsdfVolume((128, 128, 128), s, (0.0, 0.0, 0.0), tau, 64.0, device=0, store=True)
    vol.setStream(stream.cuda_stream)
    dm = rmd.Depthmap(W, H, fx, cx, fy, cy, device=0)
    rows = []

    def publisher(kind, v):
        if kind != "volume_esdf":
            return
        box = nd.esdfCameraBox()
        t_win, _ = timed(stream, torch, v.computeEsdf)
        t_box, _ = timed(stream, torch, lambda: v.computeEsdf(*box))
        rows.append((t_box, t_win, [int(x) for x in box[1]]))

    nd = node.DepthmapNode(dm, publisher=publisher, volume=vol, follow_volume=True, esdf=True, esdf_camera_margin=32)
    for k in range(N):
        fr = seq.frame(k, want_depth=False)
        nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
    vol.sync()
    tb, tw = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
    return {"keyframes": len(rows), "box_ms_median": round(float(np.median(tb)), 3),
            "box_ms_max": round(float(tb.max()), 3), "window_ms_median": round(float(np.median(tw)), 3),
            "extra_ms_per_keyframe_median": round(float(np.median(tb - tw)), 3),
            "box_dims": [r[2] for r in rows], "stored_bricks_at_end": int(vol.storeInfo()[0])}


def main():
    import torch
    if rmd.device_count() < 1 or not torch.cuda.is_available():
        raise RuntimeError("volume_esdf_box_probe.py needs an H100")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    torch.cuda.set_device(0)
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    frames = [seq.frame(k) for k in range(0, 200, 25)]
    lo, hi = scene_box(seq, frames)
    cam = rmd.PinholeCamera(*seq.camera)
    stream = torch.cuda.Stream()
    result = {"gpu": gpu_info()}
    for n, m in CASES:
        result[f"{n}^3 in {m}^3"] = box_case(torch, stream, seq, frames, cam, lo, hi, n, m)
    result["node_c2_margin_32"] = node_case(torch, stream)
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
