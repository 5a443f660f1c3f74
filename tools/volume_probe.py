"""Device time of the TSDF volume's operations (DESIGN.md 4.8, 6) on bench.py's c2 scene (VGA): integration of one
keyframe's depth and state map into a 256^3 and a 512^3 grid over the scene, surface-point extraction, the
triangle mesh (rmd_volume_mesh_device, vertices and triangles) and a VGA raycast, and the intensity channel's
variants of integration (the frame's image fused too), surface extraction and raycast next to the plain ones, and the
surface normals and the raycast with normals next to the surface points and the plain raycast.  Each time is the median of REPEATS runs after WARMUP, measured with CUDA events on the volume's stream.
The achieved bandwidth of an integration counts 16 B per updated voxel (record read + write) and 8 B per pixel
(depth + state) over its kernel time, against the 3.35 TB/s of the H100 SXM data sheet.  Prints one JSON line with
the GPU's name and power limit.  GPU box only."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import _native, multi_gpu, synth  # noqa: E402

W, H = 640, 480
GRIDS = (256, 512)
WARMUP, REPEATS = 3, 20
HBM_BYTES_PER_S = 3.35e12


def scene_box(seq, frames):
    """Bounding box of the frames' ground-truth points (float64)."""
    fx, fy, cx, cy = seq.camera
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    ray = np.stack([(xx - cx) / fx, (yy - cy) / fy, np.ones_like(xx)], -1)
    ray /= np.linalg.norm(ray, axis=-1, keepdims=True)
    pts = []
    for fr in frames:
        T = fr.T_world_cam.astype(np.float64)
        pts.append(((ray * fr.depth[..., None]) @ T[:, :3].T + T[:, 3]).reshape(-1, 3))
    pts = np.concatenate(pts)
    return pts.min(0), pts.max(0)


def timed(stream, torch, fn):
    times = []
    for r in range(WARMUP + REPEATS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        if r >= WARMUP:
            times.append(a.elapsed_time(b))
    return float(np.median(times)), times


def main():
    import torch
    if rmd.device_count() < 1 or not torch.cuda.is_available():
        raise RuntimeError("volume_probe.py needs an H100")
    torch.cuda.set_device(0)
    L = _native.lib()
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    lo, hi = scene_box(seq, [seq.frame(k) for k in range(0, 200, 25)])
    fr = seq.frame(100)
    cam = rmd.PinholeCamera(*seq.camera)
    depth = rmd.DeviceImage(W, H, "float32")
    depth.setDevData(fr.depth)
    conv = rmd.DeviceImage(W, H, "int32")
    conv.setDevData(np.ones((H, W), np.int32))              # every pixel CONVERGED: the state map is read
    out = rmd.DeviceImage(W, H, "float32")
    image = rmd.DeviceImage(W, H, "float32")
    image.setDevData(fr.image)
    out_i = rmd.DeviceImage(W, H, "float32")
    out_n = rmd.DeviceImage(4 * W, H, "float32")            # float4 normals
    T = np.ascontiguousarray(fr.T_cam_world.reshape(12))
    c = ctypes.c_float
    stream = torch.cuda.Stream()
    result = {}
    for n in GRIDS:
        s = float(np.float32((hi - lo).max() / (n - 1 - 16)))   # tau = 4 voxels, padded by 2 tau
        v = rmd.TsdfVolume((n, n, n), s, lo - 8 * s, 4 * s, 64.0, device=0, intensity=True)
        v.setStream(stream.cuda_stream)

        def integrate():
            _native.check(L.rmd_volume_integrate_depth(v.handle, W, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy),
                                                       T.ctypes.data, depth.data, depth.pitch, conv.data, conv.pitch))

        integrate()
        v.sync()
        updated = int((v.download()[1] > 0).sum())
        v.reset()
        ms_int, runs_int = timed(stream, torch, integrate)

        def integrate_intensity():
            _native.check(L.rmd_volume_integrate_depth_intensity(
                v.handle, W, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy), T.ctypes.data, depth.data, depth.pitch,
                conv.data, conv.pitch, image.data, image.pitch))

        ms_int_i, runs_int_i = timed(stream, torch, integrate_intensity)
        count = ctypes.c_size_t()
        points = rmd.DeviceImage(4 * 4 * n * n, 1, "float32")   # room for 4 n^2 points

        def extract():
            _native.check(L.rmd_volume_surface_points_device(v.handle, points.data, 4 * n * n, ctypes.byref(count)))

        ms_pts, runs_pts = timed(stream, torch, extract)

        def extract_intensity():
            _native.check(L.rmd_volume_surface_intensity_device(v.handle, points.data, 4 * n * n, ctypes.byref(count)))

        ms_pts_i, runs_pts_i = timed(stream, torch, extract_intensity)

        def extract_normals():
            _native.check(L.rmd_volume_surface_normals_device(v.handle, points.data, 4 * n * n, ctypes.byref(count)))

        ms_pts_n, runs_pts_n = timed(stream, torch, extract_normals)
        n_tri = ctypes.c_size_t()
        tris = rmd.DeviceImage(3 * 8 * n * n, 1, "int32")         # room for 8 n^2 triangles

        def mesh():
            _native.check(L.rmd_volume_mesh_device(v.handle, points.data, 4 * n * n, tris.data, 8 * n * n,
                                                   ctypes.byref(count), ctypes.byref(n_tri)))

        ms_mesh, runs_mesh = timed(stream, torch, mesh)
        assert count.value <= 4 * n * n and n_tri.value <= 8 * n * n

        def raycast():
            _native.check(L.rmd_volume_raycast(v.handle, W, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy),
                                               T.ctypes.data, out.data, out.pitch))

        ms_ray, runs_ray = timed(stream, torch, raycast)

        def raycast_intensity():
            _native.check(L.rmd_volume_raycast_intensity(v.handle, W, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy),
                                                         T.ctypes.data, out.data, out.pitch, out_i.data, out_i.pitch))

        ms_ray_i, runs_ray_i = timed(stream, torch, raycast_intensity)

        def raycast_normals():
            _native.check(L.rmd_volume_raycast_normals(v.handle, W, H, c(cam.fx), c(cam.fy), c(cam.cx), c(cam.cy),
                                                       T.ctypes.data, out.data, out.pitch, out_n.data, out_n.pitch))

        ms_ray_n, runs_ray_n = timed(stream, torch, raycast_normals)
        v.sync()
        hit = int((out.getDevData() > 0).sum())
        algo_bytes = 16 * updated + 8 * W * H
        result[f"{n}^3"] = {
            "voxel_size_m": s, "voxels": n ** 3, "voxels_updated": updated,
            "integrate_ms": ms_int, "integrate_ms_runs": runs_int,
            "integrate_algorithmic_bytes": algo_bytes,
            "integrate_bandwidth_TBps": algo_bytes / (ms_int * 1e-3) / 1e12,
            "integrate_share_of_3.35TBps": algo_bytes / (ms_int * 1e-3) / HBM_BYTES_PER_S,
            "record_stream_bytes": 8 * n ** 3,
            "surface_points": int(count.value), "surface_points_ms": ms_pts, "surface_points_ms_runs": runs_pts,
            "surface_points_record_bandwidth_TBps": 8 * n ** 3 / (ms_pts * 1e-3) / 1e12,
            "mesh_vertices": int(count.value), "mesh_triangles": int(n_tri.value), "mesh_ms": ms_mesh,
            "mesh_ms_runs": runs_mesh, "mesh_over_surface_points": ms_mesh / ms_pts,
            "raycast_vga_ms": ms_ray, "raycast_vga_ms_runs": runs_ray, "raycast_pixels_hit": hit,
            "integrate_intensity_ms": ms_int_i, "integrate_intensity_ms_runs": runs_int_i,
            "integrate_intensity_over_plain": ms_int_i / ms_int,
            "surface_intensity_ms": ms_pts_i, "surface_intensity_ms_runs": runs_pts_i,
            "surface_intensity_over_points": ms_pts_i / ms_pts,
            "raycast_intensity_vga_ms": ms_ray_i, "raycast_intensity_vga_ms_runs": runs_ray_i,
            "raycast_intensity_over_plain": ms_ray_i / ms_ray,
            "surface_normals_ms": ms_pts_n, "surface_normals_ms_runs": runs_pts_n,
            "surface_normals_over_points": ms_pts_n / ms_pts,
            "raycast_normals_vga_ms": ms_ray_n, "raycast_normals_vga_ms_runs": runs_ray_n,
            "raycast_normals_over_plain": ms_ray_n / ms_ray}
        del v
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "nvidia-smi unavailable"
    print(json.dumps({"probe": "volume", "scene": f"c2 {W}x{H}, frame 100 ground truth, grid over frames 0-199",
                      "gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "grids": result}))


if __name__ == "__main__":
    main()
