"""Device time of the TSDF volume's ESDF (DESIGN.md 4.8, 6) on volume_probe.py's scene: bench.py's c2 sequence (VGA),
a 256^3 and a 512^3 grid over it, eight keyframes' ground-truth depth fused.

  * compute: rmd_volume_esdf, the median of REPEATS runs after WARMUP, CUDA events on the volume's stream; the
    per-pass split (z, y, x) from a torch.profiler run of its own;
  * query: 10^6 random points in the window through rmd_volume_esdf_query_device, timed the same way;
  * bandwidth: the bytes each pass issues, counted from the kernel's loads and stores (below), over its time, against
    the 3.35 TB/s of the H100 SXM data sheet.

Bytes per voxel, per pass (a stack entry is a uint16, one per voxel and set that is a site; the z pass has one site
per voxel, the y and x passes are counted at two, their upper bound):
  z: records 8 (sweep 1) + 8 (sweep 2) + 8 (the record of each stack entry read back) + output 4 + stack 2 + 2 = 32
  y: input 4 + 4 + 4 * 2 (stack entries read back) + output 4 + stack 4 + 4 = 28
  x: input 4 + 4 + 4 * 2 + record weight 8 + snapshot 8 + stack 4 + 4 = 40
Prints one JSON line with the GPU's name and power limit.  GPU box only."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import multi_gpu, synth  # noqa: E402
from volume_probe import HBM_BYTES_PER_S, REPEATS, W, H, WARMUP, scene_box, timed  # noqa: E402

GRIDS = (256, 512)
PASS_BYTES = {"z": 32, "y": 28, "x": 40}
N_QUERY = 10 ** 6


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def pass_split(torch, v, stream):
    """Mean device time (ms) of each pass over REPEATS computes, from the profiler's kernel records."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(stream):
            for _ in range(REPEATS):
                v.computeEsdf()
        v.sync()
    ms = {"z": 0.0, "y": 0.0, "x": 0.0}
    for e in prof.events():
        for tag, name in (("z", "volume_esdf_kernel<0>"), ("y", "volume_esdf_kernel<1>"),
                          ("x", "volume_esdf_kernel<2>")):
            if name in e.name:
                ms[tag] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return {k: t / REPEATS for k, t in ms.items()}


def main():
    import torch
    if rmd.device_count() < 1 or not torch.cuda.is_available():
        raise RuntimeError("volume_esdf_probe.py needs an H100")
    torch.cuda.set_device(0)
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    frames = [seq.frame(k) for k in range(0, 200, 25)]
    lo, hi = scene_box(seq, frames)
    cam = rmd.PinholeCamera(*seq.camera)
    stream = torch.cuda.Stream()
    result = {"gpu": gpu_info()}
    rng = np.random.default_rng(0)
    for n in GRIDS:
        s = float(np.float32((hi - lo).max() / (n - 1 - 16)))
        v = rmd.TsdfVolume((n, n, n), s, lo - 8 * s, 4 * s, 64.0, device=0)
        v.setStream(stream.cuda_stream)
        for fr in frames:
            v.integrateDepth(fr.depth, cam, fr.T_cam_world)
        v.sync()
        med, _ = timed(stream, torch, v.computeEsdf)
        split = pass_split(torch, v, stream)
        d, w = v.downloadEsdf()
        pts = (v.origin + rng.uniform(0, 1, (N_QUERY, 3)) * (n - 1) * s).astype(np.float32)
        xyzw = torch.zeros((N_QUERY, 4), dtype=torch.float32, device="cuda")
        xyzw[:, :3] = torch.from_numpy(pts).cuda()
        dg = torch.empty((N_QUERY, 4), dtype=torch.float32, device="cuda")
        wq = torch.empty(N_QUERY, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        q_med, _ = timed(stream, torch, lambda: v.esdfQueryDevice(xyzw.data_ptr(), N_QUERY, dg.data_ptr(),
                                                                  wq.data_ptr()))
        vox = n ** 3
        passes = {}
        for k, t in split.items():
            gbs = PASS_BYTES[k] * vox / (t * 1e-3) / 1e9 if t > 0 else float("nan")
            passes[k] = {"ms": round(t, 3), "bytes_per_voxel": PASS_BYTES[k], "GB_per_s": round(gbs, 1),
                         "share_of_3.35TB/s": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)}
        total_bytes = sum(PASS_BYTES.values()) * vox
        result[f"{n}^3"] = {
            "compute_ms_median": round(med, 3),
            "passes": passes,
            "compute_GB_per_s": round(total_bytes / (med * 1e-3) / 1e9, 1),
            "unavoidable_16B_per_voxel_ms_at_3.35TB/s": round(16 * vox / HBM_BYTES_PER_S * 1e3, 3),
            "query_1e6_points_ms": round(q_med, 4),
            "query_points_per_s": round(N_QUERY / (q_med * 1e-3), -6),
            "occupied_voxels": int((d < 0).sum()), "known_voxels": int((w > 0).sum()),
            "esdf_MiB": 16 * vox / 2 ** 20,
        }
        del v
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
