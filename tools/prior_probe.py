"""What the keyframe depth prior (DESIGN.md 4.7) buys on the node's protocol: the c2 VGA 200-frame sequence with
device-resident frames, re-keyframing as rmd::DepthmapNode does (10 % converged or 0.5 m from the reference), the new
keyframe's prior taken in place from the one it replaces (SeedMatrix.setPriorPropagation).  For each sigma^2 fraction
f (0 = off) prints, on one JSON line: the number of keyframes, the mean number of frames a keyframe needs to reach the
threshold, the total device time of the fused update kernels (CUDA events around every update), and the median
|mu - ground truth| of the seeds converged when each keyframe was published.  GPU box only."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import multi_gpu, synth  # noqa: E402

W, H, N = 640, 480, 200
FRACS = (0.0, 1 / 64, 1 / 16, 1 / 4)
REPEATS = 3


def run(f, dev_frames, poses, depth, dmin, dmax, stream, torch):
    g = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*synth.dataset_camera(W, H)), device=0)
    g.setStream(stream.cuda_stream)
    g.setPriorPropagation(f)
    pairs, to_thresh, errors, keyframes = [], [], [], 0
    ref, take_ref = 0, True
    for k in range(N):
        if take_ref:
            g.setReferenceImageDevice(dev_frames[k].data_ptr(), W * 4, poses[k], dmin, dmax)
            ref, take_ref, keyframes = k, False, keyframes + 1
            continue
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        g.updateDevice(dev_frames[k].data_ptr(), W * 4, poses[k])
        b.record(stream)
        pairs.append((a, b))
        if 100.0 * g.getConvergedCount() / (W * H) > 10.0 or g.getDistFromRef() > 0.5:
            conv = g.downloadConvergence() == 1
            if 100.0 * conv.mean() > 10.0:
                to_thresh.append(k - ref)
            errors.append(np.abs(g.downloadDepthmap() - depth[ref])[conv])
            take_ref = True
    torch.cuda.synchronize()
    kernel_ms = sum(a.elapsed_time(b) for a, b in pairs)
    err = np.concatenate(errors) if errors else np.zeros(0, np.float32)
    return {"keyframes": keyframes, "mean_frames_to_10pct": float(np.mean(to_thresh)) if to_thresh else None,
            "keyframes_reaching_10pct": len(to_thresh), "fused_kernel_ms": kernel_ms, "updates": len(pairs),
            "published_seeds": int(err.size), "median_abs_error_m": float(np.median(err)) if err.size else None}


def main():
    import torch
    if rmd.device_count() < 1 or not torch.cuda.is_available():
        raise RuntimeError("prior_probe.py needs an H100")
    torch.cuda.set_device(0)
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    frames = [seq.frame(k) for k in range(N)]
    dmin, dmax = float(frames[0].depth.min()), float(frames[0].depth.max())
    dev_frames = torch.from_numpy(np.stack([fr.image for fr in frames])).cuda()
    poses = [np.ascontiguousarray(fr.T_cam_world.reshape(12)) for fr in frames]
    depth = [fr.depth for fr in frames]
    stream = torch.cuda.Stream()
    run(0.0, dev_frames, poses, depth, dmin, dmax, stream, torch)   # warm-up: module load, first launches
    results = {str(f): [] for f in FRACS}
    for _ in range(REPEATS):      # alternate the settings so drift on a shared host hits them alike
        for f in FRACS:
            results[str(f)].append(run(f, dev_frames, poses, depth, dmin, dmax, stream, torch))
    out = {}
    for f, rs in results.items():
        r = dict(rs[0])
        times = [x["fused_kernel_ms"] for x in rs]
        r["fused_kernel_ms"] = float(np.median(times))
        r["fused_kernel_ms_runs"] = times
        out[f] = r
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "nvidia-smi unavailable"
    print(json.dumps({"probe": "prior", "sequence": f"c2 {W}x{H}, {N} frames, device-resident",
                      "gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "by_sigma_sq_frac": out}))


if __name__ == "__main__":
    main()
