"""What the keyframe depth prior from the TSDF volume (DESIGN.md 4.8) buys on the node's protocol: the c2 VGA
200-frame sequence with device-resident frames, re-keyframing as rmd::DepthmapNode does (10 % converged or 0.5 m
from the reference), every finished keyframe denoised and fused into a 512^3 volume (the grid of
tests/test_volume.py::test_what_fusion_buys_on_c2).  Arms: no prior, the in-place splat (f = 1/16), the volume prior
at f in {1/64, 1/16, 1/4}, and splat and volume together (1/16 each), alternated over 3 repeats.  Per arm, one JSON
line: the number of keyframes; per keyframe the prior's coverage of the interior and the share of it within 1 % of the
range of the truth; the mean number of update frames to 10 % converged; the device time of the fused update kernels
(CUDA events around every update); per keyframe the prior kernel's time (events around the call) next to
rmd_volume_raycast of the same view; the median |mu - truth| of the published converged seeds.  GPU box only."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import _native, multi_gpu, synth  # noqa: E402
from test_volume_oracle import ground_truth_points, scene_grid  # noqa: E402

W, H, N = 640, 480, 200
F16 = rmd.PRIOR_SIGMA_SQ_FRAC
ARMS = (("off", 0.0, 0.0), ("splat 1/16", F16, 0.0), ("volume 1/64", 0.0, 1 / 64), ("volume 1/16", 0.0, F16),
        ("volume 1/4", 0.0, 1 / 4), ("splat + volume 1/16", F16, F16))
REPEATS = 3


def run(splat, vol_f, ctx):
    torch, stream, dev_frames, poses, depth, dmin, dmax, v = (ctx[k] for k in (
        "torch", "stream", "dev_frames", "poses", "depth", "dmin", "dmax", "volume"))
    cam = rmd.PinholeCamera(*synth.dataset_camera(W, H))
    g = rmd.SeedMatrix(W, H, cam, device=0)
    g.setStream(stream.cuda_stream)
    g.setPriorPropagation(splat)
    den = rmd.DepthmapDenoiser(W, H, device=0)
    den.setLargeSigmaSq(dmax - dmin)
    den.setStream(stream.cuda_stream)
    v.setStream(stream.cuda_stream)
    v.reset()
    img, ray = rmd.DeviceImage(W, H, "float32"), rmd.DeviceImage(W, H, "float32")
    pairs, prior_ev, ray_ev, kfs, errors = [], [], [], [], []
    ref, take_ref = 0, True
    ev = lambda: torch.cuda.Event(enable_timing=True)   # noqa: E731
    for k in range(N):
        if take_ref:
            g.setReferenceImageDevice(dev_frames[k].data_ptr(), W * 4, poses[k], dmin, dmax)
            if vol_f:
                a, b, c = ev(), ev(), ev()
                a.record(stream)
                g.priorFromVolume(v, vol_f)
                b.record(stream)
                prior_ev.append((a, b))
                _native.check(_native.lib().rmd_volume_raycast(
                    v.handle, W, H, cam.fx, cam.fy, cam.cx, cam.cy, poses[k].ctypes.data, ray.data, ray.pitch))
                c.record(stream)
                ray_ev.append((b, c))
            mu, s2, conv = g.downloadDepthmap(), g.downloadSigmaSq(), g.downloadConvergence()
            interior = conv != rmd.ConvergenceStates.BORDER
            prior = interior & (s2 != s2.max())
            good = prior & (np.abs(mu - depth[k]) <= 0.01 * (dmax - dmin))
            kfs.append({"frame": k, "coverage": float(prior.sum() / interior.sum()),
                        "within_1pct": float(good.sum() / max(1, prior.sum()))})
            ref, take_ref = k, False
            continue
        a, b = ev(), ev()
        a.record(stream)
        g.updateDevice(dev_frames[k].data_ptr(), W * 4, poses[k])
        b.record(stream)
        pairs.append((a, b))
        if 100.0 * g.getConvergedCount() / (W * H) > 10.0 or g.getDistFromRef() > 0.5:
            conv = g.downloadConvergence() == 1
            kfs[-1]["frames"] = k - ref
            kfs[-1]["reached_10pct"] = bool(100.0 * conv.mean() > 10.0)
            errors.append(np.abs(g.downloadDepthmap() - depth[ref])[conv])
            den.denoiseSeedsToDevice(g, img.data, img.pitch, 0.5, 200)   # the node's fuseDenoisedInto
            v.integrate(g, img)
            take_ref = True
    torch.cuda.synchronize()
    err = np.concatenate(errors) if errors else np.zeros(0, np.float32)
    reached = [kf["frames"] for kf in kfs if kf.get("reached_10pct")]
    later = kfs[1:]
    return {"keyframes": len(kfs),
            "coverage_per_keyframe": [round(kf["coverage"], 4) for kf in kfs],
            "within_1pct_per_keyframe": [round(kf["within_1pct"], 4) for kf in kfs],
            "mean_coverage_kf2_on": float(np.mean([kf["coverage"] for kf in later])) if later else None,
            "mean_within_1pct_kf2_on": float(np.mean([kf["within_1pct"] for kf in later])) if later else None,
            "mean_frames_to_10pct": float(np.mean(reached)) if reached else None,
            "keyframes_reaching_10pct": len(reached),
            "fused_kernel_ms": sum(a.elapsed_time(b) for a, b in pairs), "updates": len(pairs),
            "prior_kernel_ms_per_keyframe": [round(a.elapsed_time(b), 4) for a, b in prior_ev],
            "raycast_ms_per_keyframe": [round(a.elapsed_time(b), 4) for a, b in ray_ev],
            "published_seeds": int(err.size), "median_abs_error_m": float(np.median(err)) if err.size else None}


def main():
    import torch
    if rmd.device_count() < 1 or not torch.cuda.is_available():
        raise RuntimeError("volume_prior_probe.py needs an H100")
    torch.cuda.set_device(0)
    seq = synth.SyntheticSequence(W, H, seed=multi_gpu.keyframe_seed(0))    # bench.py's c2 sequence
    frames = [seq.frame(k) for k in range(N)]
    pts = np.concatenate([ground_truth_points(frames[k], seq.camera).reshape(-1, 3)
                          for k in list(range(0, N, 25)) + [N - 1]])
    s, origin = scene_grid(pts, 512, 4.0)
    ctx = {"torch": torch, "stream": torch.cuda.Stream(),
           "dev_frames": torch.from_numpy(np.stack([fr.image for fr in frames])).cuda(),
           "poses": [np.ascontiguousarray(fr.T_cam_world.reshape(12)) for fr in frames],
           "depth": [fr.depth for fr in frames],
           "dmin": float(frames[0].depth.min()), "dmax": float(frames[0].depth.max()),
           "volume": rmd.TsdfVolume((512, 512, 512), s, origin, np.float32(4.0) * s, 64.0, device=0)}
    run(F16, F16, ctx)   # warm-up: module load, first launches
    results = {name: [] for name, _, _ in ARMS}
    for _ in range(REPEATS):      # alternate the arms so drift on a shared host hits them alike
        for name, splat, vol_f in ARMS:
            results[name].append(run(splat, vol_f, ctx))
    out = {}
    for name, rs in results.items():
        r = dict(rs[0])
        for key in ("fused_kernel_ms",):
            r[key + "_runs"] = [x[key] for x in rs]
            r[key] = float(np.median(r[key + "_runs"]))
        prior = [t for x in rs for t in x["prior_kernel_ms_per_keyframe"]]
        ray = [t for x in rs for t in x["raycast_ms_per_keyframe"]]
        r["median_prior_kernel_ms"] = float(np.median(prior)) if prior else None
        r["median_raycast_ms"] = float(np.median(ray)) if ray else None
        out[name] = r
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "nvidia-smi unavailable"
    print(json.dumps({"probe": "volume_prior", "sequence": f"c2 {W}x{H}, {N} frames, device-resident, 512^3 volume",
                      "voxel_mm": float(s) * 1000, "gpu": torch.cuda.get_device_name(0),
                      "nvidia_smi_name_power_limit": q}))
    for name, r in out.items():
        print(json.dumps({"arm": name, **r}))


if __name__ == "__main__":
    main()
