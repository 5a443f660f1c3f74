"""Timing of the moving TSDF volume (DESIGN.md 4.8, 6): rmd_volume_shift, the three spills and the spill mesh (with
its intensities and normals) at 256^3 and 512^3, with the intensity channel, on a volume fused from one ground-truth
VGA frame.

CUDA events on the volume's stream, warm (one untimed call each first), the variants alternating within each of
`--reps` rounds; the median per variant.  The shift moves (8 + 8) B per voxel per channel; it is reported as bytes
over time against the H100 SXM's 3.35 TB/s data-sheet figure.  A spill reads what the surface passes read and is
reported against rmd_volume_surface_points / _intensity / _normals of the same grid; the spill mesh against
rmd_volume_mesh, its intensities and normals against the surface calls of the same kind.

    python tools/volume_shift_probe.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import rpg_open_remode_b200 as rmd  # noqa: E402
from rpg_open_remode_b200 import synth  # noqa: E402

HBM_TBPS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    W, H = 640, 480
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0900)
    f0 = seq.frame(0)
    fx, fy, cx, cy = seq.camera
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    ray = np.stack([(xx - cx) / fx, (yy - cy) / fy, np.ones_like(xx)], -1)
    ray /= np.linalg.norm(ray, axis=-1, keepdims=True)
    T = f0.T_world_cam.astype(np.float64)
    pts = ((ray * f0.depth[..., None]) @ T[:, :3].T + T[:, 3]).reshape(-1, 3)
    cam = rmd.PinholeCamera(*seq.camera)
    stream = torch.cuda.Stream()
    out = {"gpu": torch.cuda.get_device_name(0), "reps": args.reps}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    for n in (256, 512):
        lo, hi = pts.min(0), pts.max(0)
        s = float(((hi - lo) / (n - 1 - 16)).max())
        v = rmd.TsdfVolume((n, n, n), s, lo - 8 * s, 4 * s, 64.0, device=0, intensity=True)
        v.setStream(stream.cuda_stream)
        v.integrateDepth(f0.depth, cam, f0.T_cam_world, None, f0.image)
        # the shift moves by d and back: the 8-voxel margin around the surface keeps it whole.  The spills are
        # taken for a larger offset that drops part of the surface (they do not change the grid).
        d, ds = (3, -2, 1), (n // 4, -n // 8, n // 16)
        ops = {
            "shift": lambda: (v.shift(d), v.shift((-d[0], -d[1], -d[2]))),
            "spill_points": lambda: v.spillPoints(ds),
            "spill_intensity": lambda: v.spillIntensity(ds),
            "spill_normals": lambda: v.spillNormals(ds),
            "surface_points": lambda: v.surfacePoints(),
            "surface_intensity": lambda: v.surfaceIntensity(),
            "surface_normals": lambda: v.surfaceNormals(),
            "mesh": lambda: v.mesh(),
            "spill_mesh": lambda: v.spillMesh(ds),
            "spill_mesh_intensity": lambda: v.spillMeshIntensity(ds),
            "spill_mesh_normals": lambda: v.spillMeshNormals(ds),
        }
        for fn in ops.values():
            fn()
        v.sync()
        times = {k: [] for k in ops}
        for _ in range(args.reps):
            for k, fn in ops.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                fn()
                b.record(stream)
                b.synchronize()
                times[k].append(a.elapsed_time(b) / (2 if k == "shift" else 1))
        med = {k: float(np.median(t)) for k, t in times.items()}
        shift_bytes = 2 * 2 * 8 * n ** 3   # tsdf and intensity channels, one load and one store of 8 B each
        row = {f"{k}_ms": round(m, 4) for k, m in med.items()}
        row["spread_ms"] = {k: round(float(np.percentile(t, 90) - np.percentile(t, 10)), 4) for k, t in times.items()}
        row["shift_TBps"] = round(shift_bytes / (med["shift"] * 1e-3) / 1e12, 3)
        row["shift_of_peak"] = round(row["shift_TBps"] / HBM_TBPS, 3)
        for kind in ("points", "intensity", "normals"):
            row[f"spill_over_surface_{kind}"] = round(med[f"spill_{kind}"] / med[f"surface_{kind}"], 3)
        row["spill_mesh_over_mesh"] = round(med["spill_mesh"] / med["mesh"], 3)
        for kind in ("intensity", "normals"):
            row[f"spill_mesh_over_surface_{kind}"] = round(med[f"spill_mesh_{kind}"] / med[f"surface_{kind}"], 3)
        sv, st, _ = v.spillMesh(ds)
        mv, mt = v.mesh()
        row["spill_mesh_vertices_triangles"] = [len(sv), len(st)]
        row["mesh_vertices_triangles"] = [len(mv), len(mt)]
        row["spill_points"] = len(v.spillPoints(ds))
        row["surface_points"] = len(v.surfacePoints())
        out[f"{n}^3"] = row
        del v
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
