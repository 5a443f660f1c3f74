"""Timing of the TSDF volume's brick store (DESIGN.md 6): a slab shift with the store against the same shift without
it, and mapMesh on a map of a few windows, at 256^3 and 512^3 with the intensity channel.

Each window holds a synthetic sphere shell, known in a band 4 voxels wide.  A round is a shift by +slab along z
followed by one by -slab: with the store, both move a slab of bricks out (evict) and the second brings the first
slab's bricks back (restore), with one flag read-back each.  The two volumes alternate within each round; the median
of the rounds is printed, as milliseconds per shift (CUDA events around the pair, over the volume's stream).

    python tools/volume_store_probe.py [--rounds 15] [--slab 32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import rpg_open_remode_b200 as rmd  # noqa: E402


def shell(n, s):
    k, j, i = np.meshgrid(*(np.arange(n, dtype=np.float32),) * 3, indexing="ij")
    r = np.sqrt((i - n / 2) ** 2 + (j - n / 2) ** 2 + (k - n / 2) ** 2)
    t = np.clip((r - 0.45 * n) / 4.0, -1, 1).astype(np.float32)   # reaches within 0.05 n of every face
    w = (np.abs(t) < 1).astype(np.float32)
    return t, w


def volume(n, store):
    v = rmd.TsdfVolume((n, n, n), 0.01, (0, 0, 0), 0.04, 64.0, device=0, intensity=True, store=store)
    t, w = shell(n, 0.01)
    v.upload(t, w)
    v.uploadIntensity(np.full_like(t, 0.5), w)
    return v


def timed(fn, stream):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--slab", type=int, default=32)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu, "rounds": args.rounds, "slab": args.slab}
    for n in (256, 512):
        stream = torch.cuda.Stream()
        vols = {store: volume(n, store) for store in (False, True)}
        for v in vols.values():
            v.setStream(stream.cuda_stream)
        d = np.array([0, 0, args.slab])
        times = {False: [], True: []}
        for r in range(args.rounds + 2):
            for store, v in vols.items():
                ms = timed(lambda: (v.shift(d), v.shift(-d)), stream) / 2
                if r >= 2:
                    times[store].append(ms)
        slab_bytes = n * n * args.slab * 16   # records + colour records of one slab
        vs = vols[True]
        assert vs.storeInfo()[0] > 0, "the slab holds no known voxel: nothing was stored"
        out[f"{n}"] = {"shift_ms_plain": float(np.median(times[False])),
                       "shift_ms_store": float(np.median(times[True])),
                       "slab_MiB": slab_bytes / 2 ** 20, "store_bricks": vs.storeInfo()[0],
                       "store_MiB": vs.storeInfo()[1] / 2 ** 20}
        # mapMesh on a map of four windows: the shell painted at four offsets
        for dd in ((n // 2, 0, 0), (0, n // 2, 0), (-n // 2, 0, n // 2)):
            vs.shift(dd)
            t, w = shell(n, 0.01)
            vs.upload(t, w)
        vs.sync()
        mesh_ms = []
        for r in range(max(3, args.rounds // 3)):
            t0 = time.perf_counter()
            mv, mt, _, _ = vs.mapMesh()
            mesh_ms.append(1e3 * (time.perf_counter() - t0))
        out[f"{n}"].update({"mapMesh_ms": float(np.median(mesh_ms)), "mapMesh_vertices": int(len(mv)),
                            "mapMesh_triangles": int(len(mt)), "map_bricks": vs.storeInfo()[0]})
        del vols, vs
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
