"""Sensitivity of the VGA 200-frame sequence time to the staged kernel's tuning knobs (GPU box)."""
import os, sys, itertools, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import rpg_open_remode_b200 as rmd
from rpg_open_remode_b200 import synth

W, H, N = (int(v) for v in os.environ.get('RMD_PROBE_SIZE', '640,480,200').split(','))
RUN = int(os.environ['RMD_PROBE_RUN']) if 'RMD_PROBE_RUN' in os.environ else None   # OPT_TUNE_RUN_CHUNKS (unset: the default)
seq = synth.SyntheticSequence(W, H, seed=0x5EED0002)
frames = np.empty((N, H, W), np.float32); poses = np.empty((N, 12), np.float32)
for k in range(N):
    f = seq.frame(k, want_depth=(k == 0)); frames[k] = f.image; poses[k] = f.T_cam_world.reshape(12)
    if k == 0: dmin, dmax = float(f.depth.min()), float(f.depth.max())
dev = torch.device("cuda", 0); stream = torch.cuda.Stream(dev); torch.cuda.set_stream(stream)
d_frames = torch.from_numpy(frames).to(dev)
g = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera), patch_side=int(os.environ.get('RMD_PROBE_PATCH', '5'))); g.setStream(stream.cuda_stream); g.setOption(rmd.OPT_KERNEL_VARIANT, rmd.VARIANT_STAGED)

def full(cfg):
    cfg = tuple(cfg)
    cfg = cfg + (0,) * max(0, 12 - len(cfg))
    return cfg + (64,) * (13 - len(cfg))


def run(cfg):
    cfg = full(cfg)
    for opt, val in zip((10, 11, 12, 13, 14, 15, 16, 17, 5, 6, 18, 19, 20), cfg): g.setOption(opt, val)
    if RUN is not None: g.setOption(rmd.OPT_TUNE_RUN_CHUNKS, RUN)
    best = 1e9; seg = None
    for rep in range(4):
        g.setReferenceImageDevice(d_frames[0].data_ptr(), W * 4, poses[0], dmin, dmax)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record(stream)
        g.updateDeviceBatch(d_frames[1].data_ptr(), W * H * 4, W * 4, poses[1:20]); ev[1].record(stream)
        g.updateDeviceBatch(d_frames[20].data_ptr(), W * H * 4, W * 4, poses[20:100]); ev[2].record(stream)
        g.updateDeviceBatch(d_frames[100].data_ptr(), W * H * 4, W * 4, poses[100:]); ev[3].record(stream)
        torch.cuda.synchronize()
        tot = ev[0].elapsed_time(ev[3])
        if tot < best:
            best = tot; seg = [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]
    return best, seg

# (split_max, split_min_items, split_items_per_cta, sparse_max_seeds, heavy_min_items, split_avg_pct, pdl, warp_tile_seeds,
#  chain_frames, seed_mode_pct[, grid_ctas[, ctas_per_sm]])
BASE = (16, 512, 384, 16, 128, 50, 1, 8)
CONFIGS = [BASE + (1, 0, 0, 2), BASE + (8, 0, 0, 2), BASE + (1, 0, 0, 3), BASE + (8, 0, 0, 3)]
if len(sys.argv) > 1:
    CONFIGS = [tuple(int(v) for v in a.split(",")) for a in sys.argv[1:]]
for cfg in CONFIGS:
    tot, seg = run(cfg)
    print(("run %d " % RUN if RUN is not None else "") + "split_max %2d min_items %4d per_cta %4d sparse %3d heavy_min %5d avg_pct %3d pdl %d warp_tiles %d chain %d seed_pct %d grid %d ctas/sm %d wt_cands %d : total %.2f ms (%.0f fps)  frames1-19 %.2f  20-99 %.2f  100-end %.2f ms" %
          (*full(cfg), tot, (N - 1) / tot * 1e3, *seg), flush=True)
