"""The staged search's run length (RMD_OPT_TUNE_RUN_CHUNKS: 4-candidate chunks per work item) must never
show in the results.

The VGA 200-frame sequence of the benchmark's c2 workload is run to the end with fixed run lengths from one
chunk per item (the chunk-major list) to a whole search per item, with the automatic per-tile choice, and with
the direct variant (one thread per pixel, no work list at all); the maps after 199 updates are compared bit for
bit.  Split tiles (several CTAs per tile, which must agree on the run length), chained launches and batched
launches of several keyframes run the same search code and are covered too.
"""
import numpy as np
import pytest

import rpg_open_remode_b200 as rmd
from rpg_open_remode_b200 import synth

pytestmark = pytest.mark.gpu

W, H, N = 640, 480, 200
FIELDS = ("conv", "mu", "sigma_sq", "a", "b")


@pytest.fixture(scope="module")
def c2():
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0002)
    frames = [seq.frame(k, want_depth=(k == 0)) for k in range(N)]
    images = np.stack([f.image for f in frames]).astype(np.float32)
    poses = np.stack([f.T_cam_world.reshape(12) for f in frames]).astype(np.float32)
    depth = frames[0].depth
    return seq, images, poses, float(depth.min()), float(depth.max())


def _snap(g):
    return {"conv": g.downloadConvergence(), "mu": g.downloadDepthmap(), "sigma_sq": g.downloadSigmaSq(),
            "a": g.downloadA(), "b": g.downloadB()}


def _same(A, B, what):
    for name in FIELDS:
        assert np.array_equal(A[name], B[name]), f"{what}: {name} differs at {(A[name] != B[name]).sum()} pixels"


def _new(c2, variant, knobs=()):
    seq, images, poses, dmin, dmax = c2
    g = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera))
    g.setOption(rmd.OPT_KERNEL_VARIANT, variant)
    g.setOption(rmd.OPT_SEED_MODE_PCT, 0)     # tile-major staged launches on every frame
    for opt, val in knobs:
        g.setOption(opt, val)
    g.setReferenceImage(images[0], poses[0], dmin, dmax)
    return g


def _run_host(g, c2):
    _, images, poses, _, _ = c2
    for k in range(1, N):
        g.update(images[k], poses[k])
    return _snap(g)


@pytest.fixture(scope="module")
def want(c2):
    return _run_host(_new(c2, rmd.VARIANT_DIRECT), c2)


@pytest.fixture(scope="module")
def want_run1(c2):
    return _run_host(_new(c2, rmd.VARIANT_STAGED, [(rmd.OPT_TUNE_RUN_CHUNKS, 1)]), c2)


def test_one_chunk_per_item_equals_direct(want, want_run1):
    _same(want_run1, want, "run 1 vs direct")


@pytest.mark.parametrize("run", [0, 2, 3, 4, 36])
def test_run_length_does_not_change_results(c2, want, want_run1, run):
    got = _run_host(_new(c2, rmd.VARIANT_STAGED, [(rmd.OPT_TUNE_RUN_CHUNKS, run)]), c2)
    _same(got, want_run1, f"run {run} vs run 1")
    _same(got, want, f"run {run} vs direct")


@pytest.mark.parametrize("run", [0, 4])
def test_split_tiles_with_runs(c2, want, run):
    knobs = [(rmd.OPT_TUNE_RUN_CHUNKS, run), (rmd.OPT_TUNE_SPLIT_MAX, 32), (rmd.OPT_TUNE_SPLIT_MIN_ITEMS, 1),
             (rmd.OPT_TUNE_SPLIT_ITEMS_PER_CTA, 32), (rmd.OPT_TUNE_SPLIT_AVG_PCT, 1), (rmd.OPT_TUNE_HEAVY_MIN_ITEMS, 1)]
    _same(_run_host(_new(c2, rmd.VARIANT_STAGED, knobs), c2), want, f"split tiles, run {run}")


@pytest.mark.parametrize("run", [0, 3])
def test_chained_device_batches_with_runs(c2, want, run):
    import torch
    _, images, poses, _, _ = c2
    dense = torch.from_numpy(images).to(torch.device("cuda", 0))
    g = _new(c2, rmd.VARIANT_STAGED, [(rmd.OPT_TUNE_RUN_CHUNKS, run), (rmd.OPT_CHAIN_FRAMES, 8)])
    g.updateDeviceBatch(dense[1].data_ptr(), W * H * 4, W * 4, poses[1:20])
    g.updateDeviceBatch(dense[20].data_ptr(), W * H * 4, W * 4, poses[20:100])
    g.updateDeviceBatch(dense[100].data_ptr(), W * H * 4, W * 4, poses[100:])
    _same(_snap(g), want, f"chained device batches, run {run}")
    torch.cuda.synchronize()


def test_batched_keyframes_with_runs(c2):
    """rmd_seeds_update_many: one launch serves several keyframes, each with its own run setting."""
    seq, images, poses, dmin, dmax = c2
    cam = rmd.PinholeCamera(*seq.camera)
    starts, runs = [0, 5, 11], [2, 0, 36]
    batch = [rmd.SeedMatrix(W, H, cam) for _ in starts]
    alone = [rmd.SeedMatrix(W, H, cam) for _ in starts]
    for g, run in zip(batch, runs):
        g.setOption(rmd.OPT_SEED_MODE_PCT, 0)
        g.setOption(rmd.OPT_TUNE_RUN_CHUNKS, run)
    for g in alone:
        g.setOption(rmd.OPT_KERNEL_VARIANT, rmd.VARIANT_DIRECT)
    for k in range(N):
        live = [i for i, s0 in enumerate(starts) if k > s0]
        if live:
            rmd.SeedMatrix.updateMany([batch[i] for i in live], images[k], poses[k])
            for i in live:
                alone[i].update(images[k], poses[k])
        for i, s0 in enumerate(starts):
            if k == s0:
                batch[i].setReferenceImage(images[k], poses[k], dmin, dmax)
                alone[i].setReferenceImage(images[k], poses[k], dmin, dmax)
    for i in range(len(starts)):
        _same(_snap(batch[i]), _snap(alone[i]), f"keyframe {i}, run {runs[i]}")


def test_option_range():
    g = rmd.SeedMatrix(64, 48, rmd.PinholeCamera(50.0, 50.0, 32.0, 24.0))
    for bad in (-1, 37):
        with pytest.raises(rmd.RmdError):
            g.setOption(rmd.OPT_TUNE_RUN_CHUNKS, bad)
    for ok in (0, 1, 36):
        g.setOption(rmd.OPT_TUNE_RUN_CHUNKS, ok)
