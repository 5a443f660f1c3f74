"""Every seed of ONE fused depth-filter update on the GPU against the float64 reference (tests/f64_depth_filter.py).

Each case downloads the full state before the update, runs one update with RMD_OPT_RECORD_MATCHES, downloads
everything and checks every pixel: absorbing seeds untouched bit for bit; the state equal to the float64
classification; NO_MATCH only when the float64 best score is < 0.5 + eps, with b' = b + 1 and mu, sigma^2, a
bit-identical; a recorded match that is a float64 comb candidate within 1e-3 px, an eps-arg-max scoring >= 0.5 - eps,
and mu, sigma^2, a, b within the float64 update's per-seed bound from that very match.  Seeds the error model calls
ambiguous are counted and printed, not checked; there must be few of them.  The cases are the shapes and paths where
kernels go wrong: sequence states (search-heavy first frames, split and warp-tile frames, retired tiles), ragged
sizes, 7x7, VGA, every organisation of the kernel on one state, degenerate states, poses and images, and a planted
bug (7-bit texture weights) that the checker must catch.
"""
import numpy as np
import pytest

import f64_depth_filter as F
import rpg_open_remode_b200 as rmd
from rpg_open_remode_b200 import synth

pytestmark = pytest.mark.gpu

STATE_FIELDS = ((rmd.FIELD_MU, "mu"), (rmd.FIELD_SIGMA_SQ, "sigma_sq"), (rmd.FIELD_A, "a"), (rmd.FIELD_B, "b"))
IDENTITY = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _snap(g):
    return dict(mu=g.downloadDepthmap(), sigma_sq=g.downloadSigmaSq(), a=g.downloadA(), b=g.downloadB(),
                conv=g.downloadConvergence())


def _same_state(A, B):
    return all(np.array_equal(A[k].view(np.int32), B[k].view(np.int32)) for k in ("mu", "sigma_sq", "a", "b", "conv"))


def _handle(seq, patch=5, knobs=()):
    g = rmd.SeedMatrix(seq.width, seq.height, rmd.PinholeCamera(*seq.camera), patch_side=patch)
    g.setOption(rmd.OPT_RECORD_MATCHES, 1)
    for opt, val in knobs:
        g.setOption(opt, val)
    return g


class Case:
    """A keyframe (reference image, pose, depth range) and the frames that follow it."""

    def __init__(self, seq, ref_img=None, T_ref=None):
        self.seq = seq
        f0 = seq.frame(0)
        self.ref = f0.image if ref_img is None else ref_img
        self.T_ref = f0.T_cam_world if T_ref is None else T_ref
        self.dmin, self.dmax = float(f0.depth.min()), float(f0.depth.max())

    def start(self, g):
        g.setReferenceImage(self.ref, self.T_ref, self.dmin, self.dmax)

    def frame_model(self, curr, T_curr_world, patch=5):
        T_cr = F.se3_mul_f32(T_curr_world, F.se3_inv_f32(self.T_ref))
        return F.Frame(self.ref, curr, self.seq.camera, T_cr, self.dmin, self.dmax, patch=patch)


def _check(name, fr, pre, g, trust_conv=True, cache=None, search_mask=None, expect_fail=False, flat_ok=False):
    post = _snap(g)
    rep = F.check_frame(fr, pre, post, g.downloadEpipolarMatches(), trust_conv=trust_conv, search_mask=search_mask,
                        search_cache=cache)
    print(f"{name}: {rep}")
    if expect_fail:
        return rep
    assert rep.n_fail == 0, f"{name}: {rep}"
    # flat patches leave the NCC score to rounding (0 / 0 in exact arithmetic); only the degenerate-image cases
    # plant them on purpose, everywhere else they count against the same 0.1 %
    n_amb = rep.n_ambiguous - (rep.n_undetermined if flat_ok else 0)
    assert n_amb <= max(1, 0.001 * rep.n_updated), f"{name}: {rep}"
    return rep


def _run_to(case, g, n):
    """setReferenceImage and frames 1 .. n-1; returns the state before frame n."""
    case.start(g)
    for k in range(1, n):
        f = case.seq.frame(k, want_depth=False)
        g.update(f.image, f.T_cam_world)
    return _snap(g)


def _checked_update(case, g, n, patch=5):
    f = case.seq.frame(n, want_depth=False)
    g.update(f.image, f.T_cam_world)
    return case.frame_model(f.image, f.T_cam_world, patch)


# ------------------------------------------------------------------------------------------ sequence states

@pytest.mark.parametrize("size,patch,n", [((320, 240), 5, 1), ((320, 240), 5, 4), ((320, 240), 5, 13),
                                          ((320, 240), 5, 40), ((320, 240), 5, 120), ((101, 77), 5, 7),
                                          ((33, 17), 5, 5), ((203, 131), 7, 9)])
def test_sequence_state_every_seed(size, patch, n):
    seq = synth.SyntheticSequence(*size, seed=0x5EED0001)
    case = Case(seq)
    g = _handle(seq, patch)
    pre = _run_to(case, g, n)
    fr = _checked_update(case, g, n, patch)
    _check(f"{size} {patch}x{patch} frame {n}", fr, pre, g)


def test_vga_frame_40_edge_and_busiest_tiles():
    """VGA: every seed's state is checked; the float64 search runs on every seed of 64 tiles (32 x 8): the image's
    corner and edge tiles and the tiles with the most search work (the ones the staged kernel splits)."""
    seq = synth.SyntheticSequence(640, 480, seed=0x5EED0002)
    case = Case(seq)
    g = _handle(seq)
    pre = _run_to(case, g, 40)
    fr = _checked_update(case, g, 40)
    W, H = 640, 480
    tx, ty = W // 32, H // 8
    with np.errstate(invalid="ignore"):
        work = np.where(pre["conv"] == F.UPDATE, np.sqrt(np.maximum(pre["sigma_sq"], 0)), 0)
    work = np.nan_to_num(work).reshape(ty, 8, tx, 32).sum(axis=(1, 3))
    edge = np.zeros((ty, tx), bool)
    edge[[0, 0, -1, -1, 0, -1, ty // 2, ty // 2], [0, -1, 0, -1, tx // 2, tx // 2, 0, -1]] = True
    edge[0, ::5] = edge[-1, ::5] = True
    busy = np.zeros((ty, tx), bool)
    busy.flat[np.argsort(np.where(edge, -1, work).ravel())[::-1][:64 - int(edge.sum())]] = True
    tiles = edge | busy
    mask = np.repeat(np.repeat(tiles, 8, axis=0), 32, axis=1)
    assert tiles.sum() == 64
    _check("VGA frame 40, 64 tiles", fr, pre, g, search_mask=mask)


# ------------------------------------------------------------------------------------------ organisations

ORGS = {
    "direct": [(rmd.OPT_KERNEL_VARIANT, rmd.VARIANT_DIRECT)],
    "staged": [],
    "all_sparse": [(rmd.OPT_TUNE_SPARSE_MAX_SEEDS, 256), (rmd.OPT_TUNE_SPLIT_MAX, 1), (rmd.OPT_TUNE_PDL, 2)],
    "split_everything": [(rmd.OPT_TUNE_SPLIT_MAX, 32), (rmd.OPT_TUNE_SPLIT_MIN_ITEMS, 1),
                         (rmd.OPT_TUNE_SPLIT_ITEMS_PER_CTA, 1), (rmd.OPT_TUNE_SPLIT_AVG_PCT, 1),
                         (rmd.OPT_TUNE_HEAVY_MIN_ITEMS, 1)],
    "run_chunks_1": [(rmd.OPT_TUNE_RUN_CHUNKS, 1)],
    "run_chunks_2": [(rmd.OPT_TUNE_RUN_CHUNKS, 2)],
    "run_chunks_9": [(rmd.OPT_TUNE_RUN_CHUNKS, 9)],
    "seed_major": [(rmd.OPT_SEED_MODE_PCT, 100)],   # seed-major from the third or fourth frame on
}


@pytest.mark.parametrize("n", [4, 40])
def test_organisations_every_seed(qvga_sequence, n):
    """The same state checked through every organisation of the kernel; the float64 search is computed once."""
    case = Case(qvga_sequence)
    cache, pre0, fr = {}, None, None
    for name, knobs in ORGS.items():
        g = _handle(qvga_sequence, knobs=knobs)
        pre = _run_to(case, g, n)
        if pre0 is None:
            pre0 = pre
        assert _same_state(pre, pre0), name
        fr = _checked_update(case, g, n)
        _check(f"{name}, frame {n}", fr, pre, g, cache=cache)
    # rmd_seeds_update_many: the state in slot 3 of 8 keyframes updated together
    hs = [_handle(qvga_sequence) for _ in range(8)]
    for h in hs:
        case.start(h)
    for k in range(1, n + 1):
        f = qvga_sequence.frame(k, want_depth=False)
        if k == n:
            pre = _snap(hs[3])
            assert _same_state(pre, pre0)
        rmd.SeedMatrix.updateMany(hs, f.image, f.T_cam_world)
    _check(f"update_many slot 3, frame {n}", fr, pre, hs[3], cache=cache)
    # planted bug on the real kernel: 7-bit texture weights from the same state must be caught
    g = _handle(qvga_sequence)
    pre = _run_to(case, g, n)
    g.setOption(rmd.OPT_TEX_FRAC_BITS, 7)
    _checked_update(case, g, n)
    rep = _check(f"7-bit weights, frame {n}", fr, pre, g, cache=cache, expect_fail=True)
    # a weight moved by at most 1/256 flips the arg-max beyond eps only rarely: two seeds at frames 4 and 40
    assert rep.fail.get("search", 0) >= 1, f"the planted 7-bit weights were not caught: {rep}"


# ------------------------------------------------------------------------------------------ degenerate states

def _degenerate(dmin, dmax):
    """Per-seed (mu, sigma^2, a, b) rows of the degenerate kinds."""
    mu0, s0 = 0.5 * (dmin + dmax), ((dmax - dmin) ** 2) / 36.0
    tiny = np.float32(np.finfo(np.float32).smallest_subnormal)
    return np.array([
        (mu0, 0.0, 10, 10), (mu0, tiny, 10, 10), (mu0, -1e-12, 10, 10), (mu0, np.nan, 10, 10), (mu0, np.inf, 10, 10),
        (mu0, 1e30, 10, 10),
        (0.05, 0.0009, 10, 10),            # mu - 3 sigma < 0.01: the low end is clamped
        (dmin, s0, 10, 10), (10 * dmax, s0, 10, 10),
        (mu0, s0, 1, 1),                   # (a - 1) / (a + b - 2) = 0 / 0
        (mu0, s0, 1e6, 1), (mu0, s0, 1, 1e6), (mu0, s0 * 1e-3, 30, 2),
    ], np.float64)


@pytest.mark.parametrize("layout", ["stripes", "isolated"])
def test_degenerate_states(qvga_sequence, layout):
    """Degenerate seeds uploaded in stripes (every 32 x 8 tile mixes them with normal seeds) or isolated among
    converged seeds (tiles with a handful of live seeds take the warp-tile path)."""
    seq = qvga_sequence
    case = Case(seq)
    g = _handle(seq)
    st = _run_to(case, g, 4)
    rows = _degenerate(case.dmin, case.dmax)
    H, W = seq.height, seq.width
    ys, xs = np.mgrid[0:H, 0:W]
    if layout == "stripes":
        sel = (ys % 8 == 3) | (xs % 32 == 7)
    else:
        sel = (ys % 8 == 4) & (xs % 32 == 11)
        conv_like = ~sel
        st["sigma_sq"][conv_like] = np.float32(1e-6)
        st["a"][conv_like], st["b"][conv_like] = np.float32(50), np.float32(2)
    kind = (xs + 3 * ys) % len(rows)
    for i, name in enumerate(("mu", "sigma_sq", "a", "b")):
        st[name][sel] = rows[kind[sel], i].astype(np.float32)
    for fid, name in STATE_FIELDS:
        g.uploadState(fid, st[name])
    pre = _snap(g)
    fr = _checked_update(case, g, 4)
    _check(f"degenerate states, {layout}", fr, pre, g, trust_conv=False)


# ------------------------------------------------------------------------------------------ degenerate poses

def _pose(t=(0.0, 0.0, 0.0), rot_deg=0.0):
    c, s = np.cos(np.radians(rot_deg)), np.sin(np.radians(rot_deg))
    T = np.array([[c, 0, s, t[0]], [0, 1, 0, t[1]], [-s, 0, c, t[2]]], np.float64)
    return T.astype(np.float32)


@pytest.mark.parametrize("name", ["identity", "pure_rotation", "forward", "backward", "tiny_baseline", "out_of_image"])
def test_degenerate_poses(small_sequence, name):
    """From a fresh keyframe at the identity pose: zero motion (defined deviation 1), a pure rotation (every depth
    projects to one point), motion along the optical axis (epipole inside the image), a 1e-5 baseline (tau cancels
    completely: the bounds are huge, the branch and finiteness still count), a lateral motion that takes most mean
    projections out of the image (no candidates, NO_MATCH)."""
    seq = small_sequence
    case = Case(seq, T_ref=IDENTITY)
    mid = 0.5 * (case.dmin + case.dmax)
    T = {"identity": IDENTITY, "pure_rotation": _pose(rot_deg=2.0), "forward": _pose((0, 0, -0.05 * mid)),
         "backward": _pose((0, 0, 0.05 * mid)), "tiny_baseline": _pose((1e-5, 0, 0)),
         "out_of_image": _pose((1.5 * mid, 0, 0))}[name]
    g = _handle(seq)
    case.start(g)
    pre = _snap(g)
    curr = seq.frame(1, want_depth=False).image
    g.update(curr, T)
    if name == "tiny_baseline":
        # tau cancels completely and the triangulated point's side of the camera is a matter of rounding: the model
        # calls most updates ambiguous; what is checked is the rest, the search, and that no NaN is ever stored
        rep = _check(f"pose {name}", case.frame_model(curr, T), pre, g, expect_fail=True)
        assert rep.n_fail == 0, rep
        post = _snap(g)
        live = np.isin(post["conv"], (F.UPDATE, F.NO_MATCH))
        assert not np.isnan(post["mu"][live]).any() and not np.isnan(post["a"][live]).any()
        return
    rep = _check(f"pose {name}", case.frame_model(curr, T), pre, g)
    if name == "out_of_image":
        assert (g.downloadConvergence() == F.NO_MATCH).mean() > 0.25, rep


# ------------------------------------------------------------------------------------------ degenerate images

@pytest.mark.parametrize("name", ["constant_block", "saturated", "checkerboard"])
def test_degenerate_images(small_sequence, name):
    """A constant block in both images (const_templ_denom ~ 0: the score is a rounding residue times
    rsqrt(FLT_MIN), the seed must be ambiguous or agree), 0 / 255 saturated regions of 8-bit frames, and a
    one-pixel checkerboard where the weight quantisation decides the arg-max."""
    seq = small_sequence
    f0, f1 = seq.frame(0), seq.frame(1, want_depth=False)
    ref, curr = f0.image_u8.copy(), f1.image_u8.copy()
    if name == "constant_block":
        ref[40:50, 60:70] = 128
        curr[38:52, 58:72] = 128
    elif name == "saturated":
        for img in (ref, curr):
            img[20:50, 20:50] = 0
            img[60:100, 90:140] = 255
    else:
        yy, xx = np.mgrid[0:40, 0:60]
        for img in (ref, curr):
            img[30:70, 50:110] = 255 * ((yy + xx) % 2)
    to_f = lambda u8: (u8.astype(np.float32) * np.float32(1.0 / 255.0)).astype(np.float32)
    case = Case(seq, ref_img=to_f(ref))
    g = _handle(seq)
    case.start(g)
    pre = _snap(g)
    g.update(to_f(curr), f1.T_cam_world)
    _check(f"image {name}", case.frame_model(to_f(curr), f1.T_cam_world), pre, g, flat_ok=True)


# ------------------------------------------------------------------------------------------ seed initialisation

@pytest.mark.parametrize("size,patch", [((320, 240), 5), ((101, 77), 5), ((33, 17), 5), ((203, 131), 7),
                                        ((203, 131), 5)])
def test_seed_init_template_statistics(size, patch):
    """sum_templ within the fp32 summation bound of the float64 sum, const_templ_denom within its propagated bound,
    per pixel, including the clamped edge ring."""
    seq = synth.SyntheticSequence(*size, seed=0x5EED0040 + size[0])
    case = Case(seq)
    g = _handle(seq, patch)
    case.start(g)
    St, eSt, ctd, ectd = F.templ_stats(case.ref, patch)
    d_st = np.abs(g.downloadSumTempl().astype(np.float64) - St)
    d_ctd = np.abs(g.downloadConstTemplDenom().astype(np.float64) - ctd)
    assert (d_st <= eSt).all(), f"sum_templ: {(d_st > eSt).sum()} pixels outside the bound"
    assert (d_ctd <= ectd).all(), f"const_templ_denom: {(d_ctd > ectd).sum()} pixels outside the bound"
