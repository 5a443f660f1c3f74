"""Keyframe depth prior (csrc/prior.cu, DESIGN.md 4.7): a new keyframe takes its prior from the CONVERGED seeds of
another keyframe, forward-splatted into the new reference view.

  * CPU: the oracle (oracle/rmd_oracle_propagate.c, bound by prior_oracle.py) against an independent numpy float32
    evaluation on random states and poses, and known answers.
  * GPU: the product against the oracle bit for bit (sources that last ran the staged kernel, the direct kernel and
    seed-major mode; 5x5 and 7x7; differing sizes), the in-place and cross-handle forms against each other, the
    default (off) against a fresh handle, the kernel organisations against each other from a propagated prior,
    what the prior does for convergence and accuracy, and every error code.
"""
import numpy as np
import pytest

import oracle_binding as ob
import prior_oracle as po

F = np.float32
EMPTY = np.uint32(0xFFFFFFFF)


def _numpy_splat(mu, conv, src_cam, T_world_ref, dst_size, dst_cam, T_curr_world, dmin, dmax):
    """The splat in numpy float32, one rounding per operation.  Returns the z-buffer and, per accepted point, how
    close u + 0.5 or v + 0.5 came to an integer (pixels where rounding could go either way)."""
    h, w = mu.shape
    dw, dh = dst_size
    fx, fy, cx, cy = (F(c) for c in src_cam)
    yy, xx = np.mgrid[0:h, 0:w]
    sel = conv == 1
    x, y, m = xx[sel].astype(F), yy[sel].astype(F), mu[sel].astype(F)
    vx, vy = (x - cx) / fx, (y - cy) / fy
    inv = F(1) / np.sqrt((vx * vx + vy * vy) + F(1) * F(1))
    q = ((vx * inv) * m, (vy * inv) * m, (F(1) * inv) * m)
    A = np.asarray(T_world_ref, F).reshape(3, 4)
    wp = [((A[r, 0] * q[0] + A[r, 1] * q[1]) + A[r, 2] * q[2]) + A[r, 3] for r in range(3)]
    B = np.asarray(T_curr_world, F).reshape(3, 4)
    p = [((B[r, 0] * wp[0] + B[r, 1] * wp[1]) + B[r, 2] * wp[2]) + B[r, 3] for r in range(3)]
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2])
        dfx, dfy, dcx, dcy = (F(c) for c in dst_cam)
        u = (dfx * p[0]) / p[2] + dcx
        v = (dfy * p[1]) / p[2] + dcy
        tu, tv = np.floor(u + F(0.5)), np.floor(v + F(0.5))
        ok = (p[2] > 0) & (d >= F(dmin)) & (d <= F(dmax)) & (tu >= 0) & (tu < dw) & (tv >= 0) & (tv < dh)
    z = np.full(dh * dw, EMPTY, np.uint32)
    idx = tv[ok].astype(np.int64) * dw + tu[ok].astype(np.int64)
    np.minimum.at(z, idx, d[ok].view(np.uint32))
    frac = lambda t: np.abs((t + F(0.5)) - np.round(t + F(0.5)))
    near = np.minimum(frac(u[ok]), frac(v[ok])) < 1e-3
    return z.reshape(dh, dw), idx[near], int(ok.sum())


def _rot(rng, angle):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _pose(R, t):
    return np.concatenate([np.asarray(R, F), np.asarray(t, F).reshape(3, 1)], axis=1).astype(F)


@pytest.mark.parametrize("src_size,dst_size,seed", [((160, 120), (160, 120), 1), ((320, 240), (160, 120), 2),
                                                    ((96, 72), (200, 150), 3), ((640, 480), (640, 480), 4)])
def test_oracle_splat_equals_numpy_float32(src_size, dst_size, seed):
    rng = np.random.default_rng(0x9A10 + seed)
    (sw, sh), (dw, dh) = src_size, dst_size
    mu = rng.uniform(0.8, 2.5, (sh, sw)).astype(F)
    conv = rng.integers(0, 6, (sh, sw)).astype(np.int32)
    scam = tuple(float(F(c)) for c in (481.2 * sw / 640, -480.0 * sh / 480, (sw - 1) / 2, (sh - 1) / 2))
    dcam = tuple(float(F(c)) for c in (481.2 * dw / 640, -480.0 * dh / 480, (dw - 1) / 2, (dh - 1) / 2))
    T_world_ref = _pose(_rot(rng, 0.3), rng.normal(size=3))
    # destination: a small motion away from the source camera
    T_world_dst = _pose(_rot(rng, 0.08) @ T_world_ref[:, :3], T_world_ref[:, 3] + rng.normal(scale=0.1, size=3))
    T_curr_world = ob.se3_inv(T_world_dst)
    dmin, dmax = 1.0, 2.2
    got, n_got = po.prior_splat(mu, conv, scam, T_world_ref, (dw, dh), dcam, T_curr_world, dmin, dmax)
    want, near, n_want = _numpy_splat(mu, conv, scam, T_world_ref, (dw, dh), dcam, T_curr_world, dmin, dmax)
    assert n_got == n_want > 0.05 * (conv == 1).sum()
    # only a pixel a point reached from within 1e-3 px of a rounding boundary may differ
    differ = np.flatnonzero(got.ravel() != want.ravel())
    assert np.isin(differ, near).all(), differ[~np.isin(differ, near)][:10]
    assert (got != EMPTY).sum() > 0.01 * dw * dh


def test_oracle_known_answers():
    W, H = 64, 48
    cam = (50.0, -50.0, 31.5, 23.5)
    I = np.eye(4, dtype=F)[:3]
    rng = np.random.default_rng(7)
    mu = rng.uniform(1.0, 2.0, (H, W)).astype(F)
    conv = rng.integers(0, 6, (H, W)).astype(np.int32)
    f, dmin, dmax, patch = 1 / 16, 0.5, 3.0, 5
    sig_max = F(F(F(dmax) - F(dmin)) * F(F(dmax) - F(dmin))) / F(36)
    # identity pose, same camera: every CONVERGED interior pixel lands on itself with |d - mu| of a few ulp
    mu_o, s2, a, b, cv = po.propagate_prior(mu, conv, cam, I, (W, H), cam, I, patch, dmin, dmax, f)
    interior = cv != ob.BORDER
    hit = interior & (conv == ob.CONVERGED)
    assert hit.sum() > 100
    assert np.all(np.abs(mu_o[hit] - mu[hit]) <= 4 * np.spacing(mu[hit]))
    assert np.all(s2[hit] == F(f) * sig_max) and np.all(a == 10) and np.all(b == 10)
    rest = ~hit
    assert np.all(mu_o[rest] == F((F(dmin) + F(dmax)) / F(2))) and np.all(s2[rest] == sig_max)
    assert np.all(cv[interior] == ob.UPDATE)
    # two source points on one target pixel: the nearer wins
    c2 = np.zeros((H, W), np.int32)
    c2[23, 31] = c2[23, 32] = ob.CONVERGED
    m2 = np.full((H, W), 2.0, F)
    m2[23, 32] = 1.25
    tiny = (1.0, -1.0, 5.0, 5.0)    # 11 x 11 view of focal length 1: both rays land on its centre pixel
    z, n = po.prior_splat(m2, c2, cam, I, (11, 11), tiny, I, dmin, dmax)
    assert n == 2 and (z != EMPTY).sum() == 1
    assert abs(float(z[5, 5].view(F)) - 1.25) <= 4 * np.spacing(F(1.25))
    # dropped: behind the camera, outside [min, max], outside the image
    behind = _pose(np.diag([-1.0, 1.0, -1.0]), [0, 0, 0])
    assert po.prior_splat(mu, conv, cam, I, (W, H), cam, behind, dmin, dmax)[1] == 0
    assert po.prior_splat(mu, conv, cam, I, (W, H), cam, I, 2.5, 3.0)[1] == 0
    assert po.prior_splat(mu, conv, cam, I, (W, H), cam, I, 0.1, 0.9)[1] == 0
    aside = _pose(np.eye(3), [-100.0, 0, 0])
    assert po.prior_splat(mu, conv, cam, I, (W, H), cam, aside, dmin, 1e6)[1] == 0
    # a source without CONVERGED seeds gives exactly the uniform initialisation
    none = po.propagate_prior(mu, np.zeros_like(conv), cam, I, (W, H), cam, I, patch, dmin, dmax, f)
    uniform = po.prior_apply(np.full((H, W), EMPTY, np.uint32), patch, dmin, dmax, f)
    for got, want in zip(none, uniform):
        assert np.array_equal(got, want)
    assert np.all(uniform[1] == sig_max) and np.all(uniform[0] == F((F(dmin) + F(dmax)) / F(2)))
    border = np.zeros((H, W), bool)
    border[:patch, :] = border[:, :patch] = border[H - patch:, :] = border[:, W - patch:] = True
    assert np.array_equal(uniform[4] == ob.BORDER, border)


# ------------------------------------------------------------------ GPU: the product
def _snap(g):
    return {"conv": g.downloadConvergence(), "mu": g.downloadDepthmap(), "sigma_sq": g.downloadSigmaSq(),
            "a": g.downloadA(), "b": g.downloadB()}


def _same(A, B, what):
    for name in ("conv", "mu", "sigma_sq", "a", "b"):
        assert np.array_equal(A[name], B[name]), f"{what}: {name} differs at {(A[name] != B[name]).sum()} pixels"


def _source(seq, n_updates, variant="staged", patch=5, frames=None):
    import rpg_open_remode_b200 as rmd
    g = rmd.SeedMatrix(seq.width, seq.height, rmd.PinholeCamera(*seq.camera), patch_side=patch)
    g.setOption(rmd.OPT_KERNEL_VARIANT, rmd.VARIANT_DIRECT if variant == "direct" else rmd.VARIANT_STAGED)
    if variant == "seed":
        g.setOption(rmd.OPT_SEED_MODE_PCT, 100)
    frames = frames or [seq.frame(k, want_depth=(k == 0)) for k in range(n_updates + 1)]
    f0 = frames[0]
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    g.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    for k in range(1, n_updates + 1):
        g.update(frames[k].image, frames[k].T_cam_world)
    return g, frames, dmin, dmax


@pytest.mark.gpu
@pytest.mark.parametrize("size,n,variant,patch,dst", [
    ((320, 240), 30, "staged", 5, None),
    ((320, 240), 100, "direct", 5, None),
    ((320, 240), 100, "seed", 5, None),
    ((320, 240), 30, "direct", 7, None),
    ((640, 480), 100, "staged", 7, None),
    ((640, 480), 30, "seed", 5, None),
    ((640, 480), 100, "staged", 5, (320, 240)),
])
def test_product_prior_equals_oracle(size, n, variant, patch, dst):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = size
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0400 + W + n)
    src, frames, dmin, dmax = _source(seq, n, variant, patch)
    mu_s, conv_s = src.downloadDepthmap(), src.downloadConvergence()
    assert (conv_s == 1).sum() > 0.02 * W * H
    K = n + 1
    fK = seq.frame(K)
    dw, dh = dst or size
    dcam = synth.dataset_camera(dw, dh)
    img = fK.image if dst is None else synth.SyntheticSequence(dw, dh, seed=1).frame(0).image
    # a narrower range on the resized case: part of the points fall outside it
    lo, hi = (dmin, dmax) if dst is None else (dmin, 0.5 * (dmin + dmax))
    f = 1 / 16
    g = rmd.SeedMatrix(dw, dh, rmd.PinholeCamera(*dcam), patch_side=patch)
    g.setReferenceImage(img, fK.T_cam_world, lo, hi)
    g.propagatePriorFrom(src, f)
    got = _snap(g)
    cam = [float(F(c)) for c in seq.camera]
    want = po.propagate_prior(mu_s, conv_s, cam, ob.se3_inv(frames[0].T_cam_world), (dw, dh),
                              [float(F(c)) for c in dcam], fK.T_cam_world, patch, lo, hi, f)
    _same(got, dict(zip(("mu", "sigma_sq", "a", "b", "conv"), want)), f"{size} {n} {variant} p{patch} -> {dw}x{dh}")
    prior = (got["sigma_sq"] != got["sigma_sq"][0, 0]) & (got["conv"] != rmd.ConvergenceStates.BORDER)
    assert prior.sum() > 0.01 * dw * dh
    # the source is untouched and can still be updated
    assert np.array_equal(src.downloadDepthmap(), mu_s)
    src.update(fK.image, fK.T_cam_world)
    src.sync()


@pytest.mark.gpu
def test_in_place_and_cross_handle_forms_agree():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, n, f = 320, 240, 40, 1 / 16
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0410)
    frames = [seq.frame(k, want_depth=(k == 0)) for k in range(n + 4)]
    dmin, dmax = float(frames[0].depth.min()), float(frames[0].depth.max())
    cam = rmd.PinholeCamera(*seq.camera)
    fK = frames[n + 1]
    dev = rmd.DeviceImage(W, H, "float32")
    dev.setDevData(fK.image)
    cases = ("float", "u8 undistorted", "device")
    for case in cases:
        handles = [rmd.SeedMatrix(W, H, cam) for _ in range(3)]
        A, B, C = handles
        if case == "u8 undistorted":
            for g in handles:
                g.initUndistortionMap(0.05, -0.02, 0.001, 0.0005)
        key = (lambda fr: fr.image_u8) if case == "u8 undistorted" else (lambda fr: fr.image)
        for g in (A, B):
            g.setReferenceImage(key(frames[0]), frames[0].T_cam_world, dmin, dmax)
            for k in range(1, n + 1):
                g.update(key(frames[k]), frames[k].T_cam_world)
        _same(_snap(A), _snap(B), f"{case}: identical sources")
        A.setPriorPropagation(f)
        if case == "device":
            A.setReferenceImageDevice(dev.data, dev.pitch, fK.T_cam_world, dmin, dmax)
        else:
            A.setReferenceImage(key(fK), fK.T_cam_world, dmin, dmax)
        C.setReferenceImage(key(fK), fK.T_cam_world, dmin, dmax)
        C.propagatePriorFrom(B, f)
        SA, SC = _snap(A), _snap(C)
        _same(SA, SC, case)
        assert (SA["sigma_sq"] != SA["sigma_sq"][0, 0]).sum() > 0.01 * W * H, case
        assert np.array_equal(A.downloadSumTempl(), C.downloadSumTempl())
        # both keyframes go on identically
        for k in (n + 2, n + 3):
            A.update(key(frames[k]), frames[k].T_cam_world)
            C.update(key(frames[k]), frames[k].T_cam_world)
        _same(_snap(A), _snap(C), f"{case}, after two updates")


@pytest.mark.gpu
def test_default_is_unchanged():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0420)
    src, frames, dmin, dmax = _source(seq, 40)
    fK = seq.frame(41)
    off = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera))
    off.setPriorPropagation(0.25)
    off.setPriorPropagation(0.0)
    for g in (src, off):
        if g is off:
            g.setReferenceImage(frames[0].image, frames[0].T_cam_world, dmin, dmax)
            for k in range(1, 41):
                g.update(frames[k].image, frames[k].T_cam_world)
        g.setReferenceImage(fK.image, fK.T_cam_world, dmin, dmax)
    fresh = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera))
    fresh.setReferenceImage(fK.image, fK.T_cam_world, dmin, dmax)
    F0 = _snap(fresh)
    for g in (src, off):
        _same(_snap(g), F0, "option off")
        assert np.array_equal(g.downloadSumTempl(), fresh.downloadSumTempl())
        assert np.array_equal(g.downloadConstTemplDenom(), fresh.downloadConstTemplDenom())
    # a source without CONVERGED seeds: a successful no-op
    empty = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera))
    empty.setReferenceImage(frames[0].image, frames[0].T_cam_world, dmin, dmax)
    fresh.propagatePriorFrom(empty, 0.5)
    _same(_snap(fresh), F0, "empty source")


@pytest.mark.gpu
def test_organisations_agree_from_a_propagated_prior():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    W, H, n, N = 320, 240, 30, 25
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0430)
    src, frames, dmin, dmax = _source(seq, n)
    later = [seq.frame(k, want_depth=False) for k in range(n + 1, n + 2 + N)]
    fK = later[0]
    cam = rmd.PinholeCamera(*seq.camera)

    def target(variant):
        g = rmd.SeedMatrix(W, H, cam)
        g.setOption(rmd.OPT_KERNEL_VARIANT, variant)
        g.setReferenceImage(fK.image, fK.T_cam_world, dmin, dmax)
        g.propagatePriorFrom(src, 1 / 16)
        return g

    staged, direct = target(rmd.VARIANT_STAGED), target(rmd.VARIANT_DIRECT)
    many = [target(rmd.VARIANT_STAGED) for _ in range(8)]
    for fr in later[1:]:
        staged.update(fr.image, fr.T_cam_world)
        direct.update(fr.image, fr.T_cam_world)
        rmd.SeedMatrix.updateMany(many, fr.image, fr.T_cam_world)
    S = _snap(staged)
    assert (S["conv"] == 1).sum() > 0.02 * W * H
    _same(_snap(direct), S, "direct")
    for i, g in enumerate(many):
        _same(_snap(g), S, f"updateMany keyframe {i}")
        assert g.getConvergedCount() == staged.getConvergedCount() == int((S["conv"] == 1).sum())


@pytest.mark.gpu
def test_error_codes():
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    INVALID, NOT_INIT = -1, -2
    W, H = 160, 120
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0440)
    cam = rmd.PinholeCamera(*seq.camera)
    f0, f1 = seq.frame(0), seq.frame(1, want_depth=False)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    src, dst = rmd.SeedMatrix(W, H, cam), rmd.SeedMatrix(W, H, cam)

    def code(fn, *args):
        with pytest.raises(rmd.RmdError) as e:
            fn(*args)
        return e.value.code

    assert code(dst.propagatePriorFrom, src, 0.5) == NOT_INIT          # dst has no reference
    dst.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    assert code(dst.propagatePriorFrom, src, 0.5) == NOT_INIT          # src has no reference
    src.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    for bad in (0.0, -0.5, 1.5, float("nan")):
        assert code(dst.propagatePriorFrom, src, bad) == INVALID, bad
    for bad in (-0.5, 1.5, float("nan")):
        assert code(dst.setPriorPropagation, bad) == INVALID, bad
    assert code(dst.propagatePriorFrom, dst, 0.5) == INVALID          # src == dst
    dst.propagatePriorFrom(src, 1.0)
    dst.update(f1.image, f1.T_cam_world)
    assert code(dst.propagatePriorFrom, src, 0.5) == NOT_INIT          # dst updated since its reference
    dst.setReferenceImage(f1.image, f1.T_cam_world, dmin, dmax)
    dst.propagatePriorFrom(src, 0.5)                                    # ... until the next one
    if rmd.device_count() >= 2:
        other = rmd.SeedMatrix(W, H, cam, device=1)
        other.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
        assert code(dst.propagatePriorFrom, other, 0.5) == INVALID    # different devices
    # KeyframeSet: the prior must come from another live slot
    from rpg_open_remode_b200 import node
    ks = node.KeyframeSet(W, H, cam, n=2)
    with pytest.raises(ValueError):
        ks.setReferenceImage(1, f0.image, f0.T_cam_world, dmin, dmax, prior_from=0)
    ks.setReferenceImage(0, f0.image, f0.T_cam_world, dmin, dmax)
    with pytest.raises(ValueError):
        ks.setReferenceImage(0, f0.image, f0.T_cam_world, dmin, dmax, prior_from=0)
    ks.update(f1.image, f1.T_cam_world)
    ks.setReferenceImage(1, f1.image, f1.T_cam_world, dmin, dmax, prior_from=0)
    assert ks.update(f1.image, f1.T_cam_world) == 2


@pytest.mark.gpu
def test_depthmap_node_forwards_the_option():
    """DepthmapNode re-keyframes through Depthmap.setReferenceImage; with the option on, the new keyframe starts
    from the old one's converged seeds."""
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import node, synth
    W, H = 320, 240
    seq = synth.SyntheticSequence(W, H, seed=0x5EED0450)
    fx, fy, cx, cy = seq.camera
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    dm = rmd.Depthmap(W, H, fx, cx, fy, cy)
    dm.setPriorPropagation(1 / 16)
    nd = node.DepthmapNode(dm)
    k, keyframes = 0, 0
    while keyframes < 2 and k < 150:
        fr = seq.frame(k, want_depth=False)
        was = nd.state_
        nd.denseInputCallback(fr.image_u8, rmd.SE3(fr.T_world_cam.reshape(12)), dmin, dmax)
        keyframes += was == node.TAKE_REFERENCE_FRAME
        k += 1
    assert keyframes == 2
    s2 = dm.seeds_.downloadSigmaSq()
    sig_max = F(F(F(dmax) - F(dmin)) ** 2) / F(36)
    assert (s2 == F(F(1 / 16) * sig_max)).sum() > 0.01 * W * H


# ------------------------------------------------------------------ GPU: what the prior is for
# Bars measured on an H100 SXM 80 GB (DESIGN.md 5): the prior must not make the second keyframe converge later,
# converge fewer seeds or be less accurate, beyond these tolerances.
FRAMES_SLACK = 1          # frames to 10 % converged: with <= without + this
COUNT_RATIO = 0.95        # converged seeds after M frames: with >= this x without
ERROR_RATIO = 1.10        # median |mu - ground truth| of the converged seeds: with <= this x without


def _second_keyframe(seq, f, M, max_frames=120):
    """Keyframe 0, re-keyframe by the node's rule (10 % converged or 0.5 m), then M frames of the second
    keyframe.  Returns (prior statistics, frames to 10 % converged, converged count, median error)."""
    import rpg_open_remode_b200 as rmd
    W, H = seq.width, seq.height
    g = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera))
    g.setPriorPropagation(f)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    g.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    k = 0
    while True:
        k += 1
        fr = seq.frame(k, want_depth=False)
        g.update(fr.image, fr.T_cam_world)
        if 100.0 * g.getConvergedCount() / (W * H) > 10.0 or g.getDistFromRef() > 0.5 or k >= max_frames:
            break
    fK = seq.frame(k + 1)
    g.setReferenceImage(fK.image, fK.T_cam_world, dmin, dmax)
    S = _snap(g)
    interior = S["conv"] != rmd.ConvergenceStates.BORDER
    prior = interior & (S["sigma_sq"] != S["sigma_sq"].max())
    good = prior & (np.abs(S["mu"] - fK.depth) <= 0.01 * (dmax - dmin))
    stats = {"keyframe_switch_frame": k, "prior_share": float(prior.sum() / interior.sum()),
             "prior_within_1pct_share": float(good.sum() / max(1, prior.sum()))}
    to_thresh = None
    for j in range(1, M + 1):
        fr = seq.frame(k + 1 + j, want_depth=False)
        g.update(fr.image, fr.T_cam_world)
        if to_thresh is None and 100.0 * g.getConvergedCount() / (W * H) > 10.0:
            to_thresh = j
    S = _snap(g)
    conv = S["conv"] == 1
    err = float(np.median(np.abs(S["mu"] - fK.depth)[conv])) if conv.any() else float("inf")
    return stats, (to_thresh or M + 1), int(conv.sum()), err


@pytest.mark.gpu
@pytest.mark.parametrize("size,seed", [((320, 240), 0x5EED0001), ((640, 480), 0x5EED0002)])
def test_prior_speeds_up_the_next_keyframe(size, seed):
    import rpg_open_remode_b200 as rmd
    from rpg_open_remode_b200 import synth
    seq = synth.SyntheticSequence(*size, seed=seed)
    M = 40
    s_on, n_on, c_on, e_on = _second_keyframe(seq, rmd.PRIOR_SIGMA_SQ_FRAC, M)
    s_off, n_off, c_off, e_off = _second_keyframe(seq, 0.0, M)
    print(f"\n{size}: switch at frame {s_on['keyframe_switch_frame']}, prior on {100 * s_on['prior_share']:.1f} % of "
          f"the interior, {100 * s_on['prior_within_1pct_share']:.1f} % of those within 1 % of the range | frames to "
          f"10 %: {n_on} with, {n_off} without | after {M} frames: {c_on} / {c_off} converged, median error "
          f"{e_on:.5f} / {e_off:.5f} m")
    assert s_off["prior_share"] == 0.0 and s_on["prior_share"] > 0.05
    assert n_on <= n_off + FRAMES_SLACK
    assert c_on >= COUNT_RATIO * c_off
    assert e_on <= ERROR_RATIO * e_off
