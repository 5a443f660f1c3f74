"""Every pixel of every TV-L1 denoiser iterate against the float64 model (tests/f64_denoiser.py).

The denoiser hands out u after k iterations and is deterministic, so each case runs k = 0 ... K as separate calls
and checks the chain: the model follows the kernel's own u_{k-1} and u_head_{k-1}, tracks the dual with a bound
that grows linearly in k, and requires every u_k inside its per-pixel bound, u = mu bit for bit where the threshold's
middle branch is decided, and NaN / inf where they must be.  The risky places of the temporally blocked kernel
(48 x 24 tiles, 8-pixel halo, 8 iterations per launch, pixel pairs) are covered by the shapes and by K = 17
(two full launches and a short one).
"""
import numpy as np
import pytest

import f64_denoiser as fd
import rpg_open_remode_b200 as rmd
from rpg_open_remode_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
LAM = 0.5


def _check(inputs, chain, rng_d, lam, what, max_amb_frac=1e-3):
    rep = fd.check_chain(inputs, chain, rng_d, lam, fast=True)
    n = inputs[0].size
    print(f"\n{what}: {rep.summary()}")
    assert rep.n_fail == 0, (what, rep.first)
    assert rep.n_ambiguous <= max(8, max_amb_frac * n), (what, rep.n_ambiguous)
    return rep


def _seed_chain(den, g, lam, K):
    for k in range(K + 1):
        yield den.denoiseSeeds(g, lam, k)


def _planar_chain(den, imgs, lam, K):
    for k in range(K + 1):
        yield den.denoise(*imgs, lam, k)


def _upload(inputs):
    out = []
    for v in inputs:
        H, W = v.shape
        d = rmd.DeviceImage(W, H, "float32")
        d.setDevData(v)
        out.append(d)
    return out


def _filter(W, H, n_updates, trap=0, seed=0x5EED0001):
    seq = synth.SyntheticSequence(W, H, seed=seed)
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    g = rmd.SeedMatrix(W, H, rmd.PinholeCamera(*seq.camera))
    g.setReferenceImage(f0.image, f0.T_cam_world, dmin, dmax)
    for k in range(1, n_updates + 1):
        f = seq.frame(k, want_depth=False)
        g.update(f.image, f.T_cam_world)
    if trap:
        # trapped seeds: sigma^2 NaN (the filter's own state after sigma^2 went <= 0)
        s2 = g.downloadSigmaSq()
        r = np.random.default_rng(trap)
        s2[r.integers(0, H, trap), r.integers(0, W, trap)] = np.nan
        g.uploadState(rmd.FIELD_SIGMA_SQ, s2)
    inputs = (g.downloadDepthmap(), g.downloadSigmaSq(), g.downloadA(), g.downloadB())
    return g, inputs, dmax - dmin


@pytest.mark.parametrize("W,H,n_updates,K", [(320, 240, 15, 200), (640, 480, 15, 200), (1280, 720, 10, 40),
                                             (1920, 1080, 8, 40)], ids=["qvga", "vga", "720p", "1080p"])
def test_filter_output(W, H, n_updates, K):
    g, inputs, rng_d = _filter(W, H, n_updates, trap=64)
    assert np.isnan(inputs[1]).sum() >= 64
    den = rmd.DepthmapDenoiser(W, H)
    den.setLargeSigmaSq(rng_d)
    rep = _check(inputs, _seed_chain(den, g, LAM, K), rng_d, LAM, f"filter {W}x{H} K={K}")
    print(f"  median bound at K / (1e-4 range) = {rep.bound_median[-1] / (1e-4 * rng_d):.3g}")


def _random_state(W, H, seed, rng_d=2.0):
    r = np.random.default_rng(seed)
    mu = (1.0 + rng_d * r.random((H, W))).astype(F32)
    s2 = (rng_d ** 2 / 36 * r.random((H, W)) ** 3).astype(F32)
    a = (10 * r.random((H, W)) + 0.5).astype(F32)
    b = (10 * r.random((H, W)) + 0.5).astype(F32)
    return [mu, s2, a, b], rng_d


@pytest.mark.parametrize("W", [1, 2, 3, 47, 48, 49, 95, 96, 97])
def test_shapes_around_the_tile(W):
    """Both sides of the 48 x 24 tile, odd widths (split pixel pairs), widths that leave row padding."""
    for H in (1, 2, 23, 24, 25):
        inputs, rng_d = _random_state(W, H, seed=W * 100 + H)
        den = rmd.DepthmapDenoiser(W, H)
        den.setLargeSigmaSq(rng_d)
        imgs = _upload(inputs)
        _check(inputs, _planar_chain(den, imgs, LAM, 17), rng_d, LAM, f"{W}x{H} K=17")


PW, PH = 101, 53     # three tile columns (seams at 48, 96), three tile rows (seams at 24, 48)


def _planar_cases():
    base, rng_d = _random_state(PW, PH, seed=99)
    cases = []

    def case(name, mu=None, s2=None, a=None, b=None, rng=rng_d, lam=LAM, K=17):
        v = [np.array(x if x is not None else y, F32) for x, y in zip((mu, s2, a, b), base)]
        cases.append(pytest.param(v, rng, lam, K, id=name))

    flat = np.full((PH, PW), 2.0, F32)
    imp = flat.copy()
    for (y, x) in ((0, 0), (0, PW - 1), (PH - 1, 0), (PH - 1, PW - 1), (23, 47), (24, 48), (24, 47), (23, 48),
                   (47, 95), (48, 96), (10, PW - 1), (PH - 1, 30), (PH - 2, PW - 2)):
        imp[y, x] = 2.0 + rng_d * (0.5 if (x + y) % 2 else -0.5)
    case("impulses", mu=imp)
    yy, xx = np.mgrid[0:PH, 0:PW]
    case("checkerboard", mu=np.where((xx + yy) % 2 == 0, 1.0 + rng_d, 1.0))
    case("constant", mu=flat)
    case("constant_lambda0", mu=flat, lam=0.0)
    sp = base[0].copy()
    sp[5, 5], sp[30, 47], sp[PH - 1, PW - 1] = np.nan, np.inf, -np.inf
    sp[12, 60], sp[40, 20] = 1e37, -1e37
    sp[20, 90] = 3e38
    sp[2, 48], sp[3, 48], sp[24, 24] = 1e-40, -1e-40, 1e-39
    case("special_mu", mu=sp)
    s2 = base[1].copy()
    s2[::7, ::5] = np.nan
    s2[1::7, ::5] = 0.0
    s2[2::7, ::5] = -1.0
    s2[3::7, ::5] = np.inf
    case("special_sigma_sq", s2=s2)
    a, b = base[2].copy(), base[3].copy()
    a[::6, ::4], b[::6, ::4] = 1.0, -1.0
    a[3::6, ::4], b[3::6, ::4] = 0.0, 0.0
    case("a_plus_b_zero", a=a, b=b)
    r = np.random.default_rng(5)
    case("tiny_range", mu=(1.0 + 1e-3 * r.random((PH, PW))), s2=(1e-7 * r.random((PH, PW))), rng=1e-3)
    for lam in (0.0, 0.5, 1e4):
        case(f"lambda_{lam:g}", lam=lam, K=24)
    return cases


@pytest.mark.parametrize("inputs,rng_d,lam,K", _planar_cases())
def test_planar_inputs(inputs, rng_d, lam, K):
    den = rmd.DepthmapDenoiser(PW, PH)
    den.setLargeSigmaSq(rng_d)
    imgs = _upload(inputs)
    rep = _check(inputs, _planar_chain(den, imgs, lam, K), rng_d, lam, f"planar lam={lam} range={rng_d}")
    if lam >= 1e4 or np.ptp(inputs[0][np.isfinite(inputs[0])]) == 0:
        # tau * lambda far above every step, or p = 0 throughout: u = mu bit for bit at every k
        assert min(rep.middle[1:]) == PW * PH


def test_organisations_agree_bit_for_bit():
    """denoiseSeeds, planar denoise and denoiseSeedsToDevice into a wider-pitched image give the same bits, on the
    handle's own stream and on a user stream."""
    import torch
    W, H = 161, 97
    g, inputs, rng_d = _filter(W, H, 8, seed=0x5EED0042)
    den = rmd.DepthmapDenoiser(W, H)
    den.setLargeSigmaSq(rng_d)
    wide = rmd.DeviceImage(W + 45, H, "float32")
    for K in (0, 1, 8, 17, 40):
        a = den.denoiseSeeds(g, LAM, K)
        b = den.denoise(g.getMu(), g.getSigmaSq(), g.getA(), g.getB(), LAM, K)
        wide.zero()
        den.denoiseSeedsToDevice(g, wide.data, wide.pitch, LAM, K)
        den.sync()
        c = wide.getDevData()[:, :W]
        assert a.view(np.int32).tolist() == b.view(np.int32).tolist() == c.view(np.int32).tolist(), K
        assert not wide.getDevData()[:, W:].any()       # nothing written beyond the width
        s = torch.cuda.Stream()
        den.setStream(s.cuda_stream)
        d = den.denoiseSeeds(g, LAM, K)
        den.setStream(0)
        assert np.array_equal(a.view(np.int32), d.view(np.int32)), K
    _check(inputs, _seed_chain(den, g, LAM, 17), rng_d, LAM, f"organisations {W}x{H}")
