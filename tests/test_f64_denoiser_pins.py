"""Pins of the float64 TV-L1 denoiser model (tests/f64_denoiser.py), without a GPU.

* The IEEE CPU oracle's iterates k = 0 ... 40 pass the chain check with the IEEE error model (QVGA filter state and
  ragged sizes down to 1 x 1).
* A vectorised numpy-fp32 emulation of the kernel's Jacobi sweep (FMA forms, rsqrt, a * rcp(b) divisions) passes
  with the fast-math error model.
* Seven planted bugs in that emulation are caught, each by a reported number of pixels.
* The bound is not vacuous: its median at k = 200 is far below the old 1e-4 * range end-of-run bar.
"""
import numpy as np
import pytest

import f64_denoiser as fd
import oracle_binding as ob

F32 = np.float32
LAM = 0.5


def _filter_state(seq, n_updates):
    """(mu, sigma^2, a, b, range) of the CPU oracle's depth filter after `n_updates` frames."""
    f0 = seq.frame(0)
    dmin, dmax = float(f0.depth.min()), float(f0.depth.max())
    o = ob.OracleSeeds(seq.width, seq.height, *seq.camera, patch=5)
    o.set_reference(f0.image, f0.T_cam_world, dmin, dmax)
    for k in range(1, n_updates + 1):
        f = seq.frame(k, want_depth=False)
        o.update(f.image, f.T_cam_world)
    return (o.mu.copy(), o.sigma_sq.copy(), o.a.copy(), o.b.copy()), dmax - dmin


def _random_state(W, H, seed, rng_d=2.0):
    r = np.random.default_rng(seed)
    mu = (1.0 + rng_d * r.random((H, W))).astype(F32)
    s2 = (rng_d ** 2 / 36 * r.random((H, W)) ** 3).astype(F32)
    a = (10 * r.random((H, W)) + 0.5).astype(F32)
    b = (10 * r.random((H, W)) + 0.5).astype(F32)
    return (mu, s2, a, b), rng_d


@pytest.fixture(scope="module")
def qvga_state(qvga_sequence):
    return _filter_state(qvga_sequence, 15)


@pytest.fixture(scope="module")
def small_state(small_sequence):
    return _filter_state(small_sequence, 12)


# ------------------------------------------------------------------ numpy-fp32 emulation of the kernel

def _fma(a, b, c):
    # float64 holds a * b exactly; the one addition is then rounded twice (to float64, to float32), which may cost
    # a last-bit difference against a true FMA -- this is an emulation under test, not a bit-exact replica
    return (a.astype(np.float64) * b + c).astype(F32)


def _rcp(x):
    with np.errstate(divide="ignore"):
        return (1.0 / x.astype(np.float64)).astype(F32)


def emulate(inputs, depth_range, lam, K, bug=None):
    """The kernel's Jacobi sweep in numpy fp32 (csrc/denoiser.cu operation forms).  Returns [u_0, ..., u_K].
    `bug` plants one of the defects the chain check must catch."""
    mu, s2, a, b = (np.asarray(v, F32) for v in inputs)
    H, W = mu.shape
    c = fd.constants(lam, depth_range)
    sigma, tau, tl, lss = F32(c["sigma"]), F32(c["tau"]), F32(c["tl"]), F32(c["lss"])
    theta = F32(1.0) if bug == "theta1" else F32(0.5)
    with np.errstate(all="ignore"):
        E = a * _rcp(a + b)
        gp = _fma(E, s2, (F32(1) - E) * lss) * _rcp(np.asarray(lss))
        g = gp if bug == "no_clamp" else np.fmax(gp, F32(1))
    x = np.arange(W)[None, :]
    y = np.arange(H)[:, None]
    e_own = x >= W - 1
    if bug == "east_pair":        # the pair's second pixel (odd column) tests against W - 2
        e_own = np.where(x % 2 == 1, x >= W - 2, e_own)
    xe = np.where(e_own, x, x + 1)
    ys = np.minimum(y + 1, H - 1)
    u, uh = mu.copy(), mu.copy()
    uh_old = uh
    px = np.zeros_like(mu)
    py = np.zeros_like(mu)
    out = [u.copy()]
    for it in range(K):
        with np.errstate(all="ignore"):
            uh_e = uh[:, xe[0]]
            if bug == "stale_seam" and it % 8 == 7:
                # a halo one pixel short: the last iteration of a launch reads the tile seam's east column one
                # iteration old
                seam = (x[0] % 48 == 47) & (x[0] < W - 1)
                uh_e[:, seam] = uh_old[:, xe[0]][:, seam]
            uh_s = uh[ys[:, 0], :]
            centre = uh if bug == "uhead_centre" else u
            gx = uh_e - centre
            gy = uh_s - centre
            tx = _fma(g * gx, sigma, px)
            ty = _fma(g * gy, sigma, py)
            len_sq = _fma(tx, tx, ty * ty)
            if bug == "proj_sq":
                inv = np.where(len_sq > 1, _rcp(len_sq), F32(1))
            else:
                inv = np.where(len_sq > 1, (1.0 / np.sqrt(len_sq.astype(np.float64))).astype(F32), F32(1))
            px, py = tx * inv, ty * inv
            cx = np.where((x != 0) & (x >= W - 1), F32(0), px)
            wx = np.where(x == 0, F32(0), np.roll(px, 1, axis=1))
            last_row = (y != 0) & (y >= H - 1)
            cy = py if bug == "last_row_py" else np.where(last_row, F32(0), py)
            ny = np.where(y == 0, F32(0), np.roll(py, 1, axis=0))
            div = ((cx - wx) + cy) - ny
            temp = _fma(tau * g, div, u)
            dx = temp - mu
            nu = np.where(dx > tl, temp - tl, np.where(dx < -tl, temp + tl, mu))
            uh_old = uh
            uh = _fma(np.full_like(nu, theta), nu - u, nu)
            u = nu
        out.append(u.copy())
    return out


BUGS = ["east_pair", "uhead_centre", "theta1", "last_row_py", "stale_seam", "no_clamp", "proj_sq"]


# ------------------------------------------------------------------ the IEEE oracle

def _oracle_chain(inputs, depth_range, lam, K):
    mu, s2, a, b = inputs
    for k in range(K + 1):
        yield ob.denoise(mu, s2, a, b, depth_range, lam, k)


def test_oracle_chain_qvga(qvga_state):
    inputs, rng_d = qvga_state
    rep = fd.check_chain(inputs, _oracle_chain(inputs, rng_d, LAM, 40), rng_d, LAM, fast=False)
    print("\nIEEE oracle QVGA:", rep.summary())
    assert rep.n_fail == 0, rep.first
    assert rep.n_ambiguous == 0
    assert rep.ratio_max > 0          # the check looked at finite pixels


@pytest.mark.parametrize("W,H", [(1, 1), (1, 7), (2, 2), (3, 1), (3, 2), (5, 3), (49, 25), (97, 2), (2, 50)])
def test_oracle_chain_ragged(W, H):
    inputs, rng_d = _random_state(W, H, seed=W * 1000 + H)
    rep = fd.check_chain(inputs, _oracle_chain(inputs, rng_d, LAM, 40), rng_d, LAM, fast=False)
    print(f"\nIEEE oracle {W}x{H}:", rep.summary())
    assert rep.n_fail == 0, rep.first
    assert rep.n_ambiguous == 0


# ------------------------------------------------------------------ the emulation and its planted bugs

@pytest.mark.parametrize("size", [(160, 120), (97, 49), (1, 3), (3, 1)])
def test_emulation_passes(small_state, size):
    if size == (160, 120):
        inputs, rng_d = small_state
    else:
        inputs, rng_d = _random_state(*size, seed=7)
    rep = fd.check_chain(inputs, emulate(inputs, rng_d, LAM, 40), rng_d, LAM, fast=True)
    print(f"\nemulation {size}:", rep.summary())
    assert rep.n_fail == 0, rep.first
    assert rep.n_ambiguous == 0


def test_planted_bugs_are_caught(small_state):
    """Each planted defect fails the chain check; the number of failing (k, pixel) pairs is reported.  The
    inputs are the small filter state cropped to an odd width (so the last pixel pair is split) with a seam column
    inside, and a random state of the same width whose last rows are not flat (the filter state's are)."""
    (mu, s2, a, b), rng_d = small_state
    crop = tuple(np.ascontiguousarray(v[:, :97]) for v in (mu, s2, a, b))
    cases = [(crop, rng_d), _random_state(97, 49, seed=11)]
    caught = {}
    for bug in BUGS:
        n = []
        for inputs, r in cases:
            rep = fd.check_chain(inputs, emulate(inputs, r, LAM, 24, bug=bug), r, LAM, fast=True)
            n.append(rep.n_fail)
        caught[bug] = sum(n)
        print(f"\nplanted {bug:13s}: {n[0]} + {n[1]} failing pixel-iterates (filter state 97x120 + random 97x49)")
    missed = [b for b, n in caught.items() if n == 0]
    assert not missed, f"planted bugs not caught: {missed} ({caught})"


def test_bound_is_not_vacuous(qvga_state):
    """Median bound at k = 200 on the emulated kernel, against the old end-of-run bar 1e-4 * range."""
    inputs, rng_d = qvga_state
    rep = fd.check_chain(inputs, emulate(inputs, rng_d, LAM, 200), rng_d, LAM, fast=True)
    med = rep.bound_median[-1]
    print(f"\nQVGA K=200: {rep.summary()}; median bound / (1e-4 range) = {med / (1e-4 * rng_d):.3g}")
    assert rep.n_fail == 0, rep.first
    assert 0 < med < 0.05 * 1e-4 * rng_d
