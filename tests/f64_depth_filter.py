"""Float64 restatement of ONE fused depth-filter update, with per-seed error bounds.

Test infrastructure: vectorised over seeds with numpy, written from the reference's sources (cited per step, paths
relative to the reference tree), not from csrc/depth_filter_math.cuh.  It restates the operation, not the kernel's
fused multiply-add forms, and derives for every seed how far an fp32 implementation may lie from it:

* the search (src/epipolar_match.cu:38-140) is checked apart from the update.  A 1-ulp difference may flip the
  arg-max to the neighbouring candidate 0.7 px away, after which mu and sigma^2 legitimately differ by a lot, so the
  checker asks whether the implementation's chosen candidate is an eps-arg-max of the float64 scores, with a forward
  error bound eps per candidate;
* the update (src/triangulation.cu:30-68, src/seed_update.cu:40-121) is re-run in float64 from the implementation's
  OWN match, K times with every operation perturbed by its stated maximum relative error; the bound of a field is
  4 x the largest deviation + 4 ulp of the fp32 value, and a branch the draws disagree on marks the seed ambiguous;
* classification (src/seed_check.cu:29-67) marks a seed ambiguous when a threshold quantity lies within its
  perturbation spread of 0.7, epsilon or 0.05.

Parameters as the product sets them (rpg_open_remode_b200/csrc/c_api.cu, finish_set_reference / prepare_update,
after src/seed_matrix.cu:96-104): eta_inlier 0.7, eta_outlier 0.05, epsilon = range / 1000, one_pix_angle =
2 atan2(1, 2 fx) (include/rmd/pinhole_camera.cuh:55-59), search extent 100 px (CMakeLists.txt:53), NCC acceptance
0.5 (src/epipolar_match.cu:131), bilinear weights with 8 fractional bits (DESIGN.md 5.2).
"""
from __future__ import annotations

import numpy as np

UPDATE, CONVERGED, BORDER, DIVERGED, NO_MATCH = 0, 1, 2, 3, 4
U = 2.0 ** -24                    # unit roundoff of fp32
FLT_MIN = float(np.finfo(np.float32).tiny)
FLT_MAX = float(np.finfo(np.float32).max)
STEP = np.float32(0.7)            # src/epipolar_match.cu:88
MAX_EXTENT = 100.0                # RMD_MAX_EXTENT_EPIPOLAR_SEARCH, CMakeLists.txt:53
NCC_ACCEPT = 0.5                  # src/epipolar_match.cu:131
ETA_IN, ETA_OUT = float(np.float32(0.7)), float(np.float32(0.05))

# Stated maximum errors of the operations -use_fast_math turns approximate (PTX ISA, "Floating-point instructions";
# CUDA C++ Programming Guide, "Mathematical functions", intrinsic and single-precision tables).  Relative unless noted.
FAST = {
    "rcp": 2.0 ** -23,            # rcp.approx.ftz.f32: 1 ulp
    "div": 2.0 ** -22,            # x / y under -prec-div=false: 2 ulp
    "rsqrt": 2.0 ** -22.9,        # rsqrt.approx.f32
    "sqrt": 2.0 ** -22.9,         # sqrtf under -prec-sqrt=false: x * rsqrt.approx(x)
    "ex2": 2.0 ** -22.5,          # ex2.approx.ftz.f32
    "sin": 2.0 ** -20.9,          # sin.approx.f32, ABSOLUTE, |x| <= pi
    "acos": 2.0 ** -21,           # acosf: 2 ulp stated; doubled for the approximate sqrt it calls under fast math
}
IEEE = {k: U for k in FAST}       # the CPU oracle: correctly rounded operations (libm within an ulp)


class Arith:
    """Float64 arithmetic over per-seed arrays.  With `rng`, every operation's result is multiplied by (1 + u d),
    u ~ U[-1, 1] per seed, d = 2^-24 for plain fp32 operations and the stated error of approximate ones.  Results
    are held to the fp32 range (overflow to inf; under fast math, flush-to-zero of subnormals) in every draw."""

    def __init__(self, n, fast, rng=None):
        self.n, self.fast, self.rng = n, fast, rng
        self.d = FAST if fast else IEEE

    def _u(self):
        return self.rng.uniform(-1.0, 1.0, self.n)

    def range(self, x):
        x = np.where(np.abs(x) > FLT_MAX, np.copysign(np.inf, x), x)
        if self.fast:
            x = np.where(np.abs(x) < FLT_MIN, 0.0 * x, x)
        return x

    def r(self, x, d=U):
        if self.rng is not None:
            x = x * (1.0 + d * self._u())
        return self.range(x)

    def add(self, x, y): return self.r(x + y)
    def sub(self, x, y): return self.r(x - y)
    def mul(self, x, y): return self.r(x * y)
    def f32(self, x): return self.r(x)

    def rcp(self, x):
        with np.errstate(divide="ignore", invalid="ignore"):
            return self.r(1.0 / x, self.d["rcp"])

    def div(self, x, y):
        # the kernel writes divisions as x * rcp.approx(y); the reference's x / y compiles to the same under fast math
        if self.fast:
            return self.mul(x, self.rcp(y))
        with np.errstate(divide="ignore", invalid="ignore"):
            return self.r(x / y)

    def sqrt(self, x):
        with np.errstate(invalid="ignore"):
            return self.r(np.sqrt(x), self.d["sqrt"])

    def rsqrt(self, x):
        with np.errstate(divide="ignore", invalid="ignore"):
            return self.r(1.0 / np.sqrt(x), self.d["rsqrt"] if self.fast else U)

    def exp(self, x):
        if self.fast:   # __expf: ex2.approx(x * log2(e))
            x = self.mul(x, 1.4426950408889634)
            with np.errstate(over="ignore"):
                return self.r(np.exp2(x), self.d["ex2"])
        with np.errstate(over="ignore"):
            return self.r(np.exp(x))

    def sin(self, x):
        y = np.sin(x)
        if self.rng is not None:
            y = y + (self.d["sin"] if self.fast else U * np.abs(y)) * self._u()
        return self.range(y)

    def acos(self, x):
        with np.errstate(invalid="ignore"):
            return self.r(np.arccos(x), self.d["acos"])

    def pose(self, T):
        """3x4 fp32 pose as 12 per-seed arrays, each entry perturbed at 1 ulp."""
        T = np.asarray(T, np.float32).reshape(12)
        out = []
        for v in T:
            e = np.full(self.n, float(v))
            if self.rng is not None:
                e = e + float(np.spacing(np.abs(v))) * self._u()
            out.append(e)
        return out


class Frame:
    """One update's inputs that are shared by all seeds: images, camera, poses, depth range, patch."""

    def __init__(self, ref, curr, cam, T_curr_ref, min_depth, max_depth, patch=5, tex_frac_bits=8):
        self.ref = np.asarray(ref, np.float32).astype(np.float64)
        self.curr = np.asarray(curr, np.float32).astype(np.float64)
        self.H, self.W = self.ref.shape
        self.P = patch
        self.fx, self.fy, self.cx, self.cy = (float(np.float32(c)) for c in cam)
        self.T_curr_ref = np.asarray(T_curr_ref, np.float32).reshape(3, 4)
        self.T_ref_curr = se3_inv_f32(self.T_curr_ref)
        f32 = np.float32
        self.depth_range = float(f32(max_depth) - f32(min_depth))                # c_api.cu finish_set_reference
        self.epsilon = float(f32(self.depth_range) / f32(1000.0))
        self.one_pix_angle = float(f32(np.arctan2(f32(1.0), f32(2.0) * f32(self.fx))) * f32(2.0))
        self.tex_frac_bits = tex_frac_bits


def se3_inv_f32(T):
    """include/rmd/se3.cuh:81-97 in fp32 with the products and sums in source order."""
    d = np.asarray(T, np.float32).reshape(12)
    r = np.zeros(12, np.float32)
    r[0], r[1], r[2] = d[0], d[4], d[8]
    r[4], r[5], r[6] = d[1], d[5], d[9]
    r[8], r[9], r[10] = d[2], d[6], d[10]
    r[3] = -d[0] * d[3] - d[4] * d[7] - d[8] * d[11]
    r[7] = -d[1] * d[3] - d[5] * d[7] - d[9] * d[11]
    r[11] = -d[2] * d[3] - d[6] * d[7] - d[10] * d[11]
    return r.reshape(3, 4)


def se3_mul_f32(A, B):
    """se3.cuh:146-162 in fp32, source order (T_curr_ref = T_curr_world * T_world_ref, src/seed_matrix.cu:124)."""
    A, B = np.asarray(A, np.float32).reshape(12), np.asarray(B, np.float32).reshape(12)
    t = np.zeros(12, np.float32)
    for row in range(3):
        L = A[4 * row:4 * row + 4]
        for col in range(3):
            t[4 * row + col] = L[0] * B[col] + L[1] * B[4 + col] + L[2] * B[8 + col]
        t[4 * row + 3] = L[3] + L[0] * B[3] + L[1] * B[7] + L[2] * B[11]
    return t.reshape(3, 4)


def ulp32(v):
    v = np.abs(np.asarray(v, np.float64))
    with np.errstate(invalid="ignore", over="ignore"):
        return np.spacing(np.minimum(v, FLT_MAX).astype(np.float32)).astype(np.float64)


def _spread(draws, v0):
    """4 x the largest |draw - exact| + 4 ulp(fp32 value); inf where a draw is not finite."""
    with np.errstate(invalid="ignore"):
        dev = np.max(np.abs(np.stack(draws) - v0), axis=0)
    dev = np.where(np.isfinite(dev), dev, np.inf)
    return 4.0 * dev + 4.0 * ulp32(v0)


# ------------------------------------------------------------------------------------------------ classification

def classify(fr, xs, ys, mu, s2, a, b, prev, trust_conv, draws=32, seed=1):
    """src/seed_check.cu:29-67 per seed.  Returns (state, ambiguous)."""
    n = len(xs)
    W, H, P = fr.W, fr.H, fr.P
    state = np.full(n, UPDATE, np.int32)
    absorb = np.isin(prev, (BORDER, CONVERGED, DIVERGED)) if trust_conv else np.zeros(n, bool)
    border = (xs > W - P - 1) | (ys > H - P - 1) | (xs < P) | (ys < P)                        # :37-42

    def q(ar):
        ab = ar.add(a, b)
        return ar.div(a, ab), ar.div(ar.sub(a, 1.0), ar.sub(ab, 2.0))

    with np.errstate(invalid="ignore", divide="ignore"):
        q_in, q_out = q(Arith(n, True))
        rng = np.random.default_rng(seed)
        d_in = _spread([q(Arith(n, True, rng))[0] for _ in range(draws)], q_in)
        d_out = _spread([q(Arith(n, True, rng))[1] for _ in range(draws)], q_out)
        conv = (q_in > ETA_IN) & (s2 < fr.epsilon)                                          # :54-55
        div = ~conv & (q_out < ETA_OUT)                                                      # :59
        amb = (np.abs(q_in - ETA_IN) <= d_in) | (np.abs(q_out - ETA_OUT) <= d_out)
    state[conv] = CONVERGED
    state[div] = DIVERGED
    state[border] = BORDER
    state[absorb] = prev[absorb]
    amb &= ~border & ~absorb
    return state, amb


# ------------------------------------------------------------------------------------------------ search

def _bearing(ar, fr, u, v):
    """normalize(cam.cam2world(u, v)): pinhole_camera.cuh:40-46, helper_math.h:1309-1313."""
    px, py = ar.div(ar.sub(u, fr.cx), fr.fx), ar.div(ar.sub(v, fr.cy), fr.fy)
    inv = ar.rsqrt(ar.add(ar.add(ar.mul(px, px), ar.mul(py, py)), 1.0))
    return ar.mul(px, inv), ar.mul(py, inv), inv


def _project(ar, fr, T, p):
    """cam.world2cam(T * p): se3.cuh:111-125, pinhole_camera.cuh:48-53."""
    X, Y, Z = (ar.add(ar.add(ar.add(ar.mul(T[4 * r], p[0]), ar.mul(T[4 * r + 1], p[1])), ar.mul(T[4 * r + 2], p[2])),
                      T[4 * r + 3]) for r in range(3))
    return ar.add(ar.div(ar.mul(fr.fx, X), Z), fr.cx), ar.add(ar.div(ar.mul(fr.fy, Y), Z), fr.cy)


def _segment(ar, fr, xs, ys, mu, s2):
    """src/epipolar_match.cu:60-75 and the two defined deviations of DESIGN.md 5.3."""
    T = ar.pose(fr.T_curr_ref)
    sigma = ar.sqrt(s2)
    f = _bearing(ar, fr, xs.astype(np.float64), ys.astype(np.float64))
    scale = lambda d: [ar.mul(c, d) for c in f]
    mean = _project(ar, fr, T, scale(mu))
    lo = _project(ar, fr, T, scale(np.fmax(ar.sub(mu, ar.mul(3.0, sigma)), 0.01)))           # :68-69
    hi = _project(ar, fr, T, scale(ar.add(mu, ar.mul(3.0, sigma))))                          # :70-71
    with np.errstate(invalid="ignore"):
        line = (ar.sub(hi[0], lo[0]), ar.sub(hi[1], lo[1]))
        len_sq = ar.add(ar.mul(line[0], line[0]), ar.mul(line[1], line[1]))
        inv = ar.rsqrt(len_sq)                                                               # :74
        zero = len_sq == 0.0                     # deviation 1: one candidate at the mean projection
        d = [np.where(zero, 0.0, ar.mul(c, inv)) for c in line]
        hl = ar.mul(np.fmin(ar.sqrt(len_sq), MAX_EXTENT), 0.5)                              # :75
        hl = np.where(np.abs(len_sq) < np.inf, hl, np.nan)   # deviation 2: NaN / infinite segment: no candidate
    return mean, d, hl


def segment(fr, xs, ys, mu, s2, fast, draws=32, seed=2):
    """Exact segment and 4 x the spread of its mean, direction and half length over perturbed draws."""
    n = len(xs)
    if fast:   # flush-to-zero of the fp32 inputs
        s2 = np.where(np.abs(s2) < FLT_MIN, 0.0 * s2, s2)
        mu = np.where(np.abs(mu) < FLT_MIN, 0.0 * mu, mu)
    mean, d, hl = _segment(Arith(n, fast), fr, xs, ys, mu, s2)
    rng = np.random.default_rng(seed)
    D = [_segment(Arith(n, fast, rng), fr, xs, ys, mu, s2) for _ in range(draws)]
    with np.errstate(invalid="ignore"):
        d_mean = np.maximum(_spread([x[0][0] for x in D], mean[0]), _spread([x[0][1] for x in D], mean[1]))
        d_dir = np.maximum(_spread([x[1][0] for x in D], d[0]), _spread([x[1][1] for x in D], d[1]))
        d_hl = _spread([x[2] for x in D], hl)
    return mean, d, hl, d_mean, d_dir, d_hl


def comb(hl, max_cand=160):
    """Candidate l values: the reference's fp32 accumulation l = -half_length; l <= half_length; l += 0.7f
    (src/epipolar_match.cu:88).  This is the definition of the positions, so it is restated in fp32.  Each row also
    holds the first l past the end (`has` False there), whose existence an implementation's half length may flip."""
    h32 = hl.astype(np.float32)
    l = -h32
    L = np.full((len(hl), max_cand + 1), np.nan, np.float32)
    live = np.isfinite(h32)
    for k in range(max_cand + 1):
        if not live.any():
            break
        L[live, k] = l[live]
        live &= l <= h32
        l = np.where(live, l + STEP, l)
    L = L.astype(np.float64)
    with np.errstate(invalid="ignore"):
        has = L <= h32[:, None]
    return L, h32.astype(np.float64), has


def _templates(fr, xs, ys):
    P, r = fr.P, fr.P // 2
    dy, dx = np.meshgrid(np.arange(P) - r, np.arange(P) - r, indexing="ij")
    yy = np.clip(ys[:, None, None] + dy, 0, fr.H - 1)
    xx = np.clip(xs[:, None, None] + dx, 0, fr.W - 1)
    return fr.ref[yy, xx]


def _ncc(fr, seed_of, tpl, px, py, shift=None):
    """NCC of every listed candidate, src/epipolar_match.cu:99-123.  The texture unit samples curr at px + d + 0.5
    with 8-bit fixed-point weights (DESIGN.md 5.2): the patch is the (P+1)^2 texel block at floor(px - P/2) with
    weights floor(frac * 256 + 0.5) / 256.  Returns score, its forward error bound and the distance of frac*256 to
    the nearest rounding boundary (x and y).  `shift` = (sx, sy) moves the quantised weights by that many 1/q."""
    P = fr.P
    q = float(1 << fr.tex_frac_bits) if fr.tex_frac_bits > 0 else 0.0
    bx, by = px - (P // 2), py - (P // 2)
    if q > 0:
        tx, ty = np.floor(bx * q + 0.5), np.floor(by * q + 0.5)
        gx, gy = np.abs(bx * q - np.floor(bx * q) - 0.5), np.abs(by * q - np.floor(by * q) - 0.5)
        if shift is not None:
            tx, ty = tx + shift[0], ty + shift[1]
        i0, j0 = np.floor(tx / q), np.floor(ty / q)
        al, be = tx / q - i0, ty / q - j0
    else:
        i0, j0 = np.floor(bx), np.floor(by)
        al, be = bx - i0, by - j0
        gx = gy = np.full(len(px), np.inf)
    i0, j0 = i0.astype(np.int64), j0.astype(np.int64)
    o = np.arange(P + 1)
    v = fr.curr[np.clip(j0[:, None, None] + o[None, :, None], 0, fr.H - 1),
                np.clip(i0[:, None, None] + o[None, None, :], 0, fr.W - 1)]
    al, be = al[:, None, None], be[:, None, None]
    low = v[:, :, :-1] * (1.0 - al) + v[:, :, 1:] * al
    img = low[:, :-1, :] * (1.0 - be) + low[:, 1:, :] * be
    img_abs = np.abs(img)          # |weights| sum to 1 and images are >= 0: the bilinear rounding scale
    t = tpl[seed_of]
    n = P * P
    ax = (1, 2)
    Si, Sii, Sit = img.sum(ax), (img * img).sum(ax), (img * t).sum(ax)
    St, Stt = t.sum(ax), (t * t).sum(ax)
    ctd = n * Stt - St * St
    num = n * Sit - Si * St
    spr = n * Sii - Si * Si
    den = ctd * spr + FLT_MIN
    with np.errstate(invalid="ignore", divide="ignore"):
        score = num / np.sqrt(den)
    # forward error bound of the fp32 evaluation (running sums: gamma_{n+2}; bilinear: 4 roundings per value)
    g, e_img = (n + 2) * U, 4 * U
    A, Aq, Ait = img_abs.sum(ax), (img_abs * img_abs).sum(ax), np.abs(img * t).sum(ax)
    At = np.abs(t).sum(ax)
    eSi = (g + e_img) * A
    eSii = (g + 2 * e_img) * Aq
    eSit = (g + e_img) * Ait
    eSt, eStt = g * At, g * Stt
    ectd = n * eStt + 2 * At * eSt + U * (n * Stt + St * St)
    enum = n * eSit + At * eSi + A * eSt + 2 * U * (n * Ait + A * At)
    espr = n * eSii + 2 * A * eSi + 2 * U * (n * Aq + A * A)
    eden = np.abs(ctd) * espr + np.abs(spr) * ectd + ectd * espr + 2 * U * (np.abs(ctd * spr) + FLT_MIN)
    with np.errstate(invalid="ignore", divide="ignore"):
        rel = eden / den
        eps = enum / np.sqrt(den) + np.abs(score) * (0.5 * rel + FAST["rsqrt"] + U)
        eps = np.where(rel < 0.5, 2.0 * eps, np.inf)   # first-order bound, doubled for the second-order terms
    return score, eps, gx, gy


def search(fr, xs, ys, mu, s2, fast=True, draws=32, tap_ulps=0.0, chunk=2048):
    """Float64 search of every listed seed.  Returns a dict of per-seed arrays and per-(seed, candidate) arrays:
    L (fp32 comb), px/py, exists / accepted (True, False or ambiguous), score, eps.

    `tap_ulps`: how many ulp(px) the implementation's tap positions may move beyond the rounding of px itself (the
    CPU oracle re-adds +-0.5 per tap, the kernels sample the block at px - P/2 exactly)."""
    P, W, H = fr.P, fr.W, fr.H
    mean, d, hl, d_mean, d_dir, d_hl = segment(fr, xs, ys, mu, s2, fast, draws)
    L, h32, has = comb(hl)
    C = L.shape[1]
    with np.errstate(invalid="ignore"):
        # the implementation's l starts at its own -half_length: the end test is ambiguous within that spread
        end_amb = ~np.isnan(L) & (np.abs(L - h32[:, None]) <= 2 * d_hl[:, None] + 2e-5)
        L = np.where(has | end_amb, L, np.nan)
        px = mean[0][:, None] + L * d[0][:, None]
        py = mean[1][:, None] + L * d[1][:, None]
        pos_err = (d_mean[:, None] + np.abs(L) * d_dir[:, None] + 2 * d_hl[:, None]
                   + (0.5 + tap_ulps) * ulp32(np.maximum(np.abs(px), np.abs(py))))
        rej = (px >= W - P) | (py >= H - P) | (px < P) | (py < P)                           # :91-97
        near = ((np.abs(px - (W - P)) <= pos_err) | (np.abs(py - (H - P)) <= pos_err)
                | (np.abs(px - P) <= pos_err) | (np.abs(py - P) <= pos_err))
    acc_sure = has & ~rej & ~near & ~end_amb
    acc_any = (has | end_amb) & (~rej | near)
    score = np.full((len(xs), C), -np.inf)
    eps = np.zeros((len(xs), C))
    tpl = _templates(fr, xs, ys)
    si, ci = np.nonzero(acc_any)
    window = 1e-3 + 256.0 * pos_err[si, ci]
    for s in range(0, len(si), chunk * 64):
        sl = slice(s, s + chunk * 64)
        a, b = si[sl], ci[sl]
        sc, ep, gx, gy = _ncc(fr, a, tpl, px[a, b], py[a, b])
        # a candidate whose frac * 256 lies at a rounding boundary within its position error: add the score change
        # of moving that weight by one step of the fixed-point grid
        for axis, gap, px_, py_ in ((0, gx, px[a, b], py[a, b]), (1, gy, px[a, b], py[a, b])):
            k = np.nonzero(gap <= window[sl])[0]
            if len(k) == 0:
                continue
            fracq = (px_[k] if axis == 0 else py_[k]) - P // 2
            up = (fracq * 256 - np.floor(fracq * 256)) < 0.5    # rounded down: the other side rounds up
            sh = np.where(up, 1.0, -1.0)
            shift = (sh, 0.0) if axis == 0 else (0.0, sh)
            alt, _, _, _ = _ncc(fr, a[k], tpl, px_[k], py_[k], shift=shift)
            with np.errstate(invalid="ignore"):
                ep[k] = ep[k] + np.abs(alt - sc[k])
        score[a, b], eps[a, b] = sc, ep
    return dict(L=L, px=px, py=py, has=has, acc_sure=acc_sure, acc_any=acc_any, score=score,
                eps=eps, mean=mean, dir=d, hl=hl, h32=h32, pos_err=pos_err)


def check_search(S, matched, match_xy):
    """Per seed: for `matched` seeds the recorded match must be a comb candidate (1e-3 px) whose float64 score is
    >= max - eps and >= 0.5 - eps; for the others (NO_MATCH) the float64 best must be < 0.5 + eps.
    Returns (fail_mask, chosen_index)."""
    n = len(matched)
    with np.errstate(invalid="ignore"):
        lo = np.where(S["acc_sure"], S["score"] - S["eps"], -np.inf)
        best_lo = lo.max(axis=1) if lo.shape[1] else np.full(n, -np.inf)
        hi = np.where(S["acc_any"], S["score"] + S["eps"], -np.inf)
    fail = np.zeros(n, bool)
    # NO_MATCH: nothing certainly accepted scores surely >= 0.5
    fail |= ~matched & (best_lo >= NCC_ACCEPT)
    # matched: nearest comb index along the segment
    mx, my = match_xy[:, 0].astype(np.float64), match_xy[:, 1].astype(np.float64)
    with np.errstate(invalid="ignore"):
        l_est = (mx - S["mean"][0]) * S["dir"][0] + (my - S["mean"][1]) * S["dir"][1]
        k = np.rint((l_est - S["L"][:, 0]) / float(STEP))
    C = S["L"].shape[1]
    k = np.where(np.isfinite(k), k, -1).astype(np.int64)
    inrange = (k >= 0) & (k < C)
    kk = np.clip(k, 0, max(C - 1, 0))
    rows = np.arange(n)
    if C:
        dist = np.maximum(np.abs(S["px"][rows, kk] - mx), np.abs(S["py"][rows, kk] - my))
        on = inrange & (np.nan_to_num(dist, nan=np.inf) <= 1e-3)
        ok_idx = on & S["acc_any"][rows, kk]
        # the implementation's segment may end one candidate later than the float64 one
        hk = hi[rows, kk]
        ok_score = (hk >= best_lo) & (hk >= NCC_ACCEPT)
    else:
        ok_idx = ok_score = np.zeros(n, bool)
    fail |= matched & ~(ok_idx & ok_score)
    # a score the forward bound cannot pin down (flat template or patch: den ~ FLT_MIN, a rounding residue times
    # rsqrt(FLT_MIN)) leaves the decision to rounding: such seeds are ambiguous, not checked
    undetermined = (np.where(S["acc_any"], S["eps"], 0.0) >= 0.25).any(axis=1) if C else np.zeros(n, bool)
    return fail & ~undetermined, np.where(ok_idx, k, -1), undetermined


def templ_stats(ref, patch):
    """sum_templ and const_templ_denom of every pixel (src/seed_init.cu:39-54, clamped addressing) in float64,
    with the forward error bounds of their fp32 evaluation (running sums of P^2 terms, then the double combination
    P^2 sum_sq - sum^2 rounded to float)."""
    ref = np.asarray(ref, np.float32).astype(np.float64)
    H, W = ref.shape
    r = patch // 2
    pad = np.pad(ref, r, mode="edge")
    St = np.zeros((H, W)); Stt = np.zeros((H, W)); At = np.zeros((H, W))
    for dy in range(patch):
        for dx in range(patch):
            t = pad[dy:dy + H, dx:dx + W]
            St += t; Stt += t * t; At += np.abs(t)
    n = patch * patch
    eSt, eStt = n * U * At, (n + 1) * U * Stt
    ctd = n * Stt - St * St
    ectd = n * eStt + 2 * np.abs(St) * eSt + eSt * eSt + U * (np.abs(ctd) + n * eStt + 2 * np.abs(St) * eSt)
    return St, eSt, ctd, ectd


# ------------------------------------------------------------------------------------------------ update

def _update(ar, fr, xs, ys, match, mu, s2, a, b):
    """Triangulation (src/triangulation.cu:30-50), tau (:53-68) and the moment-matched update
    (src/seed_update.cu:58-110).  Returns (ok, mu', sigma^2', a', b'); ok is False when the point is behind the
    camera (:77-80) or the update is NaN (:100-103)."""
    T = ar.pose(fr.T_ref_curr)
    opa = ar.pose(np.full(12, fr.one_pix_angle, np.float32))[0]
    dot = lambda p, q: ar.add(ar.add(ar.mul(p[0], q[0]), ar.mul(p[1], q[1])), ar.mul(p[2], q[2]))
    f1 = _bearing(ar, fr, xs.astype(np.float64), ys.astype(np.float64))
    fc = _bearing(ar, fr, match[:, 0].astype(np.float64), match[:, 1].astype(np.float64))
    t = (T[3], T[7], T[11])
    f2 = tuple(ar.add(ar.add(ar.mul(T[4 * r], fc[0]), ar.mul(T[4 * r + 1], fc[1])), ar.mul(T[4 * r + 2], fc[2]))
               for r in range(3))
    bx, by = dot(t, f1), dot(t, f2)
    A0, A2 = dot(f1, f1), dot(f1, f2)
    A1, A3 = -A2, dot((-f2[0], -f2[1], -f2[2]), f2)
    det = ar.sub(ar.mul(A0, A3), ar.mul(A1, A2))
    lx = ar.div(ar.sub(ar.mul(A3, bx), ar.mul(A1, by)), det)
    ly = ar.div(ar.add(ar.mul(-A2, bx), ar.mul(A0, by)), det)
    pt = [ar.mul(ar.add(ar.mul(lx, f1[i]), ar.add(t[i], ar.mul(ly, f2[i]))), 0.5) for i in range(3)]
    front = ~(pt[2] < 0.0)
    depth = ar.sqrt(dot(pt, pt))
    # triangulationUncertainty
    av = [ar.sub(ar.mul(f1[i], depth), t[i]) for i in range(3)]
    t_norm, a_norm = ar.sqrt(dot(t, t)), ar.sqrt(dot(av, av))
    alpha = ar.acos(ar.div(dot(f1, t), t_norm))
    beta = ar.acos(ar.div(-dot(av, t), ar.mul(t_norm, a_norm)))
    beta_plus = ar.add(beta, opa)
    gamma_plus = ar.f32(np.pi - alpha - beta_plus)                                           # :65, in double
    tau = ar.sub(ar.div(ar.mul(t_norm, ar.sin(beta_plus)), ar.sin(gamma_plus)), depth)
    tau_sq = ar.mul(tau, tau)
    # seed_update.cu:83-110
    var_sum = ar.add(s2, tau_sq)
    s_sq = ar.div(ar.mul(tau_sq, s2), var_sum)
    m = ar.mul(s_sq, ar.add(ar.div(mu, s2), ar.div(depth, tau_sq)))
    ab = ar.add(a, b)
    dd = ar.sub(depth, mu)
    pdf = ar.mul(ar.exp(ar.div(ar.mul(-dd, dd), ar.mul(2.0, var_sum))),
                 ar.rsqrt(ar.f32(2.0 * np.pi * var_sum)))                                      # :31-37
    c1 = ar.mul(ar.div(a, ab), pdf)
    c2 = ar.mul(ar.div(b, ab), ar.div(1.0, fr.depth_range))
    nc = ar.add(c1, c2)
    c1, c2 = ar.div(c1, nc), ar.div(c2, nc)
    ab1, ab2, a1, a2 = ar.add(ab, 1.0), ar.add(ab, 2.0), ar.add(a, 1.0), ar.add(a, 2.0)
    f = ar.add(ar.mul(c1, ar.div(a1, ab1)), ar.mul(c2, ar.div(a, ab1)))
    dd12 = ar.mul(ab1, ab2)
    e = ar.add(ar.mul(c1, ar.div(ar.mul(a1, a2), dd12)), ar.mul(c2, ar.div(ar.mul(a, a1), dd12)))
    c1m = ar.mul(c1, m)
    ok = front & ~np.isnan(c1m)
    mu_p = ar.add(c1m, ar.mul(c2, mu))
    s2_p = ar.sub(ar.add(ar.mul(c1, ar.add(s_sq, ar.mul(m, m))), ar.mul(c2, ar.add(s2, ar.mul(mu, mu)))),
                  ar.mul(mu_p, mu_p))
    a_p = ar.div(ar.sub(e, f), ar.sub(f, ar.div(e, f)))
    b_p = ar.div(ar.mul(a_p, ar.sub(1.0, f)), f)
    return ok, mu_p, s2_p, a_p, b_p


def update(fr, xs, ys, match, mu, s2, a, b, fast=True, draws=32, seed=3):
    """Float64 update from the given matches: (ok, ambiguous, values[4], bounds[4])."""
    n = len(xs)
    args = [np.asarray(v, np.float64) for v in (mu, s2, a, b)]
    if fast:
        args = [np.where(np.abs(v) < FLT_MIN, 0.0 * v, v) for v in args]
    with np.errstate(all="ignore"):
        ok, *vals = _update(Arith(n, fast), fr, xs, ys, match, *args)
        rng = np.random.default_rng(seed)
        D = [_update(Arith(n, fast, rng), fr, xs, ys, match, *args) for _ in range(draws)]
        amb = np.zeros(n, bool)
        for dr in D:
            amb |= dr[0] != ok
        bounds = []
        for i, v in enumerate(vals):
            ds = [np.where(dr[0], dr[1 + i], np.nan) for dr in D]
            bd = _spread(ds, v)
            # a value the draws take both finite and not finite is ambiguous
            fin = [np.isfinite(x) for x in ds]
            amb |= ok & np.any([f != np.isfinite(v) for f in fin], axis=0)
            bounds.append(bd)
    return ok, amb, vals, bounds


def within(got, want, bound):
    """fp32 result inside [want - bound, want + bound]; NaN matches NaN, inf matches the same inf."""
    g = np.asarray(got, np.float64)
    with np.errstate(invalid="ignore"):
        both_nan = np.isnan(g) & np.isnan(want)
        same_inf = np.isinf(g) & (g == want)
        return both_nan | same_inf | (np.abs(g - want) <= bound)


# ------------------------------------------------------------------------------------------------ whole frame

class Report:
    def __init__(self):
        self.fail = {}
        self.n_checked = self.n_updated = 0
        self.ambiguous = None
        self.undetermined = None

    def add(self, name, mask):
        self.fail[name] = self.fail.get(name, 0) + int(np.count_nonzero(mask))

    @property
    def n_fail(self):
        return sum(self.fail.values())

    @property
    def n_ambiguous(self):
        return int(np.count_nonzero(self.ambiguous)) if self.ambiguous is not None else 0

    @property
    def n_undetermined(self):
        return int(np.count_nonzero(self.undetermined)) if self.undetermined is not None else 0

    def __str__(self):
        bad = {k: v for k, v in self.fail.items() if v}
        return (f"checked {self.n_checked} seeds ({self.n_updated} searched), ambiguous {self.n_ambiguous} "
                f"(of which {self.n_undetermined} with an undetermined NCC score), failing {self.n_fail} {bad}")


def check_frame(fr, pre, post, matches, trust_conv=True, fast=True, draws=32, search_mask=None, tap_ulps=0.0,
                search_cache=None):
    """Check every pixel of one update.  `pre` / `post`: dicts with mu, sigma_sq, a, b (fp32) and conv (int32) of
    shape (H, W); `matches`: (H, W, 2) recorded matches.  `search_mask` limits the float64 search to some pixels
    (the others are checked for their state only).  `search_cache` (a dict) keeps the float64 search of this state
    for reuse by other organisations of the same update.  Returns a Report."""
    H, W = fr.H, fr.W
    ys, xs = np.mgrid[0:H, 0:W]
    ys, xs = ys.ravel(), xs.ravel()
    g = {k: np.asarray(v).reshape(H * W) for k, v in pre.items()}
    p = {k: np.asarray(v).reshape(H * W) for k, v in post.items()}
    mt = np.asarray(matches, np.float32).reshape(H * W, 2)
    rep = Report()
    rep.n_checked = H * W
    bits = lambda v: np.asarray(v, np.float32).view(np.int32)
    same = {k: bits(p[k]) == bits(g[k]) for k in ("mu", "sigma_sq", "a", "b")}
    unchanged = same["mu"] & same["sigma_sq"] & same["a"] & same["b"]

    state, amb = classify(fr, xs, ys, g["mu"], g["sigma_sq"].astype(np.float64), g["a"].astype(np.float64),
                          g["b"].astype(np.float64), g["conv"], trust_conv)
    absorbing = np.isin(state, (BORDER, CONVERGED, DIVERGED)) & ~amb
    rep.add("absorbing seed changed", absorbing & ~(unchanged & (p["conv"] == state)))
    live = ~np.isin(state, (BORDER, CONVERGED, DIVERGED)) & ~amb
    rep.add("state differs", live & ~np.isin(p["conv"], (UPDATE, NO_MATCH)))
    rep.add("state differs", amb & ~np.isin(p["conv"], (UPDATE, NO_MATCH, CONVERGED, DIVERGED)))
    if search_mask is not None:
        live &= np.asarray(search_mask).reshape(H * W)
    idx = np.nonzero(live)[0]
    rep.n_updated = len(idx)
    if len(idx):
        key = "search"
        if search_cache is not None and key in search_cache:
            S = search_cache[key]
        else:
            S = search(fr, xs[idx], ys[idx], g["mu"][idx].astype(np.float64), g["sigma_sq"][idx].astype(np.float64),
                       fast, draws, tap_ulps)
            if search_cache is not None:
                search_cache[key] = S
        matched = p["conv"][idx] == UPDATE
        fail, _, undetermined = check_search(S, matched, mt[idx])
        rep.add("search", fail)
        und = np.zeros(H * W, bool)
        und[idx] = undetermined
        rep.undetermined = und
        amb[idx] |= undetermined
        nm = ~matched
        b1 = (np.float32(g["b"][idx]) + np.float32(1.0)).astype(np.float32)
        rep.add("NO_MATCH update", nm & ~((bits(p["b"][idx]) == bits(b1)) & same["mu"][idx] & same["sigma_sq"][idx]
                                           & same["a"][idx]))
        mi = idx[matched]
        ok, uamb, vals, bnds = update(fr, xs[mi], ys[mi], mt[mi], g["mu"][mi], g["sigma_sq"][mi], g["a"][mi],
                                      g["b"][mi], fast, draws)
        good = ok & ~uamb
        inside = np.ones(len(mi), bool)
        for name, v, bd in zip(("mu", "sigma_sq", "a", "b"), vals, bnds):
            inside &= within(p[name][mi], v, bd)
        rep.add("update outside bound", good & ~inside)
        rep.add("rejected update changed the seed", ~ok & ~uamb & ~unchanged[mi])
        amb[mi] |= uamb
    rep.ambiguous = amb
    return rep
