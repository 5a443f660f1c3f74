"""Float64 model of the TV-L1 denoiser that follows the implementation's own iterates, with per-pixel bounds.

Test infrastructure: vectorised over pixels with numpy, written from the reference's mathematics
(src/depthmap_denoiser.cu:46-59 weights, :62-118 one primal-dual step, :124-141 constants, :226-229 large sigma^2)
and the operation forms of csrc/denoiser.cu.

The public API hands out only the primal u after k iterations, and runs are deterministic, so a caller runs
k = 0, 1, ..., K as separate calls and passes the chain u_0 ... u_K to `check_chain`.  Every iterate u_k is a
function of u_{k-1} and u_head_{k-1}, both observable, and of the dual p_k, which the model tracks:

* u_head is observable: u_head_0 = mu and u_head_k = fma(theta, u_k - u_{k-1}, u_k) with theta = 0.5 (`u_head`).
* the dual p_k is computed in float64 from the implementation's u_{k-1} and u_head_{k-1}, and carries a bound
  dp_k >= |p_k^impl - p_k^model| (Euclidean).  Projection onto the unit disc is non-expansive, so
  dp_k <= dp_{k-1} + e_k, where e_k collects the fp32 roundings of g * grad, the FMA, len_sq, the rsqrt figure and
  the product (the branch at len_sq ~ 1 is continuous: it costs |1 - 1/len| |t|, a few ulp).  The bound grows
  linearly in k; it never compounds, because u is re-read from the implementation at every step.
* the predicted u_k is the divergence (with its edge zeros) and the soft threshold around mu, in float64 from the
  model's p_k.  Its bound adds tau g times the neighbours' dp, the roundings of div, tau * g, the FMA and
  temp -/+ tau lambda; the soft threshold is 1-Lipschitz.
* g = max((E s2 + (1 - E) L) / L, 1), E = a / (a + b): where the float64 value is decidably below 1 it is exactly
  1.0 (fmaxf); elsewhere it carries the two approximate divisions' error.  Special operands take the semantics PTX
  specifies for div.approx.ftz.f32 (a * rcp(b): rcp(0) = inf, 0 for 2^126 < |b| < 2^128, subnormals flushed).

Exact equalities are required where they must hold: u_0 = mu, the middle branch of the threshold (u = mu bit for
bit) where the model decides it with margin, NaN positions, and infinities.  A pixel whose fp32 overflow the model
cannot decide (an intermediate within 2^-16 of FLT_MAX, or a finite value with a non-finite bound) is ambiguous:
counted, reported, not checked.

`fast=True` models the sm_90a kernels (-use_fast_math: FTZ, rsqrt.approx, div.approx); `fast=False` models the IEEE
CPU oracle (oracle/rmd_oracle.c, -ffp-contract=off: every operation rounded once, sqrtf and a true division).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from f64_depth_filter import FAST, FLT_MAX, FLT_MIN, IEEE, U

F32 = np.float32
SQRT2 = float(np.sqrt(2.0))
BAND = 2.0 ** -16                   # |x| within this relative distance of FLT_MAX: overflow undecided


def constants(lam, depth_range):
    """The fp32 constants exactly as the host computes them (c_api.cu denoiser_iterate and
    rmd_denoiser_set_large_sigma_sq; the oracle uses the same expressions)."""
    L = np.sqrt(F32(8.0))
    tau = F32(0.02)
    sigma = (F32(1) / (L * L)) / tau
    theta = F32(0.5)
    lam = F32(lam)
    tl = tau * lam                   # the kernel's P.tau * P.lambda
    r = F32(depth_range)
    lss = (r * r) / F32(72.0)
    return dict(tau=float(tau), sigma=float(sigma), theta=float(theta), tl=float(tl), lss=float(lss))


def _fz(x, fast):
    """Flush-to-zero of subnormal operands / results (sm_90a under -use_fast_math)."""
    if not fast:
        return x
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(x) < FLT_MIN, 0.0 * x, x)


def _range(x, amb):
    """fp32 overflow of a float64 intermediate: beyond FLT_MAX it is +-inf; within BAND of FLT_MAX the rounding
    decides, so the pixel is ambiguous."""
    a = np.abs(x)
    amb |= (a > FLT_MAX * (1 - BAND)) & (a < FLT_MAX * (1 + BAND))
    return np.where(a > FLT_MAX, np.copysign(np.inf, x), x)


def u_head(u_prev, u, fast):
    """u_head_k = fma(theta, u_k - u_{k-1}, u_k), theta = 0.5, reproduced bit for bit (float32 arrays in and out).

    Kernel (fast): d = sub.rn.ftz(u, u_prev), then fma.rn.ftz(0.5, d, u).  0.5 * d is exact in float64 and u is an
    fp32 value, so u + 0.5 d is the sum of two 24-bit-significand numbers; rounding it first to float64 (53 >= 2 * 24 + 2
    bits) and then to float32 gives the correctly rounded sum (double rounding is innocuous for one addition of
    precision-p operands when the intermediate precision is at least 2p + 2), which is what the single-rounding FMA
    returns.  FTZ applies to the operands and to the result.
    Oracle (IEEE): nu + theta * (nu - old_u) in three correctly rounded float32 operations (gradual underflow).
    """
    u_prev = np.asarray(u_prev, F32)
    u = np.asarray(u, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        if not fast:
            return u + F32(0.5) * (u - u_prev)
        uf = _fz(u.astype(np.float64), True).astype(F32)
        pf = _fz(u_prev.astype(np.float64), True).astype(F32)
        d = _fz((uf - pf).astype(np.float64), True)
        r = (uf.astype(np.float64) + 0.5 * d).astype(F32)
        return _fz(r.astype(np.float64), True).astype(F32)


def weights(s2, a, b, lss, fast):
    """g and its bound dg (float64 arrays); `amb` marks undecidable overflow.  Kernel: s = a + b;
    E = div.approx(a, s); m = 1 - E; n = fma(E, s2, m * L); g = max(div.approx(n, L), 1).  Oracle: the same in
    correctly rounded steps with E * s2 rounded separately."""
    d = FAST if fast else IEEE
    amb = np.zeros(np.shape(s2), bool)
    A, B, S = (_fz(np.asarray(v, np.float64), fast) for v in (a, b, s2))
    L = float(_fz(np.float64(lss), fast))
    with np.errstate(all="ignore"):
        s = _fz(np.asarray(F32(A) + F32(B), np.float64), fast)   # one fp32 addition: emulated exactly
        if fast:
            # div.approx.ftz.f32 = a * rcp(b): rcp(0) = inf, rcp(|b| > 2^126) = 0, inf * 0 = NaN
            rcp = np.where(s == 0, np.copysign(np.inf, s), np.where(np.abs(s) > 2.0 ** 126, 0.0 * s, 1.0 / s))
            E = _range(A * rcp, amb)
        else:
            E = _range(A / s, amb)
        dE = np.abs(E) * d["div"]
        m = _range(1.0 - E, amb)
        dm = dE + U * np.abs(m)
        n2 = _range(m * L, amb)
        dn2 = dm * L + U * np.abs(n2)
        num = _range(E * S + n2, amb)
        dnum = dE * np.abs(S) + dn2 + U * np.abs(num) + (0.0 if fast else U * np.abs(E * S))
        if fast:
            rl = np.inf if L == 0 else (0.0 if abs(L) > 2.0 ** 126 else 1.0 / L)
            gp = _range(num * rl, amb)
        else:
            gp = _range(num / L, amb)
        dgp = dnum / abs(L) + d["div"] * np.abs(gp) + (4 * FLT_MIN if fast else 0.0)
        g = np.fmax(gp, 1.0)                                      # fmaxf / "v > 1 ? v : 1": NaN -> 1
        dg = np.where(np.isnan(gp) | (gp + dgp < 1.0), 0.0, dgp)
    dg = np.where(np.isfinite(g), dg, 0.0)
    amb |= np.isfinite(g) & ~np.isfinite(dg)
    return g, dg, amb


@dataclass
class ChainReport:
    shape: tuple
    fails: list = field(default_factory=list)        # failing pixels per k
    ambiguous: list = field(default_factory=list)    # ambiguous pixels per k
    middle: list = field(default_factory=list)       # pixels held to u = mu bit for bit, per k
    bound_max: list = field(default_factory=list)    # max finite bound per k
    bound_median: list = field(default_factory=list)
    ratio_max: float = 0.0                           # max |impl - model| / bound over checked pixels, all k
    first: dict | None = None                        # the first failing (k, y, x) with its bound terms

    @property
    def n_fail(self):
        return int(sum(self.fails))

    @property
    def n_ambiguous(self):
        return int(max(self.ambiguous) if self.ambiguous else 0)

    def summary(self):
        return (f"{self.shape[1]}x{self.shape[0]} K={len(self.fails) - 1}: fails {self.n_fail}, ambiguous max/k "
                f"{self.n_ambiguous}, exact-middle px/k {int(np.median(self.middle)) if self.middle else 0}, "
                f"bound median@K {self.bound_median[-1] if self.bound_median else 0:.3g} "
                f"max@K {self.bound_max[-1] if self.bound_max else 0:.3g}, worst |err|/bound {self.ratio_max:.3g}"
                + (f", first failure {self.first}" if self.first else ""))


class Model:
    """The float64 state (p and its bound) for one chain; `step` consumes u_{k-1}, u_head_{k-1} and u_k."""

    def __init__(self, mu, s2, a, b, depth_range, lam, fast=True):
        self.fast = fast
        self.d = FAST if fast else IEEE
        self.c = constants(lam, depth_range)
        self.mu32 = np.asarray(mu, F32)
        self.H, self.W = self.mu32.shape
        self.mu = self.mu32.astype(np.float64)
        self.g, self.dg, self.amb_g = weights(s2, a, b, self.c["lss"], fast)
        self.px = np.zeros_like(self.mu)
        self.py = np.zeros_like(self.mu)
        self.dp = np.zeros_like(self.mu)
        # pixels whose dual the model cannot decide (sticky: p is never observed); g's ambiguity feeds it
        self.amb_p = self.amb_g.copy()

    @staticmethod
    def _readers(m):
        """Pixels whose primal reads an undecided dual: the pixel itself, its east (reads p.x of x - 1) and its
        south neighbour (reads p.y of y - 1).  Everything else is re-read from the implementation each step, so an
        undecided dual does not spread further."""
        out = m.copy()
        out[:, 1:] |= m[:, :-1]
        out[1:, :] |= m[:-1, :]
        return out

    def step(self, u_prev32, uh_prev32):
        """One dual + primal step from the implementation's u_{k-1}, u_head_{k-1}.  Returns (u_model, bound,
        exact_mask, amb, bound_terms): exact_mask marks pixels whose value is decided exactly (u = mu in the middle branch, or a
        non-finite value), bound applies elsewhere."""
        fast, d, c = self.fast, self.d, self.c
        H, W = self.H, self.W
        amb = self.amb_p.copy()
        sigma, tau, tl = c["sigma"], c["tau"], c["tl"]
        fl = 4 * FLT_MIN if fast else 0.0
        with np.errstate(all="ignore"):
            # ---- dual: grad is computed exactly (fp32 subtraction of observed values)
            u = _fz(np.asarray(u_prev32, F32), fast) if fast else np.asarray(u_prev32, F32)
            uh = _fz(np.asarray(uh_prev32, F32), fast) if fast else np.asarray(uh_prev32, F32)
            uh_e = np.concatenate([uh[:, 1:], uh[:, -1:]], axis=1)     # east of the last column: itself
            uh_s = np.concatenate([uh[1:, :], uh[-1:, :]], axis=0)     # south of the last row: itself
            gx = _fz((uh_e - u).astype(np.float64), fast)
            gy = _fz((uh_s - u).astype(np.float64), fast)
            g, dg = self.g, self.dg
            prx = _range(g * gx, amb)
            pry = _range(g * gy, amb)
            tx = _range(prx * sigma + self.px, amb)
            ty = _range(pry * sigma + self.py, amb)
            # per-component rounding: g*grad (U + dg/g), fma (or mul + add in the oracle), FTZ
            # FTZ costs at most FLT_MIN, and only where a result is non-zero (an exact zero stays exact)
            ex = sigma * (dg * np.abs(gx) + U * np.abs(prx)) + U * np.abs(tx) + fl * (tx != 0)
            ey = sigma * (dg * np.abs(gy) + U * np.abs(pry)) + U * np.abs(ty) + fl * (ty != 0)
            if not fast:
                ex = ex + U * sigma * np.abs(prx)
                ey = ey + U * sigma * np.abs(pry)
            et = np.sqrt(ex * ex + ey * ey)
            len_sq = _range(tx * tx + ty * ty, amb)
            ln = np.sqrt(len_sq)
            # kernel: len_sq > 1 ? t * rsqrt(len_sq) : t; len_sq = inf gives t * 0
            inv = np.where(len_sq > 1.0, 1.0 / ln, 1.0)
            npx = tx * inv
            npy = ty * inv
            # the projection branch: exact (t * 1) when decidably inside the disc, else the rsqrt / product
            # figure plus the continuous cost of deciding the branch on a rounded len_sq
            inside = (ln + self.dp + et) * (1 + 4 * U) < 1.0
            eproj = np.where(inside, 0.0, d["rsqrt"] + 6 * U) + fl * ((npx != 0) | (npy != 0))
            dp = np.minimum(self.dp + et + eproj, 2.0 + 2 * d["rsqrt"])
            # overflowed len_sq (decided): p = t * 0 exactly, nothing carried
            dp = np.where(np.isinf(len_sq), 0.0, dp)
            dp = np.where(np.isnan(npx) | np.isnan(npy), 0.0, dp)
            amb |= np.isfinite(npx) & np.isfinite(npy) & ~np.isfinite(dp)
            self.px, self.py, self.dp = npx, npy, dp
            self.amb_p = amb.copy()
            amb = self._readers(amb)

            # ---- primal: divergence with the edge zeros (kernel :88-99 rules)
            x = np.arange(W)[None, :]
            y = np.arange(H)[:, None]
            cx = np.where((x != 0) & (x >= W - 1), 0.0, npx)
            wx = np.where(x == 0, 0.0, np.concatenate([np.zeros((H, 1)), npx[:, :-1]], axis=1))
            cy = np.where((y != 0) & (y >= H - 1), 0.0, npy)
            ny = np.where(y == 0, 0.0, np.concatenate([np.zeros((1, W)), npy[:-1, :]], axis=0))
            dpw = np.where(x == 0, 0.0, np.concatenate([np.zeros((H, 1)), dp[:, :-1]], axis=1))
            dpn = np.where(y == 0, 0.0, np.concatenate([np.zeros((1, W)), dp[:-1, :]], axis=0))
            s1 = cx - wx
            s2 = s1 + cy
            div = s2 - ny
            ddiv = SQRT2 * dp + dpw + dpn
            ddiv = ddiv + U * (np.abs(s1) + np.abs(s2) + np.abs(div) + 3 * ddiv) + 3 * fl * (ddiv + np.abs(div) > 0)
            tg = _range(tau * g, amb)
            dtg = tau * dg + U * np.abs(tg) * (g != 1.0)               # tau * 1.0 is exact
            uu = u.astype(np.float64)
            temp = _range(tg * div + uu, amb)
            # with div exactly 0 (ddiv = 0) the FMA returns u itself: no rounding
            moved = (div != 0) | (ddiv > 0)
            bt = np.where(moved, np.abs(tg) * ddiv + np.abs(div) * dtg + U * np.abs(temp) + fl, 0.0)
            if not fast:
                bt = bt + U * np.abs(tg * div)
            # ---- soft threshold around mu (exact fp32 tau * lambda)
            mu = _fz(self.mu, fast)
            dx = temp - mu
            nu = np.where(dx > tl, temp - tl, np.where(dx < -tl, temp + tl, self.mu))
            nan_t = np.isnan(temp)
            nu = np.where(nan_t, self.mu, nu)                           # NaN compares false: u = mu
            margin = bt + U * np.abs(dx) + fl * (dx != 0)
            middle = (np.abs(dx) + margin < tl * (1 - 2 * U)) | ((margin == 0) & (dx == 0))
            middle |= nan_t
            bound = margin + U * np.abs(nu) + fl
            bound = np.where(middle, 0.0, bound)
            nonfin = ~np.isfinite(nu)
            amb |= np.isfinite(nu) & ~np.isfinite(bound)
            # an infinite temp gives +-inf -/+ tl = +-inf; a finite one reaches inf only by overflow of
            # temp -/+ tl, which _range marks
            _range(nu, amb)
        exact = middle | nonfin
        return nu, bound, exact, amb, dict(dp=dp, et=et, eproj=eproj, ddiv=ddiv, bt=bt, temp=temp, tg=tg, div=div)


def check_chain(inputs, chain, depth_range, lam, fast=True):
    """inputs = (mu, s2, a, b) float32 arrays; chain = iterable of u_0, u_1, ..., u_K (float32, the
    implementation's output after k iterations).  Returns a ChainReport: failures and ambiguous pixels per k, and
    the first failing (k, y, x) together with its bound terms."""
    mu, s2, a, b = (np.asarray(v, F32) for v in inputs)
    model = Model(mu, s2, a, b, depth_range, lam, fast)
    rep = ChainReport(shape=mu.shape)
    it = iter(chain)
    u0 = np.asarray(next(it), F32)
    bad0 = u0.view(np.int32) != mu.view(np.int32)
    rep.fails.append(int(bad0.sum()))
    rep.ambiguous.append(0)
    rep.middle.append(int(mu.size))
    rep.bound_max.append(0.0)
    rep.bound_median.append(0.0)
    if bad0.any():
        y, x = np.argwhere(bad0)[0]
        rep.first = dict(k=0, y=int(y), x=int(x), got=float(u0[y, x]), want=float(mu[y, x]), rule="u_0 = mu")
    u_prev, uh_prev = u0, mu.copy()
    for k, uk in enumerate(it, start=1):
        uk = np.asarray(uk, F32)
        pred, bound, exact, amb, terms = model.step(u_prev, uh_prev)
        got = uk.astype(np.float64)
        with np.errstate(invalid="ignore"):
            err = np.abs(got - pred)
            same_bits = uk.view(np.int32) == model.mu32.view(np.int32)
            # exact pixels: the middle branch must return mu bit for bit; non-finite predictions must match
            # (NaN where NaN, the same infinity)
            mid = exact & np.isfinite(pred)
            bad = np.zeros(uk.shape, bool)
            bad |= mid & ~same_bits & ~(np.isnan(model.mu) & np.isnan(got))
            nanp = np.isnan(pred)
            bad |= nanp & ~np.isnan(got)
            infp = np.isinf(pred)
            bad |= infp & (got != pred)
            fin = ~exact
            bad |= fin & ~(err <= bound)
            bad &= ~amb
            chk = fin & ~amb & (bound > 0)
            if chk.any():
                rep.ratio_max = max(rep.ratio_max, float(np.nanmax(np.where(chk, err / np.where(chk, bound, 1), 0))))
        rep.fails.append(int(bad.sum()))
        rep.ambiguous.append(int(amb.sum()))
        rep.middle.append(int(mid.sum()))
        fb = bound[fin & ~amb & np.isfinite(bound)]
        rep.bound_max.append(float(fb.max()) if fb.size else 0.0)
        rep.bound_median.append(float(np.median(fb)) if fb.size else 0.0)
        if bad.any() and rep.first is None:
            y, x = (int(v) for v in np.argwhere(bad)[0])
            rep.first = dict(k=k, y=y, x=x, got=float(got[y, x]), want=float(pred[y, x]),
                             bound=float(bound[y, x]), exact=bool(exact[y, x]), mu=float(model.mu[y, x]),
                             g=float(model.g[y, x]), dg=float(model.dg[y, x]),
                             **{n: float(v[y, x]) for n, v in terms.items()})
        uh_prev = u_head(u_prev, uk, fast)
        u_prev = uk
    return rep
