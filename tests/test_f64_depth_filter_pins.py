"""Pins of the float64 reference (tests/f64_depth_filter.py) and its error model against the IEEE fp32 CPU oracle,
without a GPU.

The oracle runs one update stage by stage (stage_check / stage_match / stage_update; its `matches` field is a live
view, so a match can be replaced before stage_update).  With only the 2^-24 terms of the error model:
* search: the oracle's chosen candidate is an eps-arg-max of the float64 scores for every searched seed, and its
  NO_MATCH decisions agree with float64 best < 0.5 outside eps;
* update: fed the oracle's own matches, the float64 update bounds the oracle for every seed except ambiguous ones,
  which are at most 0.1 % of the searched seeds;
* the checker reports failing seeds for each planted bug.
"""
import numpy as np
import pytest

import f64_depth_filter as F
import oracle_binding as ob
from rpg_open_remode_b200 import synth

# the oracle's tap coordinates are px + offset + 0.5 - 0.5 in fp32 (oracle/rmd_oracle.c tex_linear): up to three
# roundings of the position beyond px itself
ORACLE_TAP_ULPS = 2.0


class Run:
    """An oracle keyframe run to the state before frame n, with that frame's inputs."""

    def __init__(self, size, patch, n, tex_frac_bits=8, seed=0x5EED0001):
        W, H = size
        self.seq = seq = synth.SyntheticSequence(W, H, seed=seed)
        f0 = seq.frame(0)
        self.dmin, self.dmax = float(f0.depth.min()), float(f0.depth.max())
        self.o = ob.OracleSeeds(W, H, *seq.camera, patch=patch, tex_frac_bits=tex_frac_bits)
        self.o.set_reference(f0.image, f0.T_cam_world, self.dmin, self.dmax)
        for k in range(1, n):
            f = seq.frame(k, want_depth=False)
            self.o.update(f.image, f.T_cam_world)
        self.f = seq.frame(n, want_depth=False)
        self.T_cr = ob.se3_mul(self.f.T_cam_world, ob.se3_inv(f0.T_cam_world))
        self.fr = F.Frame(f0.image, self.f.image, seq.camera, self.T_cr, self.dmin, self.dmax, patch=patch)
        self.pre = self.snap()

    def snap(self):
        o = self.o
        return dict(mu=o.mu.copy(), sigma_sq=o.sigma_sq.copy(), a=o.a.copy(), b=o.b.copy(), conv=o.convergence.copy())

    def match(self):
        self.o.stage_check()
        self.o.stage_match(self.f.image, self.T_cr)

    def update(self):
        self.o.stage_update(ob.se3_inv(self.T_cr))

    def check(self, cache=None, post=None, matches=None):
        post = self.snap() if post is None else post
        matches = self.o.matches.copy() if matches is None else matches
        return F.check_frame(self.fr, self.pre, post, matches, trust_conv=False, fast=False, tap_ulps=ORACLE_TAP_ULPS,
                             search_cache=cache)


_CACHE = {}


def _state(size, patch, n):
    key = (size, patch, n)
    if key not in _CACHE:
        r = Run(size, patch, n)
        r.match()
        matched_conv = r.o.convergence.copy()
        r.update()
        cache = {}
        rep = r.check(cache)
        _CACHE[key] = (r, cache, rep, matched_conv)
    return _CACHE[key]


STATES = [((320, 240), 5, 1), ((320, 240), 5, 4), ((320, 240), 5, 13), ((320, 240), 5, 40), ((320, 240), 5, 120),
          ((203, 131), 7, 7)]


@pytest.mark.parametrize("size,patch,n", STATES)
def test_oracle_inside_every_bound(size, patch, n):
    r, _, rep, _ = _state(size, patch, n)
    print(f"{size} {patch}x{patch} frame {n}: {rep}")
    assert rep.fail.get("search", 0) == 0, rep
    assert rep.n_fail == 0, rep
    assert rep.n_updated > 0
    assert rep.n_ambiguous <= 0.001 * rep.n_updated, rep


def test_seed_init_bounds():
    """sum_templ and const_templ_denom of the oracle's seed initialisation within the float64 bounds."""
    for size, patch in (((320, 240), 5), ((101, 77), 5), ((203, 131), 7)):
        r = Run(size, patch, 1)
        St, eSt, ctd, ectd = F.templ_stats(r.fr.ref, patch)
        assert (np.abs(r.o.sum_templ - St) <= eSt).all()
        assert (np.abs(r.o.const_templ_denom - ctd) <= ectd).all()


# ----------------------------------------------------------------------------------------- planted bugs

def test_catches_wrong_texture_weights():
    """The oracle searching the same state with 7-bit weights must fail the 8-bit model.  A weight off by at most
    1/256 moves a score by less than the gap between neighbouring candidates almost everywhere, so only a few seeds
    flip (5 of 71 300 here); exact fp32 weights (off by at most 1/512) flip none on this state."""
    bits, min_fail = 7, 3
    r0, cache, _, _ = _state((320, 240), 5, 1)
    r = Run((320, 240), 5, 1)
    ob.lib().rmd_oracle_seeds_set_tex_model(r.o._h, bits)
    r.match()
    r.update()
    rep = r.check(cache)
    print(f"{bits}-bit weights: {rep}")
    assert rep.fail.get("search", 0) >= min_fail, rep


def _rerun(n=4):
    """A fresh oracle in the cached state, stopped between stage_match and stage_update."""
    r = Run((320, 240), 5, n)
    r.match()
    return r


def test_catches_match_moved_one_step():
    """One recorded match in 500 moved one comb step along its segment: every such seed whose neighbour's float64
    score is more than eps below the maximum is reported."""
    r0, cache, _, _ = _state((320, 240), 5, 4)
    S = cache["search"]
    r = _rerun()
    H, W = r.fr.H, r.fr.W
    conv = r.o.convergence
    live = np.nonzero(conv.ravel() == F.UPDATE)[0]
    # rows of the cached search are the seeds the checker searched, in raster order
    state, amb = F.classify(r.fr, np.arange(H * W) % W, np.arange(H * W) // W, r.pre["mu"].ravel(),
                            r.pre["sigma_sq"].ravel().astype(np.float64), r.pre["a"].ravel().astype(np.float64),
                            r.pre["b"].ravel().astype(np.float64), r.pre["conv"].ravel(), False)
    searched = np.nonzero((state == F.UPDATE) & ~amb)[0]
    row = {p: i for i, p in enumerate(searched)}
    m = r.o.matches.reshape(H * W, 2)
    _, k_chosen, _ = F.check_search(S, np.ones(len(searched), bool), m[searched])
    moved = []
    for p in live[::500]:
        i = row.get(p)
        if i is None or k_chosen[i] < 0:
            continue
        k = k_chosen[i]
        step = 1 if k + 1 < S["L"].shape[1] and S["acc_sure"][i, k + 1] else -1
        if not (0 <= k + step and S["acc_sure"][i, k + step]):
            continue
        best = np.max(np.where(S["acc_sure"][i], S["score"][i] - S["eps"][i], -np.inf))
        must_flag = S["score"][i, k + step] + S["eps"][i, k + step] < best
        m[p] = (np.float32(S["px"][i, k + step]), np.float32(S["py"][i, k + step]))
        moved.append((p, must_flag))
    r.update()
    rep = r.check(cache)
    flagged = F.check_search(S, np.ones(len(searched), bool), r.o.matches.reshape(H * W, 2)[searched])[0]
    must = [p for p, f in moved if f]
    print(f"moved {len(moved)} matches, {len(must)} must be flagged: {rep}")
    assert len(must) >= 20
    assert all(flagged[row[p]] for p in must)
    assert rep.fail.get("search", 0) >= len(must)


def test_catches_no_match_without_b_increment():
    r0, cache, _, _ = _state((320, 240), 5, 4)
    r = _rerun()
    nm = r.o.convergence == F.NO_MATCH
    r.update()
    post = r.snap()
    post["b"][nm] = r.pre["b"][nm]
    rep = r.check(cache, post=post)
    print(rep)
    assert rep.fail.get("NO_MATCH update", 0) >= 0.9 * nm.sum() > 100


def test_catches_update_with_wrong_one_pixel_angle():
    """The update recomputed with one_pix_angle x 1.001 (tau and hence sigma^2 off by ~1e-3)."""
    r0, cache, _, _ = _state((320, 240), 5, 13)
    r = Run((320, 240), 5, 13)
    r.match()
    r.update()
    post = r.snap()
    H, W = r.fr.H, r.fr.W
    sel = np.nonzero((post["conv"].ravel() == F.UPDATE) & (r.pre["conv"].ravel() != F.BORDER))[0]
    xs, ys = sel % W, sel // W
    bad = F.Frame(r.fr.ref, r.fr.curr, r.seq.camera, r.T_cr, r.dmin, r.dmax)
    bad.one_pix_angle *= 1.001
    m = r.o.matches.reshape(H * W, 2)[sel]
    ok, _, vals, _ = F.update(bad, xs, ys, m, *(r.pre[k].ravel()[sel] for k in ("mu", "sigma_sq", "a", "b")),
                              fast=False, draws=1)
    for name, v in zip(("mu", "sigma_sq", "a", "b"), vals):
        flat = post[name].reshape(-1)
        flat[sel[ok]] = v[ok].astype(np.float32)
    rep = r.check(cache, post=post)
    print(rep)
    # tau moves sigma^2 only where tau^2 is not negligible against it: about 1 % of the updated seeds here
    assert rep.fail.get("update outside bound", 0) >= 300, rep


def test_catches_last_candidate_dropped():
    """A search that never scores the last accepted candidate of a segment: every seed whose float64 best is
    that candidate, by more than eps, is reported."""
    r0, cache, rep0, _ = _state((320, 240), 5, 1)
    S = cache["search"]
    r = Run((320, 240), 5, 1)
    r.match()
    H, W = r.fr.H, r.fr.W
    state, amb = F.classify(r.fr, np.arange(H * W) % W, np.arange(H * W) // W, r.pre["mu"].ravel(),
                            r.pre["sigma_sq"].ravel().astype(np.float64), r.pre["a"].ravel().astype(np.float64),
                            r.pre["b"].ravel().astype(np.float64), r.pre["conv"].ravel(), False)
    searched = np.nonzero((state == F.UPDATE) & ~amb)[0]
    acc = S["acc_sure"]
    C = acc.shape[1]
    last = np.where(acc.any(axis=1), C - 1 - np.argmax(acc[:, ::-1], axis=1), -1)
    sc = np.where(acc, S["score"], -np.inf)
    rows = np.arange(len(searched))
    sc_last = sc[rows, np.maximum(last, 0)]
    sc_wo = sc.copy()
    sc_wo[rows, np.maximum(last, 0)] = -np.inf
    k2 = np.argmax(sc_wo, axis=1)
    second = sc_wo[rows, k2]
    # seeds whose best is the last candidate by a margin larger than both bounds
    must = (last >= 0) & (sc_last - S["eps"][rows, np.maximum(last, 0)] > second + S["eps"][rows, k2]) & \
           (sc_last >= F.NCC_ACCEPT)
    conv = r.o.convergence.reshape(-1)
    m = r.o.matches.reshape(H * W, 2)
    for i in np.nonzero(must)[0]:
        p = searched[i]
        if second[i] >= F.NCC_ACCEPT:
            m[p] = (np.float32(S["px"][i, k2[i]]), np.float32(S["py"][i, k2[i]]))
            conv[p] = F.UPDATE
        else:
            conv[p] = F.NO_MATCH
    r.update()
    rep = r.check(cache)
    print(f"{int(must.sum())} seeds depend on their last candidate: {rep}")
    # (a seed whose second-best candidate sits at an end the model cannot call may still pass)
    assert must.sum() >= 100
    assert rep.fail.get("search", 0) >= 0.99 * must.sum(), rep
