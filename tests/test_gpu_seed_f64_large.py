"""Every seed of ONE fused depth-filter update against the float64 reference (tests/f64_depth_filter.py) at the
shapes bench.py times: c3 (1280x720, 5x5, seed 0x5EED0003) and c4 (1920x1080, 7x7, seed 0x5EED0004).

The small-shape checks of test_gpu_seed_f64.py rarely reach the paths the staged kernel takes here: candidate boxes
larger than the shared-memory strip (the rest of the candidates read global memory), capped 143-candidate segments
(the last l checkpoint), 7x7 paired scoring at full width, split, sparse and warp tiles late in a 500-frame sequence.

* Sequence states: frames 1, 4, 40, 200 and 499, each one update from the GPU's own pre-state.  The state of every
  seed is checked; the float64 search and update run on a sample of at most SAMPLE_TILES 32x8 tiles chosen from the
  kernel's own per-tile record (RMD_OPT_DEBUG_TIMELINE) -- overflowing strips, split, sparse and warp tiles, corner
  and edge tiles, the busiest tiles -- and the file asserts that every such path was reached at both shapes.
* Fresh blocks: at frames 200 and 499, rectangles of seeds reset to the prior setReferenceImage gives search full
  143-candidate segments, so their tiles overflow the strip; the upload makes the next update reclassify every seed.
* Every organisation of the kernel (test_gpu_seed_f64.ORGS) at c4 frames 40 and 499, bit for bit.
* The paths bench.py times: chained device-resident batches, and page-locked 8-bit frames DMA'd in place.
* Planted bugs at 1080p 7x7: texture weights with 6 and 5 fractional bits must be caught; 7 bits is reached and
  its catches reported, with the share of candidates whose eps includes a whole 1/256 weight step (the loss of
  sensitivity to the weights at this shape, test_planted_tex_bits_c4).

The host side dominates the run time (rendering 500 frames, the float64 model), so the sample is bounded; each test
prints its wall time.
"""
import time
from collections import defaultdict

import numpy as np
import pytest

import f64_depth_filter as F
import oracle_binding as ob
import rpg_open_remode_b200 as rmd
from rpg_open_remode_b200 import synth
from test_gpu_seed_f64 import ORGS, STATE_FIELDS, Case, _check, _handle, _same_state, _snap

pytestmark = pytest.mark.gpu

CONFIGS = {"c3": (1280, 720, 5, 0x5EED0003), "c4": (1920, 1080, 7, 0x5EED0004)}
N_FRAMES = 500
FRAMES = (1, 4, 40, 200, 499)
FRESH_FRAMES = (200, 499)
TILE_W, TILE_H = 32, 8
SAMPLE_TILES = 128
PER_CATEGORY = 16
MAX_CAND = 143            # candidates of a segment capped at 100 px: l = -50, -49.3, ..., 49.4
CATEGORIES = ("overflow", "split", "sparse", "warp", "edge", "busiest", "capped")
CHAIN_FRAMES = 64
WARP_TILE_MAX_SEEDS = 8   # staged_maps.cuh, the default of RMD_OPT_TUNE_WARP_TILE_SEEDS

# paths reached per configuration, summed over the checked states (asserted by test_paths_reached)
REACHED = defaultdict(lambda: defaultdict(int))
CHECKED = defaultdict(set)


@pytest.fixture(autouse=True)
def _wall_time(request):
    t0 = time.perf_counter()
    yield
    print(f"[time] {request.node.name}: {time.perf_counter() - t0:.1f} s")


class Run:
    """One configuration's sequence (rendered once: 8-bit frames, poses) and its sequence handles: `g` records
    matches, `gt` also the per-tile timeline; both take the same host float updates."""

    def __init__(self, name):
        W, H, self.patch, seed = CONFIGS[name]
        self.name = name
        self.seq = synth.SyntheticSequence(W, H, seed=seed)
        self.case = Case(self.seq)
        self.u8 = np.empty((N_FRAMES, H, W), np.uint8)
        self.poses = np.empty((N_FRAMES, 3, 4), np.float32)
        for k in range(N_FRAMES):
            f = self.seq.frame(k, want_depth=False)
            self.u8[k], self.poses[k] = f.image_u8, f.T_cam_world
        assert np.array_equal(self.image(0), self.case.ref)
        self.g = _handle(self.seq, self.patch)
        self.gt = _handle(self.seq, self.patch, [(rmd.OPT_DEBUG_TIMELINE, 1)])
        self.next = None          # the next frame the sequence handles update with
        self.done = {}            # frame -> the checked update's record

    @property
    def W(self):
        return self.seq.width

    @property
    def H(self):
        return self.seq.height

    def image(self, k):
        return ob.u8_to_float(self.u8[k])

    def frame_model(self, k):
        return self.case.frame_model(self.image(k), self.poses[k], self.patch)

    def prior(self):
        """The state setReferenceImage gives every seed."""
        g = _handle(self.seq, self.patch)
        self.case.start(g)
        return _snap(g)

    def checked(self, n):
        """Bring both handles to the state before frame n, update frame n on both, assert they agree bit for bit,
        and keep pre-state, post-state, matches, timeline and tile sample."""
        if n in self.done:
            return self.done[n]
        if self.next is None or self.next > n:
            for g in (self.g, self.gt):
                self.case.start(g)
            self.next = 1
        for k in range(self.next, n + 1):
            if k == n:
                pre = _snap(self.g)
                assert _same_state(pre, _snap(self.gt)), f"{self.name}: the timeline changed the state before frame {n}"
            for g in (self.g, self.gt):
                g.update(self.image(k), self.poses[k])
        self.next = n + 1
        post, post_t = _snap(self.g), _snap(self.gt)
        m, m_t = self.g.downloadEpipolarMatches(), self.gt.downloadEpipolarMatches()
        assert _same_state(post, post_t), f"{self.name} frame {n}: the timeline changed the update"
        assert _same_matches(post, m, m_t), f"{self.name} frame {n}: the timeline changed the matches"
        cats = tile_categories(self.gt.downloadTimeline(), post, self.W, self.H)
        rec = dict(pre=pre, post=post, matches=m, cats=cats, mask=sample_mask(cats, self.W, self.H))
        self.done[n] = rec
        return rec


def _same_matches(post, m1, m2):
    upd = post["conv"] == F.UPDATE
    return np.array_equal(m1[upd].view(np.int32), m2[upd].view(np.int32))


@pytest.fixture(scope="module")
def runs():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Run(name)
        return cache[name]
    return get


# ------------------------------------------------------------------------------------------ tile sample

def _tiles(W, H):
    return (W + TILE_W - 1) // TILE_W, (H + TILE_H - 1) // TILE_H


def live_per_tile(post, W, H):
    """Seeds the update searched (left in UPDATE or NO_MATCH), per 32x8 tile in tile order."""
    tx, ty = _tiles(W, H)
    live = np.zeros((ty * TILE_H, tx * TILE_W), np.int64)
    live[:H, :W] = np.isin(post["conv"], (F.UPDATE, F.NO_MATCH))
    return live.reshape(ty, TILE_H, tx, TILE_W).sum(axis=(1, 3)).ravel()


def tile_categories(tl, post, W, H):
    """Per-tile masks of the kernel paths, read from the debug timeline of the staged launch: [0] start stamp (lead
    CTA of the tile-organised path; warp tiles are not stamped), [7] work items, [10] candidate box w | h << 16,
    [11] strip w | rows << 16, [12] seeds to update, [13] zeff | sparse << 8."""
    tx, ty = _tiles(W, H)
    live = live_per_tile(post, W, H)
    stamped = tl[:, 0] != 0
    searched = stamped & (live > 0)
    # the reading of the record: a stamped tile's seed count is the seeds its update left live
    assert np.array_equal(tl[searched, 12], live[searched]), "timeline slot 12 disagrees with the live seeds"
    assert not (stamped & (live == 0) & (tl[:, 12] != 0)).any()
    # tiles with live seeds and no stamp are warp tiles: the previous frame listed them with at most
    # WARP_TILE_MAX_SEEDS seeds to update, and a tile's live seeds only become fewer
    assert (live[~stamped] <= WARP_TILE_MAX_SEEDS).all(), "an unstamped tile has more live seeds than a warp tile takes"
    bw, bh = tl[:, 10] & 0xffff, tl[:, 10] >> 16
    sw, rows = tl[:, 11] & 0xffff, tl[:, 11] >> 16
    zeff, sparse = tl[:, 13] & 0xff, ((tl[:, 13] >> 8) & 1).astype(bool)
    edge = np.zeros((ty, tx), bool)
    edge[[0, 0, -1, -1, 0, -1, ty // 2, ty // 2], [0, -1, 0, -1, tx // 2, tx // 2, 0, -1]] = True
    cats = {
        "overflow": searched & ~sparse & ((bw > sw) | (bh > rows)),
        "split": searched & (zeff > 1),
        "sparse": searched & sparse,
        "warp": ~stamped & (live > 0),
        "edge": edge.ravel(),
    }
    work = np.where(stamped, tl[:, 7], live)
    cats["_work"] = work
    cats["_live"] = live
    return cats


def pick_tiles(cats, must=None, cap=SAMPLE_TILES):
    """The given tiles, the corner and edge tiles, up to PER_CATEGORY tiles of each path (spread over the image),
    then the busiest tiles, SAMPLE_TILES in all."""
    n = len(cats["_work"])
    chosen = np.zeros(n, bool)
    if must is not None:
        chosen |= must
    for name in ("edge", "overflow", "split", "sparse", "warp"):
        idx = np.nonzero(cats[name] & ~chosen)[0]
        room = cap - int(chosen.sum())
        k = min(len(idx), PER_CATEGORY, max(room, 0))
        if k:
            chosen[idx[np.linspace(0, len(idx) - 1, k).round().astype(int)]] = True
    room = cap - int(chosen.sum())
    busiest = np.zeros(n, bool)
    if room > 0:
        order = np.argsort(np.where(chosen, -1, cats["_work"]), kind="stable")[::-1][:room]
        busiest[order[cats["_work"][order] > 0]] = True
    cats["busiest"] = busiest
    return chosen | busiest


def tiles_to_pixels(tiles, W, H):
    tx, ty = _tiles(W, H)
    m = np.repeat(np.repeat(tiles.reshape(ty, tx), TILE_H, axis=0), TILE_W, axis=1)
    return m[:H, :W]


def pixels_to_tiles(mask, W, H):
    tx, ty = _tiles(W, H)
    m = np.zeros((ty * TILE_H, tx * TILE_W), bool)
    m[:H, :W] = mask
    return m.reshape(ty, TILE_H, tx, TILE_W).any(axis=(1, 3)).ravel()


def sample_mask(cats, W, H, must=None):
    return tiles_to_pixels(pick_tiles(cats, must), W, H)


def record(name, label, cats, mask, cache, W, H):
    """Print and count the paths the sampled tiles took and the capped segments the float64 search met."""
    tiles = pixels_to_tiles(mask, W, H)
    counts = {c: int((cats[c] & tiles).sum()) for c in ("overflow", "split", "sparse", "warp", "edge")}
    counts["all_overflow"] = int(cats["overflow"].sum())
    counts["all_split"] = int(cats["split"].sum())
    counts["all_sparse"] = int(cats["sparse"].sum())
    counts["all_warp"] = int(cats["warp"].sum())
    counts["sample_tiles"] = int(tiles.sum())
    counts["sample_live_seeds"] = int(cats["_live"][tiles].sum())
    S = cache.get("search")
    counts["capped"] = int((S["has"].sum(axis=1) >= MAX_CAND).sum()) if S is not None else 0
    counts["busiest"] = int((cats["busiest"] & tiles).sum())
    print(f"[paths] {name} {label}: {counts}")
    for c in CATEGORIES:
        REACHED[name][c] += counts[c]
    return counts


class Recorded:
    """A recorded update served the way _check reads a handle."""

    def __init__(self, post, matches):
        self.post, self.matches = post, matches

    def downloadDepthmap(self):
        return self.post["mu"]

    def downloadSigmaSq(self):
        return self.post["sigma_sq"]

    def downloadA(self):
        return self.post["a"]

    def downloadB(self):
        return self.post["b"]

    def downloadConvergence(self):
        return self.post["conv"]

    def downloadEpipolarMatches(self):
        return self.matches


def check(name, fr, pre, g, mask, trust_conv=True, cache=None):
    """_check with the ambiguity bars of a sampled frame, which differ from _check's single bar (ambiguous <= 0.1 %
    of the searched seeds) as DESIGN.md 5.3 states: no failing seed; ambiguous seeds in the sample <= 0.1 % of the
    searched seeds; ambiguous seeds of the state check outside the sample (trust_conv=False reclassifies every seed
    of the frame) <= 0.01 % of the frame.  Seeds whose NCC score the float64 bound cannot pin down (flat patches of
    the synthetic scene's textureless areas, where the busiest tiles are) are counted apart: <= 1 % of the searched
    seeds."""
    rep = _check(name, fr, pre, g, trust_conv=trust_conv, cache=cache, search_mask=mask, expect_fail=True)
    assert rep.n_fail == 0, f"{name}: {rep}"
    amb = rep.ambiguous.reshape(mask.shape)
    und = (rep.undetermined if rep.undetermined is not None else np.zeros(amb.size, bool)).reshape(mask.shape)
    n_sample, n_rest, n_und = int((amb & mask & ~und).sum()), int((amb & ~mask).sum()), int(und.sum())
    print(f"{name}: ambiguous {n_sample} in the sample, {n_rest} elsewhere, {n_und} undetermined")
    assert n_sample <= max(1, 0.001 * rep.n_updated), f"{name}: {rep}"
    assert n_rest <= 0.0001 * rep.n_checked, f"{name}: {rep}"
    assert n_und <= max(1, 0.01 * rep.n_updated), f"{name}: {rep}"
    return rep


# ------------------------------------------------------------------------------------------ sequence states

@pytest.mark.parametrize("name,n", [(c, n) for c in CONFIGS for n in FRAMES])
def test_sequence_state(runs, name, n):
    """One update from the sequence's own state: every seed's state, the float64 search and update on the tile
    sample.  The same update with and without the debug timeline agrees bit for bit (Run.checked)."""
    run = runs(name)
    rec = run.checked(n)
    cache = {}
    check(f"{name} frame {n}", run.frame_model(n), rec["pre"], Recorded(rec["post"], rec["matches"]), rec["mask"],
          cache=cache)
    record(name, f"frame {n}", rec["cats"], rec["mask"], cache, run.W, run.H)
    CHECKED[name].add(("sequence", n))


# ------------------------------------------------------------------------------------------ fresh blocks

def fresh_rects(W, H):
    """About 64 x 48 each: one interior and tile-aligned, one touching the right and bottom borders, one straddling
    tile rows and columns."""
    return [(W // 2 - W // 2 % TILE_W, H // 2 - H // 2 % TILE_H, 64, 48), (W - 64, H - 48, 64, 48),
            (W // 4 + 17, H // 3 + 4, 64, 48)]


def fresh_state(run, n):
    """The sequence's state before frame n with the rectangles reset to setReferenceImage's prior, convergence
    UPDATE there; returns (state, rectangle mask)."""
    st = {k: v.copy() for k, v in run.checked(n)["pre"].items()}
    prior = run.prior()
    sel = np.zeros((run.H, run.W), bool)
    for x, y, w, h in fresh_rects(run.W, run.H):
        sel[y:y + h, x:x + w] = True
    for k in ("mu", "sigma_sq", "a", "b"):
        st[k][sel] = prior[k][sel]
    st["conv"][sel] = F.UPDATE
    return st, sel


def upload(run, st, knobs=()):
    g = _handle(run.seq, run.patch, knobs)
    run.case.start(g)
    for fid, k in STATE_FIELDS:
        g.uploadState(fid, st[k])
    g.uploadState(rmd.FIELD_CONVERGENCE, st["conv"])
    pre = _snap(g)
    assert _same_state(pre, st)
    return g, pre


@pytest.mark.parametrize("name,n", [(c, n) for c in CONFIGS for n in FRESH_FRAMES])
def test_fresh_blocks(runs, name, n):
    """Rectangles of prior seeds late in the sequence: full 143-candidate segments whose tiles overflow the strip.
    The upload drops the trusted convergence map, the work list and seed-major mode, so every seed is
    reclassified (trust_conv=False)."""
    run = runs(name)
    st, sel = fresh_state(run, n)
    g, pre = upload(run, st, [(rmd.OPT_DEBUG_TIMELINE, 1)])
    fr = run.frame_model(n)
    g.update(run.image(n), run.poses[n])
    post = _snap(g)
    # the product configuration (no timeline) of the same reclassifying update gives the same result
    g0, _ = upload(run, st)
    g0.update(run.image(n), run.poses[n])
    assert _same_state(_snap(g0), post), f"{name} fresh blocks, frame {n}: the timeline changed the update"
    assert _same_matches(post, g0.downloadEpipolarMatches(), g.downloadEpipolarMatches())
    del g0
    # the fresh seeds' tiles lead the sample; the other paths fill it up
    cats = tile_categories(g.downloadTimeline(), post, run.W, run.H)
    mask = sample_mask(cats, run.W, run.H, must=pixels_to_tiles(sel, run.W, run.H))
    cache = {}
    check(f"{name} fresh blocks, frame {n}", fr, pre, g, mask, trust_conv=False, cache=cache)
    counts = record(name, f"fresh blocks, frame {n}", cats, mask, cache, run.W, run.H)
    rect_tiles = pixels_to_tiles(sel, run.W, run.H)
    assert (cats["overflow"] & rect_tiles).any(), "no tile of the fresh blocks overflowed the strip"
    assert counts["capped"] > 0
    CHECKED[name].add(("fresh", n))


# ------------------------------------------------------------------------------------------ planted bugs

PLANTED_FRAME = 200
PLANTED_MAX_SEEDS = 12000


def _weight_step_share(S, patch):
    """Share of the searched candidates whose eps includes the score change of one 1/256 weight step: those whose
    frac * 256 lies within 1e-3 + 256 * pos_err of a rounding boundary (f64_depth_filter.search)."""
    acc = S["acc_any"]
    with np.errstate(invalid="ignore"):
        window = 1e-3 + 256.0 * S["pos_err"]
        gaps = [np.abs((S[k] - patch // 2) * 256 - np.floor((S[k] - patch // 2) * 256) - 0.5) for k in ("px", "py")]
        step = acc & ((gaps[0] <= window) | (gaps[1] <= window))
    return float(step.sum() / max(1, acc.sum())), float(np.median(S["pos_err"][acc]))


@pytest.mark.parametrize("bits", [7, 6, 5])
def test_planted_tex_bits_c4(runs, bits):
    """Texture weights with `bits` fractional bits instead of 8, from the 1080p 7x7 fresh-block state of frame
    PLANTED_FRAME.  The float64 search runs on every seed whose match or state the planted kernel changed against the
    8-bit kernel (up to PLANTED_MAX_SEEDS): a seed it left alone has the 8-bit kernel's result.  The bug must change
    matches (it is reached).  With 6 and 5 bits (weights off by up to 3/256 and 7/256) the check must catch it.  With
    7 bits (off by <= 1/256) it is reported, not asserted: at this shape the derived position error of a candidate
    (median ~1e-3 px) puts most candidates' weights within reach of a rounding boundary, so eps includes a full 1/256
    weight step for them and a 1/256 error is inside the bound -- the measured loss of sensitivity, printed."""
    run = runs("c4")
    n = PLANTED_FRAME
    st, _ = fresh_state(run, n)
    g8, pre = upload(run, st)
    g8.update(run.image(n), run.poses[n])
    post8, m8 = _snap(g8), g8.downloadEpipolarMatches()
    del g8
    g, _ = upload(run, st, [(rmd.OPT_TEX_FRAC_BITS, bits)])
    g.update(run.image(n), run.poses[n])
    post, m = _snap(g), g.downloadEpipolarMatches()
    upd = (post["conv"] == F.UPDATE) | (post8["conv"] == F.UPDATE)
    moved = (post["conv"] != post8["conv"]) | (upd & np.any(m.view(np.int32) != m8.view(np.int32), axis=2))
    assert moved.any(), f"{bits}-bit weights changed no match: the planted bug was not reached"
    idx = np.flatnonzero(moved)
    if len(idx) > PLANTED_MAX_SEEDS:
        idx = idx[np.linspace(0, len(idx) - 1, PLANTED_MAX_SEEDS).round().astype(int)]
    mask = np.zeros(moved.shape, bool)
    mask.ravel()[idx] = True
    cache = {}
    rep = _check(f"c4 fresh blocks, frame {n}, {bits}-bit weights ({int(moved.sum())} seeds changed, {len(idx)} "
                 f"searched)", run.frame_model(n), pre, Recorded(post, m), trust_conv=False, cache=cache,
                 search_mask=mask, expect_fail=True)
    share, pos_err = _weight_step_share(cache["search"], run.patch)
    caught = rep.fail.get("search", 0)
    print(f"[planted] c4 {bits}-bit weights: {int(moved.sum())} seeds changed, {caught} caught; eps includes a "
          f"weight step for {100 * share:.1f} % of the searched candidates (median position error {pos_err:.2e} px)")
    if bits <= 6:
        assert caught >= 1, f"the planted {bits}-bit weights were not caught: {rep}"


# ------------------------------------------------------------------------------------------ organisations

@pytest.mark.parametrize("n", [40, 499])
def test_organisations_c4(runs, n):
    """The c4 sequence state through every organisation of the kernel: each agrees with the default staged run bit
    for bit (state and matches).  The float64 search is shared; an organisation whose output equals one already
    checked bit for bit has the same report, so the float64 check runs once per distinct output."""
    run = runs("c4")
    rec = run.checked(n)
    fr = run.frame_model(n)
    cache, checked, differ = {}, [], []
    for name, knobs in ORGS.items():
        g = _handle(run.seq, run.patch, knobs)
        run.case.start(g)
        for k in range(1, n):
            g.update(run.image(k), run.poses[k])
        pre = _snap(g)
        assert _same_state(pre, rec["pre"]), f"{name}: pre-state differs from the sequence's"
        g.update(run.image(n), run.poses[n])
        post, m = _snap(g), g.downloadEpipolarMatches()
        same = _same_state(post, rec["post"]) and _same_matches(post, m, rec["matches"])
        if not same:
            differ.append(name)
        if not checked or not same:
            check(f"c4 {name}, frame {n}", fr, pre, Recorded(post, m), rec["mask"], cache=cache)
            checked.append(name)
        print(f"c4 {name}, frame {n}: bit-identical to the sequence's staged update: {same}")
        del g
    assert not differ, f"organisations that differ from the staged update: {differ}"


# ------------------------------------------------------------------------------------------ paths bench.py times

SEED_FRAMES_MAX = 16   # depth_filter.cuh: updateDeviceBatch enqueues its frames in groups of at most this many


def _chained_launches(n_frames, chain):
    """Launches of one updateDeviceBatch call: each group of SEED_FRAMES_MAX frames in launches of `chain` frames."""
    groups = [min(SEED_FRAMES_MAX, n_frames - i) for i in range(0, n_frames, SEED_FRAMES_MAX)]
    return sum((m + chain - 1) // chain for m in groups)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_bench_paths(runs, name):
    """What bench.py times, against the host float path over frames 1 .. CHAIN_FRAMES - 1:
    * `value`: updateDeviceBatch on device-resident float frames, RMD_OPT_CHAIN_FRAMES 8 and 3;
    * `e2e`: the Depthmap protocol with RMD_OPT_PINNED_INPUT on 8-bit frames in page-locked memory (one buffer per
      frame, DMA'd in place; untouched until the handle syncs), and the same frames from pageable memory.
    All equal bit for bit; then frame CHAIN_FRAMES through the pinned 8-bit path is checked against float64."""
    import torch
    run = runs(name)
    W, H, N = run.W, run.H, CHAIN_FRAMES
    cam = rmd.PinholeCamera(*run.seq.camera)
    dmin, dmax = run.case.dmin, run.case.dmax
    poses = run.poses[:N + 1].reshape(-1, 12)

    host = _handle(run.seq, run.patch)
    run.case.start(host)
    for k in range(1, N):
        host.update(run.image(k), poses[k])
    want = _snap(host)

    dense = torch.from_numpy(np.stack([run.image(k) for k in range(N)])).to("cuda")
    assert dense.stride(1) == W and dense.data_ptr() % 16 == 0
    got = {}
    for chain in (8, 3):
        g = rmd.SeedMatrix(W, H, cam, patch_side=run.patch)
        g.setOption(rmd.OPT_CHAIN_FRAMES, chain)
        g.setReferenceImageDevice(dense[0].data_ptr(), W * 4, poses[0], dmin, dmax)
        if chain == 8:
            g.updateDeviceBatch(dense[1].data_ptr(), W * H * 4, W * 4, poses[1:N])
            assert g.launchCount()[0] == _chained_launches(N - 1, 8)
        else:   # two calls: chains restart cleanly
            g.updateDeviceBatch(dense[1].data_ptr(), W * H * 4, W * 4, poses[1:20])
            g.updateDeviceBatch(dense[20].data_ptr(), W * H * 4, W * 4, poses[20:N])
            assert g.launchCount()[0] == _chained_launches(19, 3) + _chained_launches(N - 20, 3)
        g.sync()
        got[f"chain of {chain}"] = _snap(g)
    del dense
    torch.cuda.synchronize()

    fx, fy, cx, cy = run.seq.camera
    pinned = [torch.from_numpy(run.u8[k]).pin_memory() for k in range(N + 1)]
    dms = {}
    for label, frames in (("pinned 8-bit", [p.numpy() for p in pinned]), ("pageable 8-bit", list(run.u8[:N + 1]))):
        dm = rmd.Depthmap(W, H, fx, cx, fy, cy, patch_side=run.patch)
        dm.seeds_.setOption(rmd.OPT_PINNED_INPUT, 1)
        dm.seeds_.setOption(rmd.OPT_RECORD_MATCHES, 1)
        dm.setReferenceImage(frames[0], run.poses[0], dmin, dmax)
        for k in range(1, N):
            dm.update(frames[k], run.poses[k])
        dm.seeds_.sync()
        got[label] = _snap(dm.seeds_)
        dms[label] = (dm, frames)
    for label, S in got.items():
        assert _same_state(S, want), f"{name}: {label} differs from the host float path"
        print(f"{name}: {label} == host float path over frames 1..{N - 1}, bit for bit")

    # frame N through the pinned path, recorded and checked; the float path must agree with it
    dm, frames = dms["pinned 8-bit"]
    dm.seeds_.setOption(rmd.OPT_DEBUG_TIMELINE, 1)
    pre = _snap(dm.seeds_)
    dm.update(frames[N], run.poses[N])
    dm.seeds_.sync()
    post, matches = _snap(dm.seeds_), dm.seeds_.downloadEpipolarMatches()
    host.update(run.image(N), poses[N])
    assert _same_state(post, _snap(host)), f"{name}: frame {N} through the pinned 8-bit path differs from the float path"
    cats = tile_categories(dm.seeds_.downloadTimeline(), post, W, H)
    mask = sample_mask(cats, W, H)
    fr = run.case.frame_model(ob.u8_to_float(run.u8[N]), poses[N], run.patch)
    cache = {}
    check(f"{name} frame {N}, pinned 8-bit input", fr, pre, Recorded(post, matches), mask, cache=cache)
    record(name, f"frame {N}, pinned 8-bit input", cats, mask, cache, W, H)
    del dms, dm
    del pinned


# The host profile (rmd_debug_host_profile) is switched on by RMD_HOST_PROFILE when the library loads, so it is read
# in a process of its own.  Slot 1 is the time of the staging copy into the pinned ring, slot 6 counts updates.
_PROFILE_SCRIPT = r"""
import ctypes, sys
import numpy as np
import torch
import rpg_open_remode_b200 as rmd
from rpg_open_remode_b200 import _native
W, H, n = int(sys.argv[1]), int(sys.argv[2]), 4
frames = np.random.default_rng(0).integers(0, 256, (n, H, W), dtype=np.uint8)
pinned = [torch.from_numpy(f).pin_memory() for f in frames]
T = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
prof = (ctypes.c_double * 8)()
for label, fs in (("pinned", [p.numpy() for p in pinned]), ("pageable", list(frames))):
    dm = rmd.Depthmap(W, H, 1000.0, W / 2, 1000.0, H / 2)
    dm.seeds_.setOption(rmd.OPT_PINNED_INPUT, 1)
    dm.setReferenceImage(fs[0], T, 1.0, 5.0)
    dm.seeds_.sync()
    _native.lib().rmd_debug_host_profile(prof, 1)
    for k in range(1, n):
        T[0, 3] = 0.01 * k
        dm.update(fs[k], T)
    dm.seeds_.sync()
    _native.lib().rmd_debug_host_profile(prof, 1)
    print(label, prof[1], prof[6])
"""


@pytest.mark.parametrize("name", list(CONFIGS))
def test_pinned_input_is_dma_in_place(name):
    """RMD_OPT_PINNED_INPUT on page-locked 8-bit frames takes the in-place DMA branch (no staging copy), and the same
    option on pageable frames stages them: the equality of test_bench_paths compares two different paths."""
    import os
    import subprocess
    import sys
    W, H = CONFIGS[name][:2]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", _PROFILE_SCRIPT, str(W), str(H)], cwd=root, capture_output=True,
                         text=True, env=dict(os.environ, RMD_HOST_PROFILE="1"), timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    prof = {ln.split()[0]: (float(ln.split()[1]), float(ln.split()[2])) for ln in out.stdout.splitlines()
            if ln.split() and ln.split()[0] in ("pinned", "pageable")}
    print(f"{name}: staging copy seconds / updates: {prof}")
    assert prof["pinned"] == (0.0, 3.0), prof
    assert prof["pageable"][0] > 0.0 and prof["pageable"][1] == 3.0, prof


# ------------------------------------------------------------------------------------------ coverage

@pytest.mark.parametrize("name", list(CONFIGS))
def test_paths_reached(name):
    """Every path of the staged kernel this file exists for was sampled and checked at both shapes."""
    want = {("sequence", n) for n in FRAMES} | {("fresh", n) for n in FRESH_FRAMES}
    missing = sorted(want - CHECKED[name])
    assert not missing, f"{name}: run the whole module; these checks did not run: {missing}"
    got = dict(REACHED[name])
    print(f"[paths] {name} over all checks: {got}")
    for c in CATEGORIES:
        assert got.get(c, 0) > 0, f"{name}: no sampled tile took the {c} path: {got}"
