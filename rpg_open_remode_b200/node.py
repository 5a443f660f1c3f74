"""The caller of the hot path: rmd::DepthmapNode's keyframe state machine (SURVEY.md 8f row 2)
without ROS, and a set of several live keyframes fed by one frame stream.

  DepthmapNode   src/depthmap_node.cpp:36-183 + include/rmd/depthmap_node.h:30-62: TAKE_REFERENCE_FRAME /
                 UPDATE, re-keyframing when the converged percentage or the distance from the reference
                 passes its threshold, then denoise(0.5, 200) + convergence download + publish.
  KeyframeSet    what the reference cannot do (one rmd::Depthmap, so the map of a keyframe stops growing
                 the moment the next one starts): up to `n` keyframes stay live and every frame updates all of
                 them through rmd_seeds_update_many -- one upload, one fused kernel per keyframe, overlapping
                 on the GPU.

Host logic only: everything numeric happens behind rpg_open_remode_b200.api (the C-ABI).
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np

from .api import PRIOR_SIGMA_SQ_FRAC, SE3, Depthmap, SceneMesh, SeedMatrix, TsdfVolume

UPDATE, TAKE_REFERENCE_FRAME = 0, 1   # rmd::ProcessingStates::State, include/rmd/depthmap_node.h:32-36


def esdf_camera_box(dims, voxel_size: float, origin, camera_centre, margin: int):
    """DepthmapNode's ESDF box with esdf_camera_margin = margin > 0: (lo int64 [3], dims int64 [3]) in window indices,
    the bounding box of the window [0, dims) and of [c - margin, c + margin] with c = round((camera_centre - origin) /
    voxel_size) in float64, followVolume's conversion to window indices."""
    c = np.round((np.asarray(camera_centre, np.float64) - np.asarray(origin, np.float32).astype(np.float64))
                 / float(voxel_size)).astype(np.int64)
    n = np.asarray(dims, np.int64)
    lo = np.minimum(0, c - int(margin))
    return lo, np.maximum(n, c + int(margin) + 1) - lo


def _unit_max(u, X, Y):
    """max of u . q over the unit directions q of the pixel cone {l (x, y, 1): x in [X0, X1], y in [Y0, Y1], l > 0}:
    a linear function on a spherical polygon peaks at a corner ray, at u's own direction projected onto a side plane
    when that lies within the side, or at u's direction when that lies within the cone."""
    (X0, X1), (Y0, Y1) = X, Y
    cands = [np.array([x, y, 1.0]) for x in (X0, X1) for y in (Y0, Y1)]
    # the side x = X: the plane spanned by (X, 0, 1) and (0, 1, 0); likewise y = Y
    for X_ in (X0, X1):
        nrm = np.array([1.0, 0.0, -X_])
        p = u - (u @ nrm) / (nrm @ nrm) * nrm
        if p[2] > 0.0 and Y0 <= p[1] / p[2] <= Y1:
            cands.append(p)
    for Y_ in (Y0, Y1):
        nrm = np.array([0.0, 1.0, -Y_])
        p = u - (u @ nrm) / (nrm @ nrm) * nrm
        if p[2] > 0.0 and X0 <= p[0] / p[2] <= X1:
            cands.append(p)
    if u[2] > 0.0 and X0 <= u[0] / u[2] <= X1 and Y0 <= u[1] / u[2] <= Y1:
        cands.append(u)
    return max(float(u @ c) / float(np.linalg.norm(c)) for c in cands if np.linalg.norm(c) > 0.0)


def prior_view_box(dims, voxel_size: float, origin, camera, width: int, height: int, T_world_ref, max_depth: float):
    """DepthmapNode's prior box with prior_view_box=True: (lo int64 [3], dims int64 [3]) in window indices of the
    smallest box of whole voxels that contains the camera centre c and every point c + t q for the unit ray q of any
    pixel position in [0, width - 1] x [0, height - 1] and t in [0, max_depth + voxel_size], plus one voxel on every
    face for the trilinear corners (DESIGN.md 4.8).  dims: the window's (checked; the box does not depend on them);
    camera: (fx, fy, cx, cy) or a PinholeCamera; T_world_ref: 3x4 camera -> world.  Float64 throughout, from closed-form
    extremes per world axis, with esdf_camera_box's conversion to window indices.  The camera centre lies inside the
    box, so the rays the box prior marches start at the camera and are sampled at t = k * voxel_size whatever the
    box."""
    n = np.asarray(dims).reshape(-1)
    if len(n) != 3 or any(int(x) != x or x <= 0 for x in n):
        raise ValueError("prior_view_box: dims must be three whole numbers > 0")
    s = float(voxel_size)
    if not (np.isfinite(s) and s > 0.0):
        raise ValueError("prior_view_box: voxel_size must be finite and > 0")
    o = np.asarray(origin, np.float32).astype(np.float64).reshape(-1)
    if len(o) != 3 or not np.all(np.isfinite(o)):
        raise ValueError("prior_view_box: origin must be three finite numbers")
    fx, fy, cx, cy = ((camera.fx, camera.fy, camera.cx, camera.cy) if hasattr(camera, "fx")
                      else (float(x) for x in camera))
    if not all(np.isfinite([fx, fy, cx, cy])) or fx == 0.0 or fy == 0.0:
        raise ValueError("prior_view_box: the camera needs finite intrinsics and fx, fy != 0")
    if int(width) != width or int(height) != height or width < 1 or height < 1:
        raise ValueError("prior_view_box: width and height must be whole numbers >= 1")
    T = np.asarray(getattr(T_world_ref, "data", T_world_ref), np.float64).reshape(3, 4)
    if not np.all(np.isfinite(T)):
        raise ValueError("prior_view_box: T_world_ref must be finite")
    if not (np.isfinite(max_depth) and max_depth > 0.0):
        raise ValueError("prior_view_box: max_depth must be finite and > 0")
    X = sorted(((0.0 - cx) / fx, (width - 1.0 - cx) / fx))
    Y = sorted(((0.0 - cy) / fy, (height - 1.0 - cy) / fy))
    R, c = T[:, :3], T[:, 3]
    reach = float(max_depth) + s
    lo_w, hi_w = np.empty(3), np.empty(3)
    for a in range(3):
        u = R[a]   # (R q)_a = u . q
        lo_w[a] = c[a] + reach * min(0.0, -_unit_max(-u, X, Y))
        hi_w[a] = c[a] + reach * max(0.0, _unit_max(u, X, Y))
    lo = np.floor((lo_w - o) / s).astype(np.int64) - 1
    hi = np.ceil((hi_w - o) / s).astype(np.int64) + 1
    return lo, hi - lo + 1


class DepthmapNode:
    """rmd::DepthmapNode::denseInputCallback with the ROS plumbing removed.  `publisher` receives
    ("depthmap_and_pointcloud", depthmap) after a keyframe is finished (denoiseAndPublishResults,
    src/depthmap_node.cpp:165-173) and ("convergence", depthmap) every publish_conv_every_n messages
    (:157-161, :175-183)."""

    def __init__(self, depthmap: Depthmap, ref_compl_perc: float = 10.0, max_dist_from_ref: float = 0.5,
                 publish_conv_every_n: int = 10, publisher: Optional[Callable] = None,
                 volume: Optional[TsdfVolume] = None, prior_from_volume: float = 0.0, follow_volume: bool = False,
                 scene_mesh: Optional[SceneMesh] = None, esdf: bool = False, esdf_camera_margin: int = 0,
                 prior_view_box: bool = False):
        if prior_view_box and not prior_from_volume:
            raise ValueError("DepthmapNode: prior_view_box needs prior_from_volume > 0")
        if esdf_camera_margin and not esdf:
            raise ValueError("DepthmapNode: esdf_camera_margin needs esdf=True")
        if int(esdf_camera_margin) != esdf_camera_margin or esdf_camera_margin < 0:
            raise ValueError("DepthmapNode: esdf_camera_margin must be a whole number of voxels >= 0")
        if prior_from_volume and volume is None:
            raise ValueError("DepthmapNode: prior_from_volume needs a volume")
        if follow_volume and volume is None:
            raise ValueError("DepthmapNode: follow_volume needs a volume")
        if esdf and volume is None:
            raise ValueError("DepthmapNode: esdf needs a volume")
        if scene_mesh is not None and not follow_volume:
            raise ValueError("DepthmapNode: scene_mesh needs follow_volume=True")
        if scene_mesh is not None and getattr(volume, "store", False):
            raise ValueError("DepthmapNode: scene_mesh would add a revisited region of a volume with the brick store "
                             "twice; mesh its map with volume.mapMesh()")
        if not 0.0 <= prior_from_volume <= 1.0:
            raise ValueError("DepthmapNode: prior_from_volume must be in [0, 1] (0 = off)")
        self.depthmap_ = depthmap
        self.volume_ = volume   # when given, every finished keyframe is fused into it (DESIGN.md 4.8)
        # sigma^2 fraction of the new keyframe's prior raycast from volume_ (0 = off)
        self.prior_from_volume_ = float(prior_from_volume)
        # when set, that raycast marches the box around the new keyframe's view (prior_view_box), brick store
        # included, instead of the window
        self.prior_view_box_ = bool(prior_view_box)
        # when set, volume_ is shifted to stay around each keyframe's view before it is fused (DESIGN.md 4.8), and
        # the surface that leaves it is published as ("volume_spill", (points, intensity or None, normals))
        self.follow_volume_ = bool(follow_volume)
        # when given, the spill mesh of every shift is added to it, so that scene_mesh.mesh(volume) meshes the whole
        # traversed scene
        self.scene_mesh_ = scene_mesh
        # when set, the volume's ESDF is recomputed after each keyframe is fused and published as ("volume_esdf",
        # volume), ready for esdfQuery
        self.esdf_ = bool(esdf)
        # when > 0, that ESDF covers the bounding box of the window and the cube of this half-side (voxels) around the
        # finished keyframe's camera, so that the camera -- outside a following window -- can query it
        self.esdf_camera_margin_ = int(esdf_camera_margin)
        self.ref_depth_range_ = (0.0, 0.0)   # [min_depth, max_depth] of the current keyframe
        self.state_ = TAKE_REFERENCE_FRAME                      # src/depthmap_node.cpp:35
        self.ref_compl_perc_ = float(ref_compl_perc)            # :81, default 10.0
        self.max_dist_from_ref_ = float(max_dist_from_ref)      # :82, default 0.5
        self.publish_conv_every_n_ = int(publish_conv_every_n)  # :83, default 10
        self.num_msgs_ = 0
        self.publisher_ = publisher

    def denseInputCallback(self, img_8uc1, T_world_curr: SE3, min_depth: float, max_depth: float) -> None:
        self.num_msgs_ += 1                                                       # :92
        if self.depthmap_ is None:
            raise RuntimeError("depthmap not initialized")                        # :93-97
        T_curr_world = T_world_curr.inv()                                         # :128, :142
        if self.state_ == TAKE_REFERENCE_FRAME:
            if self.depthmap_.setReferenceImage(img_8uc1, T_curr_world, min_depth, max_depth):
                self.state_ = UPDATE                                              # :126-135
                self.ref_depth_range_ = (float(min_depth), float(max_depth))
                if self.prior_from_volume_:   # the volume holds every keyframe published so far
                    box = self.priorViewBox(max_depth) if self.prior_view_box_ else (None, None)
                    self.depthmap_.priorFromVolume(self.volume_, self.prior_from_volume_, *box)
        elif self.state_ == UPDATE:
            self.depthmap_.update(img_8uc1, T_curr_world)                         # :142
            perc_conv = self.depthmap_.getConvergedPercentage()                   # :143
            dist_from_ref = self.depthmap_.getDistFromRef()                       # :144
            if perc_conv > self.ref_compl_perc_ or dist_from_ref > self.max_dist_from_ref_:   # :146
                self.state_ = TAKE_REFERENCE_FRAME
                self.denoiseAndPublishResults()
        if self.publish_conv_every_n_ < self.num_msgs_:                           # :157
            self.publishConvergenceMap()
            self.num_msgs_ = 0

    def denoiseAndPublishResults(self) -> None:
        if self.follow_volume_:
            self.followVolume()
        if self.volume_ is not None:
            # the same host map as downloadDenoisedDepthmap, and the keyframe fused from the device copy
            self.depthmap_.fuseDenoisedInto(self.volume_, 0.5, 200)
        else:
            self.depthmap_.downloadDenoisedDepthmap(0.5, 200)                     # :167
        self.depthmap_.downloadConvergenceMap()                                   # :168
        if self.publisher_:
            self.publisher_("depthmap_and_pointcloud", self.depthmap_)
        if self.esdf_:
            if self.esdf_camera_margin_:
                self.volume_.computeEsdf(*self.esdfCameraBox())
            else:
                self.volume_.computeEsdf()
            if self.publisher_:
                self.publisher_("volume_esdf", self.volume_)

    def esdfCameraBox(self):
        """(lo int64 [3], dims int64 [3]) in window indices: the bounding box of the window and of the cube of
        half-side esdf_camera_margin voxels around the finished keyframe's camera centre, which followVolume's
        conversion to window indices places at round((centre - origin) / voxel_size)."""
        v = self.volume_
        T = np.asarray(self.depthmap_.getT_world_ref().data, np.float64).reshape(3, 4)
        return esdf_camera_box(v.dims, v.voxel_size, v.origin, T[:, 3], self.esdf_camera_margin_)


    def priorViewBox(self, max_depth: float):
        """prior_view_box of the keyframe just set: its camera, image and pose, and max_depth."""
        v, g = self.volume_, self.depthmap_.seeds_
        T = np.asarray(self.depthmap_.getT_world_ref().data, np.float64).reshape(3, 4)
        return prior_view_box(v.dims, v.voxel_size, v.origin, g.cam_, g.width_, g.height_, T, max_depth)

    def followVolume(self) -> None:
        """Recentre volume_ on the finished keyframe's view centre -- the camera centre plus the middle of
        [min_depth, max_depth] along the optical axis -- on every axis where that centre lies more than n / 8 voxels
        from the grid's centre index, by the whole-voxel difference; the spill is published before the shift."""
        v = self.volume_
        T = np.asarray(self.depthmap_.getT_world_ref().data, np.float64).reshape(3, 4)
        centre = T[:, 3] + 0.5 * (self.ref_depth_range_[0] + self.ref_depth_range_[1]) * T[:, 2]
        n = np.array(v.dims, np.float64)
        off = (centre - v.origin.astype(np.float64)) / v.voxel_size - 0.5 * (n - 1.0)
        d = np.where(np.abs(off) > n / 8.0, np.clip(np.round(off), -(2.0**31 - 1), 2.0**31 - 1), 0.0).astype(np.int64)
        if not d.any():
            return
        if self.publisher_:
            spill = (v.spillPoints(d), v.spillIntensity(d) if v.intensity else None, v.spillNormals(d))
            self.publisher_("volume_spill", spill)
        if self.scene_mesh_ is not None:
            self.scene_mesh_.addSpill(v, d)
        v.shift(d)

    def publishConvergenceMap(self) -> None:
        self.depthmap_.downloadConvergenceMap()                                   # :177
        if self.publisher_:
            self.publisher_("convergence", self.depthmap_)


class KeyframeSet:
    """Up to `n` live keyframes of one camera; update() feeds a frame to all of them at once."""

    def __init__(self, width: int, height: int, camera, n: int, patch_side: int = 5, device: int = -1):
        self.seeds: List[SeedMatrix] = [SeedMatrix(width, height, camera, patch_side, device) for _ in range(n)]
        self.live: List[bool] = [False] * n

    def setReferenceImage(self, slot: int, img, T_curr_world, min_depth: float, max_depth: float,
                          prior_from: Optional[int] = None, sigma_sq_frac: float = PRIOR_SIGMA_SQ_FRAC,
                          prior_volume: Optional[TsdfVolume] = None) -> None:
        """prior_from: another live slot whose converged seeds become the new keyframe's depth prior.
        prior_volume: a TSDF volume whose raycast from the new reference pose becomes the prior where it hits (over
        prior_from's where both give one)."""
        if prior_from is not None and (prior_from == slot or not self.live[prior_from]):
            raise ValueError("KeyframeSet.setReferenceImage: prior_from must be another live slot")
        self.seeds[slot].setReferenceImage(img, T_curr_world, min_depth, max_depth)
        if prior_from is not None:
            self.seeds[slot].propagatePriorFrom(self.seeds[prior_from], sigma_sq_frac)
        if prior_volume is not None:
            self.seeds[slot].priorFromVolume(prior_volume, sigma_sq_frac)
        self.live[slot] = True

    def retire(self, slot: int) -> None:
        self.live[slot] = False

    def update(self, img, T_curr_world) -> int:
        """Returns the number of keyframes the frame went to."""
        live = [s for s, on in zip(self.seeds, self.live) if on]
        if live:
            SeedMatrix.updateMany(live, img, T_curr_world)
        return len(live)

    def convergedPercentages(self) -> np.ndarray:
        return np.array([100.0 * s.getConvergedCount() / (s.width_ * s.height_) if on else np.nan
                         for s, on in zip(self.seeds, self.live)], np.float32)
