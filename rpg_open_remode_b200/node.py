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


class DepthmapNode:
    """rmd::DepthmapNode::denseInputCallback with the ROS plumbing removed.  `publisher` receives
    ("depthmap_and_pointcloud", depthmap) after a keyframe is finished (denoiseAndPublishResults,
    src/depthmap_node.cpp:165-173) and ("convergence", depthmap) every publish_conv_every_n messages
    (:157-161, :175-183)."""

    def __init__(self, depthmap: Depthmap, ref_compl_perc: float = 10.0, max_dist_from_ref: float = 0.5,
                 publish_conv_every_n: int = 10, publisher: Optional[Callable] = None,
                 volume: Optional[TsdfVolume] = None, prior_from_volume: float = 0.0, follow_volume: bool = False,
                 scene_mesh: Optional[SceneMesh] = None, esdf: bool = False, esdf_camera_margin: int = 0):
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
                    self.depthmap_.priorFromVolume(self.volume_, self.prior_from_volume_)
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
