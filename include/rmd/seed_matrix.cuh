// rmd/seed_matrix.cuh -- rmd::SeedMatrix with the reference's interface
// (include/rmd/seed_matrix.cuh:45-109): same constructor, setReferenceImage,
// update, download*, get*, getConvergedCount, getDistFromRef and (under
// RMD_BUILD_TESTS) the extra download* accessors.  A thin forwarder to the
// C-ABI (rmd_seeds_*, include/rmd_b200.h): one fused sm_90a kernel per
// update() instead of three launches and two device syncs
// (src/seed_matrix.cu:139-155).
#ifndef SEED_MATRIX_CUH
#define SEED_MATRIX_CUH

#include <cuda_runtime.h>
#include <rmd/device_image.cuh>
#include <rmd/pinhole_camera.cuh>
#include <rmd/reduction.cuh>
#include <rmd/se3.cuh>

#ifndef RMD_CORR_PATCH_SIDE
#define RMD_CORR_PATCH_SIDE 5   // CMakeLists.txt:51; 7 is also supported
#endif
#ifndef RMD_MAX_EXTENT_EPIPOLAR_SEARCH
#define RMD_MAX_EXTENT_EPIPOLAR_SEARCH 100
#endif

namespace rmd
{

namespace ConvergenceStates
{
enum ConvergenceState
{
  UPDATE = RMD_UPDATE,
  CONVERGED = RMD_CONVERGED,
  BORDER = RMD_BORDER,
  DIVERGED = RMD_DIVERGED,
  NO_MATCH = RMD_NO_MATCH,
  NOT_VISIBLE = RMD_NOT_VISIBLE
};
}
typedef ConvergenceStates::ConvergenceState ConvergenceState;

class SeedMatrix
{
public:
  SeedMatrix(const size_t &width, const size_t &height, const PinholeCamera &cam)
    : width_(width), height_(height), handle_(NULL),
      mu_(DeviceImage<float>::ViewTag(), width, height, NULL, 0),
      sigma_(DeviceImage<float>::ViewTag(), width, height, NULL, 0),
      a_(DeviceImage<float>::ViewTag(), width, height, NULL, 0),
      b_(DeviceImage<float>::ViewTag(), width, height, NULL, 0),
      convergence_(DeviceImage<int>::ViewTag(), width, height, NULL, 0)
  {
    detail::throw_on_error(rmd_seeds_create(static_cast<int>(width), static_cast<int>(height), cam.fx, cam.fy,
                                            cam.cx, cam.cy, RMD_CORR_PATCH_SIDE, -1, &handle_),
                           "SeedMatrix: unable to create");
#if RMD_BUILD_TESTS
    rmd_seeds_set_option(handle_, RMD_OPT_RECORD_MATCHES, 1);
#endif
  }

  ~SeedMatrix() { rmd_seeds_destroy(handle_); }

  bool setReferenceImage(float *host_ref_img_align_row_maj, const SE3<float> &T_curr_world,
                         const float &min_depth, const float &max_depth)
  {
    detail::throw_on_error(rmd_seeds_set_reference(handle_, host_ref_img_align_row_maj, T_curr_world.data.data,
                                                   min_depth, max_depth),
                           "SeedMatrix: unable to set the reference image");
    return true;
  }

  bool update(float *host_curr_img_align_row_maj, const SE3<float> &T_curr_world)
  {
    detail::throw_on_error(rmd_seeds_update(handle_, host_curr_img_align_row_maj, T_curr_world.data.data),
                           "SeedMatrix: unable to update");
    return true;
  }

  void downloadDepthmap(float *host_depthmap_align_row_maj) const
  {
    download(RMD_FIELD_MU, host_depthmap_align_row_maj);
  }
  void downloadConvergence(int *host_align_row_maj) const { download(RMD_FIELD_CONVERGENCE, host_align_row_maj); }

  const DeviceImage<float> &getMu() const { return view(RMD_FIELD_MU, mu_); }
  const DeviceImage<float> &getSigmaSq() const { return view(RMD_FIELD_SIGMA_SQ, sigma_); }
  const DeviceImage<float> &getA() const { return view(RMD_FIELD_A, a_); }
  const DeviceImage<float> &getB() const { return view(RMD_FIELD_B, b_); }
  const DeviceImage<int> &getConvergence() const { return view(RMD_FIELD_CONVERGENCE, convergence_); }

  size_t getConvergedCount() const
  {
    size_t n = 0;
    detail::throw_on_error(rmd_seeds_converged_count(handle_, &n), "SeedMatrix: unable to count");
    return n;
  }

  float getDistFromRef() const
  {
    float d = 0.0f;
    rmd_seeds_dist_from_ref(handle_, &d);
    return d;
  }

#if RMD_BUILD_TESTS
  void downloadSigmaSq(float *host_align_row_maj) const { download(RMD_FIELD_SIGMA_SQ, host_align_row_maj); }
  void downloadA(float *host_align_row_maj) const { download(RMD_FIELD_A, host_align_row_maj); }
  void downloadB(float *host_align_row_maj) const { download(RMD_FIELD_B, host_align_row_maj); }
  void downloadSumTempl(float *host_align_row_maj) const { download(RMD_FIELD_SUM_TEMPL, host_align_row_maj); }
  void downloadConstTemplDenom(float *host_align_row_maj) const
  {
    download(RMD_FIELD_CONST_TEMPL_DENOM, host_align_row_maj);
  }
  void downloadEpipolarMatches(float2 *host_align_row_maj) const
  {
    download(RMD_FIELD_EPIPOLAR_MATCHES, host_align_row_maj);
  }
#endif

  // Keyframe depth prior (rmd_seeds_set_prior_propagation / rmd_seeds_propagate_prior, include/rmd_b200.h):
  // in place, every later setReferenceImage starts from this keyframe's converged seeds (0 = off) ...
  void setPriorPropagation(float sigma_sq_frac)
  {
    detail::throw_on_error(rmd_seeds_set_prior_propagation(handle_, sigma_sq_frac),
                           "SeedMatrix: unable to set the prior propagation");
  }
  // ... or, right after setReferenceImage, from the converged seeds of another live keyframe.
  void propagatePriorFrom(const SeedMatrix &src, float sigma_sq_frac)
  {
    detail::throw_on_error(rmd_seeds_propagate_prior(handle_, src.handle_, sigma_sq_frac),
                           "SeedMatrix: unable to propagate the prior");
  }

  // The C-ABI handle, for rmd::DepthmapDenoiser and code that wants the
  // extended entry points (u8 frames, device-resident frames, streams).
  rmd_seeds_t *handle() const { return handle_; }

private:
  SeedMatrix(const SeedMatrix &);
  SeedMatrix &operator=(const SeedMatrix &);

  void download(int field, void *dst) const
  {
    detail::throw_on_error(rmd_seeds_download(handle_, field, dst), "SeedMatrix: unable to download");
  }

  template<typename T>
  const DeviceImage<T> &view(int field, DeviceImage<T> &img) const
  {
    void *ptr = NULL;
    size_t pitch = 0;
    detail::throw_on_error(rmd_seeds_device_ptr(handle_, field, &ptr, &pitch), "SeedMatrix: unable to export");
    img.rebind(static_cast<T*>(ptr), pitch);
    return img;
  }

  size_t width_;
  size_t height_;
  rmd_seeds_t *handle_;
  // planar views of the seed state, refreshed by the get*() accessors
  mutable DeviceImage<float> mu_, sigma_, a_, b_;
  mutable DeviceImage<int> convergence_;
};

} // rmd namespace

#endif // SEED_MATRIX_CUH
