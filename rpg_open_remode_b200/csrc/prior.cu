// prior.cu -- see prior.cuh.  Both kernels touch a few bytes per pixel once per keyframe (HBM-bound).
#include "point_cloud.cuh"
#include "prior.cuh"

namespace rmdb
{

namespace
{

// One thread per source pixel.  IEEE round-to-nearest operations throughout, so that the CPU restatement
// (oracle/rmd_oracle_propagate.c) reproduces every z-buffer entry bit for bit.
__global__ void __launch_bounds__(256) prior_splat_kernel(const PriorSplatParams P)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if(x >= P.src_width || y >= P.src_height)
    return;
  if(P.conv[(size_t)y * P.conv_stride + x] != RMD_CONVERGED)
    return;
  const float mu = P.seed[(size_t)y * P.seed_stride + x].x;
  const float3 w = back_project(P.src_cam, P.T_world_ref, x, y, mu);   // == the published point
  // p = T_curr_world * w: rotation, then translation (SE3::operator*)
  const float *T = P.T_curr_world.m;
  const float px = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], w.x), __fmul_rn(T[1], w.y)), __fmul_rn(T[2], w.z)), T[3]);
  const float py = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], w.x), __fmul_rn(T[5], w.y)), __fmul_rn(T[6], w.z)), T[7]);
  const float pz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], w.x), __fmul_rn(T[9], w.y)), __fmul_rn(T[10], w.z)), T[11]);
  if(!(pz > 0.0f))
    return;
  // depth = distance along the ray, as seed_update defines it
  const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
  if(!(d >= P.min_depth && d <= P.max_depth))   // also drops NaN
    return;
  const float u = __fadd_rn(__fdiv_rn(__fmul_rn(P.dst_cam.fx, px), pz), P.dst_cam.cx);
  const float v = __fadd_rn(__fdiv_rn(__fmul_rn(P.dst_cam.fy, py), pz), P.dst_cam.cy);
  const float tu = floorf(__fadd_rn(u, 0.5f)), tv = floorf(__fadd_rn(v, 0.5f));   // pixel centres are integers
  if(!(tu >= 0.0f && tu < (float)P.dst_width && tv >= 0.0f && tv < (float)P.dst_height))
    return;
  // d > 0: its bit pattern orders like the float, so the nearest surface wins whatever the thread order
  atomicMin(P.zbuf + (size_t)(int)tv * P.dst_width + (int)tu, __float_as_uint(d));
}

__global__ void __launch_bounds__(256) prior_apply_kernel(const PriorApplyParams P)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if(x >= P.width || y >= P.height)
    return;
  const unsigned int z = P.zbuf[(size_t)y * P.width + x];
  if(z == 0xFFFFFFFFu || P.conv[(size_t)y * P.conv_stride + x] == RMD_BORDER)
    return;
  // a = b = 10: inlier ratio 0.5, so the seed cannot be CONVERGED before new frames confirm it
  P.seed[(size_t)y * P.seed_stride + x] = make_float4(__uint_as_float(z), P.sigma_sq, 10.0f, 10.0f);
}

dim3 grid_for(int width, int height, dim3 block)
{
  return dim3((width + block.x - 1) / block.x, (height + block.y - 1) / block.y);
}

} // namespace

cudaError_t launch_prior_splat(const PriorSplatParams &P, cudaStream_t stream)
{
  const dim3 block(32, 8);
  prior_splat_kernel<<<grid_for(P.src_width, P.src_height, block), block, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_prior_apply(const PriorApplyParams &P, cudaStream_t stream)
{
  const dim3 block(32, 8);
  prior_apply_kernel<<<grid_for(P.width, P.height, block), block, 0, stream>>>(P);
  return cudaGetLastError();
}

} // namespace rmdb
