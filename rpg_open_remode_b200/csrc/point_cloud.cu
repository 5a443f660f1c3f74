// point_cloud.cu -- see point_cloud.cuh.
#include "point_cloud.cuh"

namespace rmdb
{

namespace
{

__device__ __forceinline__ bool is_converged(const PointCloudParams &P, int i)
{
  if(i >= P.width * P.height)
    return false;
  const int y = i / P.width, x = i - y * P.width;
  return P.conv[(size_t)y * P.conv_stride + x] == RMD_CONVERGED;
}

// pass 1: converged pixels per block; the last block to finish turns the block
// totals into exclusive offsets (<= ~2000 values: one warp, serial chunks)
__global__ void __launch_bounds__(POINT_CLOUD_BLOCK) point_cloud_count_kernel(const PointCloudParams P)
{
  __shared__ unsigned int warp_sum[POINT_CLOUD_BLOCK / 32];
  __shared__ bool last;
  const int base = blockIdx.x * POINT_CLOUD_PIXELS + threadIdx.x * 4;
  unsigned int n = 0;
#pragma unroll
  for(int k = 0; k < 4; ++k)
    n += is_converged(P, base + k) ? 1u : 0u;
  n = __reduce_add_sync(0xffffffffu, n);
  if((threadIdx.x & 31) == 0)
    warp_sum[threadIdx.x >> 5] = n;
  __syncthreads();
  if(threadIdx.x == 0)
  {
    unsigned int tot = 0;
    for(int w = 0; w < POINT_CLOUD_BLOCK / 32; ++w) tot += warp_sum[w];
    P.block_counts[blockIdx.x] = tot;
    __threadfence();
    last = (atomicAdd(P.total + 1, 1u) == (unsigned int)(P.n_blocks - 1));
  }
  __syncthreads();
  if(!last || threadIdx.x >= 32)
    return;
  __threadfence();
  unsigned int running = 0;
  for(int b0 = 0; b0 < P.n_blocks; b0 += 32)
  {
    const int b = b0 + (int)threadIdx.x;
    const unsigned int c = (b < P.n_blocks) ? P.block_counts[b] : 0u;
    unsigned int inc = c;
#pragma unroll
    for(int off = 1; off < 32; off <<= 1)
    {
      const unsigned int up = __shfl_up_sync(0xffffffffu, inc, off);
      if((int)threadIdx.x >= off) inc += up;
    }
    if(b < P.n_blocks)
      P.block_counts[b] = running + inc - c;
    running += __shfl_sync(0xffffffffu, inc, 31);
  }
  if(threadIdx.x == 0)
  {
    P.total[0] = running;
    P.total[1] = 0u;   // ticket ready for the next extraction
  }
}

// pass 2: back-projection of the converged pixels (back_project), written at their rank.
__global__ void __launch_bounds__(POINT_CLOUD_BLOCK) point_cloud_write_kernel(const PointCloudParams P)
{
  __shared__ unsigned int warp_off[POINT_CLOUD_BLOCK / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int base = blockIdx.x * POINT_CLOUD_PIXELS + threadIdx.x * 4;
  bool c[4];
  unsigned int n = 0;
#pragma unroll
  for(int k = 0; k < 4; ++k)
  {
    c[k] = is_converged(P, base + k);
    n += c[k] ? 1u : 0u;
  }
  unsigned int inc = n;
#pragma unroll
  for(int off = 1; off < 32; off <<= 1)
  {
    const unsigned int up = __shfl_up_sync(0xffffffffu, inc, off);
    if(lane >= off) inc += up;
  }
  if(lane == 31)
    warp_off[wid] = inc;
  __syncthreads();
  unsigned int rank = P.block_counts[blockIdx.x] + inc - n;
  for(int w = 0; w < wid; ++w) rank += warp_off[w];
#pragma unroll
  for(int k = 0; k < 4; ++k)
  {
    if(!c[k])
      continue;
    const unsigned int slot = rank++;
    if(slot >= P.capacity)
      continue;
    const int i = base + k;
    const int y = i / P.width, x = i - y * P.width;
    const float depth = P.depth[(size_t)y * P.depth_stride + (size_t)x * P.depth_comps];
    const float3 p = back_project(P.cam, P.T_world_ref, x, y, depth);
    float4 o;
    o.x = p.x; o.y = p.y; o.z = p.z;
    // the 8-bit reference image the Depthmap keeps (src/depthmap.cpp:78) is 255 * ref, exactly
    const float r255 = __fmul_rn(P.ref[(size_t)y * P.ref_stride + x], 255.0f);
    o.w = fminf(fmaxf(rintf(r255), 0.0f), 255.0f);
    P.out[slot] = o;
  }
}

} // namespace

cudaError_t launch_point_cloud(const PointCloudParams &P, cudaStream_t stream)
{
  point_cloud_count_kernel<<<P.n_blocks, POINT_CLOUD_BLOCK, 0, stream>>>(P);
  cudaError_t err = cudaGetLastError();
  if(err != cudaSuccess) return err;
  point_cloud_write_kernel<<<P.n_blocks, POINT_CLOUD_BLOCK, 0, stream>>>(P);
  return cudaGetLastError();
}

} // namespace rmdb
