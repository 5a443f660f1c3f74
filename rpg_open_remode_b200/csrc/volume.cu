// volume.cu -- see volume.cuh.  Integration and extraction stream the voxel records once (HBM-bound); the
// raycast reads the few voxels around each ray through the read-only path.
#include "volume.cuh"

#define RMD_MC_STORAGE static __constant__
#include "mc_table.h"

namespace rmdb
{

namespace
{

__device__ __forceinline__ float voxel_coord(float origin, int i, float s)
{
  return __fadd_rn(origin, __fmul_rn((float)i, s));
}

__device__ __forceinline__ bool finite_f(float a)
{
  return (__float_as_uint(a) & 0x7f800000u) != 0x7f800000u;
}

__device__ __forceinline__ float lerp_rn(float a, float b, float f)
{
  return __fadd_rn(a, __fmul_rn(f, __fsub_rn(b, a)));
}

// One thread per voxel, x fastest, so that the float2 records of a warp are contiguous.  The frustum and depth
// tests come before the record is loaded: a voxel outside the image costs no memory traffic.  INTENSITY: then a
// voxel in the band (sdf < tau) also averages the intensity at its pixel into its colour record; the condition
// does not depend on the tsdf record, and a voxel outside the band loads no colour record.
template<bool INTENSITY>
__global__ void __launch_bounds__(256) volume_integrate_kernel(const VolumeIntegrateParams P)
{
  const VolumeGrid &g = P.g;
  const unsigned int plane = (unsigned int)g.nx * (unsigned int)g.ny;
  const unsigned int n = blockIdx.x * blockDim.x + threadIdx.x;   // < 2^31 voxels: fits
  if(n >= plane * (unsigned int)g.nz)
    return;
  const int k = (int)(n / plane);
  const unsigned int rem = n - (unsigned int)k * plane;
  const int j = (int)(rem / (unsigned int)g.nx);
  const int i = (int)(rem - (unsigned int)j * (unsigned int)g.nx);
  const float wx = voxel_coord(g.ox, i, g.voxel), wy = voxel_coord(g.oy, j, g.voxel), wz = voxel_coord(g.oz, k, g.voxel);
  // p = T_curr_world * w: rotation, then translation (as prior_splat_kernel)
  const float *T = P.T_curr_world.m;
  const float px = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], wx), __fmul_rn(T[1], wy)), __fmul_rn(T[2], wz)), T[3]);
  const float py = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], wx), __fmul_rn(T[5], wy)), __fmul_rn(T[6], wz)), T[7]);
  const float pz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], wx), __fmul_rn(T[9], wy)), __fmul_rn(T[10], wz)), T[11]);
  if(!(pz > 0.0f))
    return;
  const float u = __fadd_rn(__fdiv_rn(__fmul_rn(P.cam.fx, px), pz), P.cam.cx);
  const float v = __fadd_rn(__fdiv_rn(__fmul_rn(P.cam.fy, py), pz), P.cam.cy);
  const float tu = floorf(__fadd_rn(u, 0.5f)), tv = floorf(__fadd_rn(v, 0.5f));   // the splat's rounding
  if(!(tu >= 0.0f && tu < (float)P.width && tv >= 0.0f && tv < (float)P.height))
    return;
  const int x = (int)tu, y = (int)tv;
  if(P.conv && P.conv[(size_t)y * P.conv_stride + x] != RMD_CONVERGED)
    return;
  const float d = P.depth[(size_t)y * P.depth_stride + (size_t)x * P.depth_comps];
  if(!(d > 0.0f) || (__float_as_uint(d) & 0x7f800000u) == 0x7f800000u)   // not positive, or inf / NaN
    return;
  // depth is the distance along the ray, so the signed distance is taken along the ray too
  const float r = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
  const float sdf = __fsub_rn(d, r);
  if(!(sdf >= -P.trunc))   // occluded (also drops NaN)
    return;
  const float o = fminf(1.0f, __fdiv_rn(sdf, P.trunc));
  const size_t lin = ((size_t)k * g.ny + j) * g.nx + i;
  const float2 rec = g.vox[lin];
  const float w1 = __fadd_rn(rec.y, 1.0f);
  const float t1 = __fdiv_rn(__fadd_rn(__fmul_rn(rec.x, rec.y), o), w1);
  g.vox[lin] = make_float2(t1, fminf(w1, P.max_weight));
  if(INTENSITY && sdf < P.trunc)
  {
    const float I = P.intensity[(size_t)y * P.intensity_stride + x];
    if(!finite_f(I))
      return;
    const float2 c = P.col[lin];
    const float wc1 = __fadd_rn(c.y, 1.0f);
    const float c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c.x, c.y), I), wc1);
    P.col[lin] = make_float2(c1, fminf(wc1, P.max_weight));
  }
}

// ---------------------------------------------------------------------------------------- surface points
__device__ __forceinline__ bool known_near_surface(float2 r)
{
  return r.y > 0.0f && fabsf(r.x) < 1.0f;
}

__device__ __forceinline__ bool crosses(float2 a, float2 b)
{
  return known_near_surface(b) && ((a.x > 0.0f && b.x <= 0.0f) || (a.x <= 0.0f && b.x > 0.0f));
}

// Voxel n and its +x, +y, +z neighbours: bit a of mask = a point on axis a.
struct SurfaceCell
{
  float2 a, b[3];
  int i, j, k;
  unsigned int mask;
};

__device__ __forceinline__ SurfaceCell surface_cell(const VolumeGrid &g, unsigned int n, unsigned int n_vox)
{
  SurfaceCell c;
  c.mask = 0u;
  if(n >= n_vox)
    return c;
  c.a = __ldg(g.vox + n);
  if(!known_near_surface(c.a))   // free space (tsdf 1) and unknown voxels: no neighbour loads
    return c;
  const unsigned int plane = (unsigned int)g.nx * (unsigned int)g.ny;
  c.k = (int)(n / plane);
  const unsigned int rem = n - (unsigned int)c.k * plane;
  c.j = (int)(rem / (unsigned int)g.nx);
  c.i = (int)(rem - (unsigned int)c.j * (unsigned int)g.nx);
  if(c.i + 1 < g.nx)
  {
    c.b[0] = __ldg(g.vox + (size_t)n + 1);
    c.mask |= crosses(c.a, c.b[0]) ? 1u : 0u;
  }
  if(c.j + 1 < g.ny)
  {
    c.b[1] = __ldg(g.vox + (size_t)n + g.nx);
    c.mask |= crosses(c.a, c.b[1]) ? 2u : 0u;
  }
  if(c.k + 1 < g.nz)
  {
    c.b[2] = __ldg(g.vox + (size_t)n + plane);
    c.mask |= crosses(c.a, c.b[2]) ? 4u : 0u;
  }
  return c;
}

// p_a + (t_a / (t_a - t_b)) * s along `axis`, weight min(w_a, w_b)
__device__ __forceinline__ float4 surface_point(const VolumeGrid &g, const SurfaceCell &c, int axis)
{
  const float2 b = c.b[axis];
  float4 o;
  o.x = voxel_coord(g.ox, c.i, g.voxel);
  o.y = voxel_coord(g.oy, c.j, g.voxel);
  o.z = voxel_coord(g.oz, c.k, g.voxel);
  const float step = __fmul_rn(__fdiv_rn(c.a.x, __fsub_rn(c.a.x, b.x)), g.voxel);
  if(axis == 0) o.x = __fadd_rn(o.x, step);
  else if(axis == 1) o.y = __fadd_rn(o.y, step);
  else o.z = __fadd_rn(o.z, step);
  o.w = fminf(c.a.y, b.y);
  return o;
}

// Intensity of the point of voxel n on `axis`: the colour records of its two voxels, interpolated with the
// position's factor t_a / (t_a - t_b) when both are known.
__device__ __forceinline__ float surface_intensity(const VolumeSurfaceParams &P, const SurfaceCell &c, unsigned int n,
                                                   int axis)
{
  const size_t step = axis == 0 ? (size_t)1 : axis == 1 ? (size_t)P.g.nx : (size_t)P.g.nx * (size_t)P.g.ny;
  const float2 ca = __ldg(P.col + n), cb = __ldg(P.col + (size_t)n + step);
  if(ca.y > 0.0f && cb.y > 0.0f)
    return lerp_rn(ca.x, cb.x, __fdiv_rn(c.a.x, __fsub_rn(c.a.x, c.b[axis].x)));
  return ca.y > 0.0f ? ca.x : cb.y > 0.0f ? cb.x : -1.0f;
}

// ---------------------------------------------------------------------------------------- normals
// One component of the tsdf gradient of a known voxel (record index n, tsdf t0) along an axis of index step `step`:
// the neighbours n - step (when dn) and n + step (when up) lie inside the grid and count when their weight is > 0.
__device__ __forceinline__ float gradient_component(const float2 *vox, size_t n, size_t step, bool dn, bool up,
                                                    float t0)
{
  float2 m = make_float2(0.0f, 0.0f), p = make_float2(0.0f, 0.0f);
  if(dn) m = __ldg(vox + n - step);
  if(up) p = __ldg(vox + n + step);
  const bool um = m.y > 0.0f, up_ok = p.y > 0.0f;
  if(um && up_ok) return __fmul_rn(__fsub_rn(p.x, m.x), 0.5f);
  if(up_ok) return __fsub_rn(p.x, t0);
  if(um) return __fsub_rn(t0, m.x);
  return 0.0f;
}

// The tsdf gradient of known voxel (i, j, k) with tsdf t0 (DESIGN.md 4.8): unitless, per voxel, towards tsdf > 0.
__device__ __forceinline__ float3 voxel_gradient(const VolumeGrid &g, int i, int j, int k, float t0)
{
  const size_t sy = (size_t)g.nx, sz = (size_t)g.nx * (size_t)g.ny;
  const size_t n = (size_t)k * sz + (size_t)j * sy + (size_t)i;
  return make_float3(gradient_component(g.vox, n, 1, i > 0, i + 1 < g.nx, t0),
                     gradient_component(g.vox, n, sy, j > 0, j + 1 < g.ny, t0),
                     gradient_component(g.vox, n, sz, k > 0, k + 1 < g.nz, t0));
}

// g / |g| with |g| = sqrt((gx^2 + gy^2) + gz^2); (0, 0, 0) when |g| is 0 or not finite.  The fourth component is 0.
__device__ __forceinline__ float4 unit_normal(float3 v)
{
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)), __fmul_rn(v.z, v.z)));
  if(!(len > 0.0f) || !finite_f(len))
    return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  return make_float4(__fdiv_rn(v.x, len), __fdiv_rn(v.y, len), __fdiv_rn(v.z, len), 0.0f);
}

__device__ __forceinline__ float3 lerp3_rn(float3 a, float3 b, float f)
{
  return make_float3(lerp_rn(a.x, b.x, f), lerp_rn(a.y, b.y, f), lerp_rn(a.z, b.z, f));
}

// Normal of the point of voxel a = (c.i, c.j, c.k) on `axis`: the gradients of a and of its neighbour b, interpolated
// with the position's factor t_a / (t_a - t_b), then normalised.
__device__ __forceinline__ float4 surface_normal(const VolumeGrid &g, const SurfaceCell &c, int axis)
{
  const float3 ga = voxel_gradient(g, c.i, c.j, c.k, c.a.x);
  const float3 gb = voxel_gradient(g, c.i + (axis == 0), c.j + (axis == 1), c.k + (axis == 2), c.b[axis].x);
  return unit_normal(lerp3_rn(ga, gb, __fdiv_rn(c.a.x, __fsub_rn(c.a.x, c.b[axis].x))));
}

__device__ __forceinline__ unsigned int grid_voxels(const VolumeGrid &g)
{
  return (unsigned int)g.nx * (unsigned int)g.ny * (unsigned int)g.nz;   // <= 2^31
}

// Block b covers voxels [b * VOLUME_SURF_VOXELS, (b + 1) * VOLUME_SURF_VOXELS), in VOLUME_SURF_ROUNDS rounds of
// VOLUME_SURF_BLOCK consecutive voxels (one per thread, so that loads coalesce).  The block's total of count(n), the
// outputs of voxel n, goes to B.block_offsets[b].
template<typename Count>
__device__ __forceinline__ void count_block(const VolumeBlockOffsets &B, Count count)
{
  __shared__ unsigned int warp_sum[VOLUME_SURF_BLOCK / 32];
  const unsigned int base = blockIdx.x * VOLUME_SURF_VOXELS + threadIdx.x;
  unsigned int c = 0;
#pragma unroll
  for(int r = 0; r < VOLUME_SURF_ROUNDS; ++r)
    c += count(base + r * VOLUME_SURF_BLOCK);
  c = __reduce_add_sync(0xffffffffu, c);
  if((threadIdx.x & 31) == 0)
    warp_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  if(threadIdx.x == 0)
  {
    unsigned int tot = 0;
    for(int w = 0; w < VOLUME_SURF_BLOCK / 32; ++w) tot += warp_sum[w];
    B.block_offsets[blockIdx.x] = tot;
  }
}

// The slot of this thread's first output in a round of a write pass: rank (the outputs of the block's earlier
// rounds, from its offset on) + the outputs of the threads before it in the round (a warp shuffle scan, then the
// warps before it); all = the round's outputs.  The caller syncs the block before warp_off is reused.
__device__ __forceinline__ unsigned long long round_slot(unsigned long long rank, unsigned int cnt,
                                                         unsigned int *warp_off, unsigned int &all)
{
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned int inc = cnt;
#pragma unroll
  for(int off = 1; off < 32; off <<= 1)
  {
    const unsigned int up = __shfl_up_sync(0xffffffffu, inc, off);
    if(lane >= off) inc += up;
  }
  if(lane == 31)
    warp_off[wid] = inc;
  __syncthreads();
  unsigned int before = 0;
  all = 0;
#pragma unroll
  for(int w = 0; w < VOLUME_SURF_BLOCK / 32; ++w)
  {
    const unsigned int x = warp_off[w];
    before += (w < wid) ? x : 0u;
    all += x;
  }
  return rank + before + inc - cnt;
}

__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_surface_count_kernel(const VolumeSurfaceParams P)
{
  const unsigned int n_vox = grid_voxels(P.g);
  count_block(P.b, [&](unsigned int n) { return (unsigned int)__popc(surface_cell(P.g, n, n_vox).mask); });
}

// Second level: ONE block turns the block totals (up to 2^31 / VOLUME_SURF_VOXELS = 2^20 of them) into exclusive
// offsets, VOLUME_SCAN_BLOCK * 8 totals per pass (8 consecutive per thread, then a block-wide scan of the sums).
// It serves the surface points and the mesh's triangles.
__global__ void __launch_bounds__(VOLUME_SCAN_BLOCK) volume_surface_scan_kernel(const VolumeBlockOffsets P)
{
  constexpr int PER = 8;
  __shared__ unsigned long long warp_tot[VOLUME_SCAN_BLOCK / 32];
  __shared__ unsigned long long carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if(threadIdx.x == 0)
    carry = 0ull;
  __syncthreads();
  for(unsigned int b0 = 0; b0 < P.n_blocks; b0 += VOLUME_SCAN_BLOCK * PER)
  {
    const unsigned int first = b0 + threadIdx.x * PER;
    unsigned long long v[PER], sum = 0ull;
#pragma unroll
    for(int q = 0; q < PER; ++q)
    {
      v[q] = (first + q < P.n_blocks) ? P.block_offsets[first + q] : 0ull;
      sum += v[q];
    }
    unsigned long long inc = sum;
#pragma unroll
    for(int off = 1; off < 32; off <<= 1)
    {
      const unsigned long long up = __shfl_up_sync(0xffffffffu, inc, off);
      if(lane >= off) inc += up;
    }
    if(lane == 31)
      warp_tot[wid] = inc;
    __syncthreads();
    if(wid == 0)
    {
      unsigned long long w = warp_tot[lane];
#pragma unroll
      for(int off = 1; off < 32; off <<= 1)
      {
        const unsigned long long up = __shfl_up_sync(0xffffffffu, w, off);
        if(lane >= off) w += up;
      }
      warp_tot[lane] = w;
    }
    __syncthreads();
    unsigned long long run = carry + (wid ? warp_tot[wid - 1] : 0ull) + inc - sum;
#pragma unroll
    for(int q = 0; q < PER; ++q)
    {
      if(first + q < P.n_blocks)
        P.block_offsets[first + q] = run;
      run += v[q];
    }
    __syncthreads();   // every thread has read carry and warp_tot
    if(threadIdx.x == VOLUME_SCAN_BLOCK - 1)
      carry = run;     // the last thread's running sum ends at the pass total
    __syncthreads();
  }
  if(threadIdx.x == 0)
    P.total[0] = carry;
}

// The points of cell c that spill from the kept box K: bit a stays set unless both voxel a and its neighbour on axis a
// lie inside K (b differs from a only on that axis, and b >= a >= lo there).
__device__ __forceinline__ unsigned int spill_mask(const VolumeSpillBox &K, const SurfaceCell &c)
{
  if(!c.mask)
    return 0u;
  const int p[3] = {c.i, c.j, c.k};
  bool a_in = true;
#pragma unroll
  for(int a = 0; a < 3; ++a)
    a_in = a_in && p[a] >= K.lo[a] && p[a] < K.hi[a];
  unsigned int kept = 0u;
#pragma unroll
  for(int a = 0; a < 3; ++a)
    kept |= (a_in && p[a] + 1 < K.hi[a]) ? (1u << a) : 0u;
  return c.mask & ~kept;
}

__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_spill_count_kernel(const VolumeSurfaceParams P,
                                                                               const VolumeSpillBox K)
{
  const unsigned int n_vox = grid_voxels(P.g);
  count_block(P.b, [&](unsigned int n) { return (unsigned int)__popc(spill_mask(K, surface_cell(P.g, n, n_vox))); });
}

// KEYS (the mesh path): also write every point's key 3 * voxel + axis, for all *total points whatever the capacity.
// INTENSITY: write every point's intensity to P.intensity instead of its position to P.out.  NORMALS: write every
// point's normal to P.normals instead.
template<bool KEYS, bool INTENSITY, bool NORMALS>
__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_surface_write_kernel(const VolumeSurfaceParams P)
{
  __shared__ unsigned int warp_off[VOLUME_SURF_BLOCK / 32];
  const unsigned int n_vox = grid_voxels(P.g);
  const unsigned int base = blockIdx.x * VOLUME_SURF_VOXELS + threadIdx.x;
  unsigned long long rank = P.b.block_offsets[blockIdx.x];
  for(int r = 0; r < VOLUME_SURF_ROUNDS; ++r)
  {
    const SurfaceCell c = surface_cell(P.g, base + r * VOLUME_SURF_BLOCK, n_vox);
    unsigned int all;
    unsigned long long slot = round_slot(rank, __popc(c.mask), warp_off, all);
#pragma unroll
    for(int axis = 0; axis < 3; ++axis)
    {
      if(!(c.mask & (1u << axis)))
        continue;
      if(slot < P.capacity)
      {
        if(INTENSITY)
          P.intensity[slot] = surface_intensity(P, c, base + r * VOLUME_SURF_BLOCK, axis);
        else if(NORMALS)
          P.normals[slot] = surface_normal(P.g, c, axis);
        else
          P.out[slot] = surface_point(P.g, c, axis);
      }
      if(KEYS)
        P.keys[slot] = 3ull * (base + r * VOLUME_SURF_BLOCK) + axis;
      ++slot;
    }
    rank += all;
    __syncthreads();   // warp_off is reused by the next round
  }
}

// volume_surface_write_kernel without keys, on the points that spill from K: the same blocks, rounds and ranks over
// the spill counts, so that the spill comes out in the surface points' order.  (The surface kernel's body is kept as
// it is rather than shared: inlining it into a common function reorders operands in its SASS.)
template<bool INTENSITY, bool NORMALS>
__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_spill_write_kernel(const VolumeSurfaceParams P,
                                                                               const VolumeSpillBox K)
{
  __shared__ unsigned int warp_off[VOLUME_SURF_BLOCK / 32];
  const unsigned int n_vox = grid_voxels(P.g);
  const unsigned int base = blockIdx.x * VOLUME_SURF_VOXELS + threadIdx.x;
  unsigned long long rank = P.b.block_offsets[blockIdx.x];
  for(int r = 0; r < VOLUME_SURF_ROUNDS; ++r)
  {
    SurfaceCell c = surface_cell(P.g, base + r * VOLUME_SURF_BLOCK, n_vox);
    c.mask = spill_mask(K, c);
    unsigned int all;
    unsigned long long slot = round_slot(rank, __popc(c.mask), warp_off, all);
#pragma unroll
    for(int axis = 0; axis < 3; ++axis)
    {
      if(!(c.mask & (1u << axis)) || slot >= P.capacity)
        continue;
      if(INTENSITY)
        P.intensity[slot] = surface_intensity(P, c, base + r * VOLUME_SURF_BLOCK, axis);
      else if(NORMALS)
        P.normals[slot] = surface_normal(P.g, c, axis);
      else
        P.out[slot] = surface_point(P.g, c, axis);
      ++slot;
    }
    rank += all;
    __syncthreads();   // warp_off is reused by the next round
  }
}

// ------------------------------------------------------------------------------------------------- shift
// One thread per destination voxel, x fastest: a gather, so that both the loads of a warp (one source row) and its
// stores are contiguous.
template<bool INTENSITY>
__global__ void __launch_bounds__(256) volume_shift_kernel(const VolumeShiftParams P)
{
  const VolumeGrid &g = P.g;
  const unsigned int plane = (unsigned int)g.nx * (unsigned int)g.ny;
  const unsigned int n = blockIdx.x * blockDim.x + threadIdx.x;   // < 2^31 voxels: fits
  if(n >= plane * (unsigned int)g.nz)
    return;
  const int k = (int)(n / plane);
  const unsigned int rem = n - (unsigned int)k * plane;
  const int j = (int)(rem / (unsigned int)g.nx);
  const int i = (int)(rem - (unsigned int)j * (unsigned int)g.nx);
  const int si = i + P.dx, sj = j + P.dy, sk = k + P.dz;   // |d| < n: no overflow
  float2 r = make_float2(0.0f, 0.0f), c = make_float2(0.0f, 0.0f);
  if((unsigned int)si < (unsigned int)g.nx && (unsigned int)sj < (unsigned int)g.ny &&
     (unsigned int)sk < (unsigned int)g.nz)
  {
    const size_t src = ((size_t)sk * g.ny + sj) * g.nx + si;
    r = __ldg(g.vox + src);
    if(INTENSITY)
      c = __ldg(P.col + src);
  }
  const size_t lin = ((size_t)k * g.ny + j) * g.nx + i;
  P.out[lin] = r;
  if(INTENSITY)
    P.col_out[lin] = c;
}

// --------------------------------------------------------------------------------------------------- mesh
// Case of cube n (corner c = dx + 2 dy + 4 dz at voxel n + dx + dy nx + dz nx ny; bit c = inside, tsdf <= 0), or 0
// when the cube is not meshed.  An unknown lower corner costs one load; the other seven corners come from the same
// row (L1) and the +y / +z rows and planes, which the neighbouring blocks stream through L2.
__device__ __forceinline__ unsigned int mesh_cube(const VolumeGrid &g, unsigned int n, unsigned int n_vox)
{
  if(n >= n_vox)
    return 0u;
  const float2 a = __ldg(g.vox + n);
  if(!(a.y > 0.0f))
    return 0u;
  const unsigned int plane = (unsigned int)g.nx * (unsigned int)g.ny;
  const unsigned int k = n / plane;
  const unsigned int rem = n - k * plane;
  const unsigned int j = rem / (unsigned int)g.nx;
  const unsigned int i = rem - j * (unsigned int)g.nx;
  if(i + 1u >= (unsigned int)g.nx || j + 1u >= (unsigned int)g.ny || k + 1u >= (unsigned int)g.nz)
    return 0u;
  const float2 *p = g.vox + n;
  const size_t sy = (size_t)g.nx, sz = (size_t)plane;
  const float2 r[8] = {a, __ldg(p + 1), __ldg(p + sy), __ldg(p + sy + 1), __ldg(p + sz), __ldg(p + sz + 1),
                       __ldg(p + sz + sy), __ldg(p + sz + sy + 1)};
  unsigned int cube = 0u, near = 0u;
  bool known = true;
#pragma unroll
  for(int c = 0; c < 8; ++c)
  {
    known = known && r[c].y > 0.0f;
    cube |= (r[c].x <= 0.0f ? 1u : 0u) << c;
    near |= (fabsf(r[c].x) < 1.0f ? 1u : 0u) << c;
  }
  if(!known || cube == 0u || cube == 255u)
    return 0u;
  // a crossing edge (ends differ in sign) with a truncated end: x edges pair corners c, c + 1 (mask 0x55), y edges
  // c, c + 2 (0x33), z edges c, c + 4 (0x0f)
  const unsigned int bad = (((cube ^ (cube >> 1)) & ~(near & (near >> 1))) & 0x55u) |
                           (((cube ^ (cube >> 2)) & ~(near & (near >> 2))) & 0x33u) |
                           (((cube ^ (cube >> 4)) & ~(near & (near >> 4))) & 0x0fu);
  return bad ? 0u : cube;
}

__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_mesh_count_kernel(const VolumeMeshParams P)
{
  const unsigned int n_vox = grid_voxels(P.g);
  count_block(P.b, [&](unsigned int n) { return (unsigned int)RMD_MC_NTRI[mesh_cube(P.g, n, n_vox)]; });
}

// Index of the surface point on edge e of cube n: binary search for its key among the points of the edge's voxel's
// block, [offset[b], offset[b + 1]) -- at most 3 * VOLUME_SURF_VOXELS = 6144 keys, 13 steps.  The point exists: the
// cube test is the surface-point rule on every crossing edge.
__device__ __forceinline__ int mesh_vertex(const VolumeMeshParams &P, unsigned int n, int e)
{
  const unsigned int c0 = RMD_MC_EDGE[e][0], axis = RMD_MC_EDGE[e][1];
  const unsigned int v = n + (c0 & 1u) + ((c0 >> 1) & 1u) * (unsigned int)P.g.nx +
                         ((c0 >> 2) & 1u) * (unsigned int)P.g.nx * (unsigned int)P.g.ny;   // a voxel: < 2^31
  const unsigned long long key = 3ull * v + axis;
  const unsigned int b = v / VOLUME_SURF_VOXELS;
  unsigned long long lo = P.point_offsets[b];
  unsigned long long hi = b + 1 < P.b.n_blocks ? P.point_offsets[b + 1] : P.point_total[0];
  while(lo < hi)
  {
    const unsigned long long mid = (lo + hi) >> 1;
    if(P.keys[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return (int)lo;   // < 2^31 points (the host refuses more)
}

__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_mesh_write_kernel(const VolumeMeshParams P)
{
  __shared__ unsigned int warp_off[VOLUME_SURF_BLOCK / 32];
  const unsigned int n_vox = grid_voxels(P.g);
  const unsigned int base = blockIdx.x * VOLUME_SURF_VOXELS + threadIdx.x;
  unsigned long long rank = P.b.block_offsets[blockIdx.x];
  for(int r = 0; r < VOLUME_SURF_ROUNDS; ++r)
  {
    const unsigned int n = base + r * VOLUME_SURF_BLOCK;
    const unsigned int cube = mesh_cube(P.g, n, n_vox);
    const unsigned int cnt = RMD_MC_NTRI[cube];
    unsigned int all;
    unsigned long long slot = round_slot(rank, cnt, warp_off, all);
    for(unsigned int q = 0; q < cnt && slot < P.capacity; ++q, ++slot)
    {
      int *t = P.tri + 3 * slot;
      t[0] = mesh_vertex(P, n, RMD_MC_TRIS[cube][3 * q + 0]);
      t[1] = mesh_vertex(P, n, RMD_MC_TRIS[cube][3 * q + 1]);
      t[2] = mesh_vertex(P, n, RMD_MC_TRIS[cube][3 * q + 2]);
    }
    rank += all;
    __syncthreads();   // warp_off is reused by the next round
  }
}

// ---------------------------------------------------------------------------------------------- spill mesh
// Case of cube n when it is meshed and spills from K -- one of its corners, lower corner + {0, 1} per axis, lies
// outside K -- else 0.
__device__ __forceinline__ unsigned int spill_cube(const VolumeGrid &g, const VolumeSpillBox &K, unsigned int n,
                                                   unsigned int n_vox)
{
  const unsigned int cube = mesh_cube(g, n, n_vox);
  if(!cube)
    return 0u;
  const unsigned int plane = (unsigned int)g.nx * (unsigned int)g.ny;
  const int k = (int)(n / plane);
  const unsigned int rem = n - (unsigned int)k * plane;
  const int j = (int)(rem / (unsigned int)g.nx);
  const int i = (int)(rem - (unsigned int)j * (unsigned int)g.nx);
  const bool leaves = i < K.lo[0] || i + 1 >= K.hi[0] || j < K.lo[1] || j + 1 >= K.hi[1] || k < K.lo[2] ||
                      k + 1 >= K.hi[2];
  return leaves ? cube : 0u;
}

// The spill mesh's vertices of cell c (voxel n): the points that spill from K (spill_mask), and the points that stay
// whose edge belongs to a spilling cube.  The cubes of edge (a, axis) have lower corners a - du e_u - dw e_w (du, dw
// in {0, 1}; u, w the other two axes).  Their corners on `axis` are a and a + e_axis, inside K for a staying point, so
// one of them leaves K only across u or w: that needs a within one voxel of a face of K, and only then are the <= 4
// cubes tested with mesh_cube.
__device__ __forceinline__ unsigned int spill_mesh_mask(const VolumeGrid &g, const VolumeSpillBox &K,
                                                        const SurfaceCell &c, unsigned int n, unsigned int n_vox)
{
  const unsigned int spill = spill_mask(K, c);
  const unsigned int stay = c.mask & ~spill;
  if(!stay)
    return spill;
  const unsigned int plane = (unsigned int)g.nx * (unsigned int)g.ny;
  unsigned int seam = 0u;
#pragma unroll
  for(int axis = 0; axis < 3; ++axis)
  {
    if(!(stay & (1u << axis)))
      continue;
    const int pu = axis == 0 ? c.j : c.i, pw = axis == 2 ? c.j : c.k;
    const int lu = axis == 0 ? K.lo[1] : K.lo[0], hu = axis == 0 ? K.hi[1] : K.hi[0];
    const int lw = axis == 2 ? K.lo[1] : K.lo[2], hw = axis == 2 ? K.hi[1] : K.hi[2];
    const unsigned int su = axis == 0 ? (unsigned int)g.nx : 1u, sw = axis == 2 ? (unsigned int)g.nx : plane;
    if(pu > lu && pu + 1 < hu && pw > lw && pw + 1 < hw)   // every cube of the edge lies inside K
      continue;
    bool hit = false;
#pragma unroll 1
    for(int q = 0; q < 4 && !hit; ++q)
    {
      const int du = q & 1, dw = q >> 1;
      const int cu = pu - du, cw = pw - dw;
      if(cu < 0 || cw < 0 || !(cu < lu || cu + 1 >= hu || cw < lw || cw + 1 >= hw))
        continue;
      hit = mesh_cube(g, n - (unsigned int)du * su - (unsigned int)dw * sw, n_vox) != 0u;
    }
    seam |= hit ? (1u << axis) : 0u;
  }
  return spill | seam;
}

__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_spill_mesh_count_kernel(const VolumeSurfaceParams P,
                                                                                    const VolumeSpillBox K)
{
  const unsigned int n_vox = grid_voxels(P.g);
  count_block(P.b, [&](unsigned int n) {
    return (unsigned int)__popc(spill_mesh_mask(P.g, K, surface_cell(P.g, n, n_vox), n, n_vox));
  });
}

// volume_spill_write_kernel on the spill mesh's vertices.  With P.keys, also every vertex's key 3 * voxel + axis, for
// all *total vertices whatever the capacity (as the surface kernel's KEYS instance), for mesh_vertex.
template<bool INTENSITY, bool NORMALS>
__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_spill_mesh_write_kernel(const VolumeSurfaceParams P,
                                                                                    const VolumeSpillBox K)
{
  __shared__ unsigned int warp_off[VOLUME_SURF_BLOCK / 32];
  const unsigned int n_vox = grid_voxels(P.g);
  const unsigned int base = blockIdx.x * VOLUME_SURF_VOXELS + threadIdx.x;
  unsigned long long rank = P.b.block_offsets[blockIdx.x];
  for(int r = 0; r < VOLUME_SURF_ROUNDS; ++r)
  {
    const unsigned int n = base + r * VOLUME_SURF_BLOCK;
    SurfaceCell c = surface_cell(P.g, n, n_vox);
    c.mask = spill_mesh_mask(P.g, K, c, n, n_vox);
    unsigned int all;
    unsigned long long slot = round_slot(rank, __popc(c.mask), warp_off, all);
#pragma unroll
    for(int axis = 0; axis < 3; ++axis)
    {
      if(!(c.mask & (1u << axis)))
        continue;
      if(slot < P.capacity)
      {
        if(INTENSITY)
          P.intensity[slot] = surface_intensity(P, c, n, axis);
        else if(NORMALS)
          P.normals[slot] = surface_normal(P.g, c, axis);
        else
          P.out[slot] = surface_point(P.g, c, axis);
      }
      if(P.keys)
        P.keys[slot] = 3ull * n + axis;
      ++slot;
    }
    rank += all;
    __syncthreads();   // warp_off is reused by the next round
  }
}

__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_spill_tri_count_kernel(const VolumeMeshParams P,
                                                                                   const VolumeSpillBox K)
{
  const unsigned int n_vox = grid_voxels(P.g);
  count_block(P.b, [&](unsigned int n) { return (unsigned int)RMD_MC_NTRI[spill_cube(P.g, K, n, n_vox)]; });
}

// volume_mesh_write_kernel on the cubes that spill from K; P's point offsets, total and keys are the spill mesh's
// vertices', so that mesh_vertex finds an index into them.
__global__ void __launch_bounds__(VOLUME_SURF_BLOCK) volume_spill_tri_write_kernel(const VolumeMeshParams P,
                                                                                   const VolumeSpillBox K)
{
  __shared__ unsigned int warp_off[VOLUME_SURF_BLOCK / 32];
  const unsigned int n_vox = grid_voxels(P.g);
  const unsigned int base = blockIdx.x * VOLUME_SURF_VOXELS + threadIdx.x;
  unsigned long long rank = P.b.block_offsets[blockIdx.x];
  for(int r = 0; r < VOLUME_SURF_ROUNDS; ++r)
  {
    const unsigned int n = base + r * VOLUME_SURF_BLOCK;
    const unsigned int cube = spill_cube(P.g, K, n, n_vox);
    const unsigned int cnt = RMD_MC_NTRI[cube];
    unsigned int all;
    unsigned long long slot = round_slot(rank, cnt, warp_off, all);
    for(unsigned int q = 0; q < cnt && slot < P.capacity; ++q, ++slot)
    {
      int *t = P.tri + 3 * slot;
      t[0] = mesh_vertex(P, n, RMD_MC_TRIS[cube][3 * q + 0]);
      t[1] = mesh_vertex(P, n, RMD_MC_TRIS[cube][3 * q + 1]);
      t[2] = mesh_vertex(P, n, RMD_MC_TRIS[cube][3 * q + 2]);
    }
    rank += all;
    __syncthreads();   // warp_off is reused by the next round
  }
}

// --------------------------------------------------------------------------------------------- raycast
// Trilinear interpolation of the records rec (g.vox or the intensity records, indexed alike) at grid coordinates
// (gx, gy, gz), in x, then y, then z; false if a corner lies outside the grid or has weight 0.
__device__ __forceinline__ bool sample_records(const VolumeGrid &g, const float2 *rec, float gx, float gy, float gz,
                                               float &out)
{
  const float x0 = floorf(gx), y0 = floorf(gy), z0 = floorf(gz);
  const int i0 = (x0 >= 0.0f && x0 < 2.0e9f) ? (int)x0 : -1;
  const int j0 = (y0 >= 0.0f && y0 < 2.0e9f) ? (int)y0 : -1;
  const int k0 = (z0 >= 0.0f && z0 < 2.0e9f) ? (int)z0 : -1;
  if(i0 < 0 || j0 < 0 || k0 < 0 || i0 + 1 >= g.nx || j0 + 1 >= g.ny || k0 + 1 >= g.nz)
    return false;
  const size_t plane = (size_t)g.nx * g.ny;
  const float2 *b = rec + ((size_t)k0 * g.ny + j0) * g.nx + i0;
  const float2 c000 = __ldg(b), c100 = __ldg(b + 1), c010 = __ldg(b + g.nx), c110 = __ldg(b + g.nx + 1);
  const float2 c001 = __ldg(b + plane), c101 = __ldg(b + plane + 1), c011 = __ldg(b + plane + g.nx),
               c111 = __ldg(b + plane + g.nx + 1);
  if(c000.y == 0.0f || c100.y == 0.0f || c010.y == 0.0f || c110.y == 0.0f || c001.y == 0.0f || c101.y == 0.0f ||
     c011.y == 0.0f || c111.y == 0.0f)
    return false;
  const float fx = __fsub_rn(gx, x0), fy = __fsub_rn(gy, y0), fz = __fsub_rn(gz, z0);
  const float c00 = lerp_rn(c000.x, c100.x, fx), c10 = lerp_rn(c010.x, c110.x, fx);
  const float c01 = lerp_rn(c001.x, c101.x, fx), c11 = lerp_rn(c011.x, c111.x, fx);
  out = lerp_rn(lerp_rn(c00, c10, fy), lerp_rn(c01, c11, fy), fz);
  return true;
}

// The normal at grid coordinates (gx, gy, gz): the gradients of the 8 corners of the cell (which read the cell's
// records and those of its face neighbours), interpolated trilinearly in x, then y, then z per component, then
// normalised; (0, 0, 0, 0) if a corner lies outside the grid or has weight 0.
__device__ __forceinline__ float4 sample_normal(const VolumeGrid &g, float gx, float gy, float gz)
{
  const float4 none = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  const float x0 = floorf(gx), y0 = floorf(gy), z0 = floorf(gz);
  const int i0 = (x0 >= 0.0f && x0 < 2.0e9f) ? (int)x0 : -1;
  const int j0 = (y0 >= 0.0f && y0 < 2.0e9f) ? (int)y0 : -1;
  const int k0 = (z0 >= 0.0f && z0 < 2.0e9f) ? (int)z0 : -1;
  if(i0 < 0 || j0 < 0 || k0 < 0 || i0 + 1 >= g.nx || j0 + 1 >= g.ny || k0 + 1 >= g.nz)
    return none;
  const size_t plane = (size_t)g.nx * g.ny;
  const float2 *b = g.vox + ((size_t)k0 * g.ny + j0) * g.nx + i0;
  const float2 c000 = __ldg(b), c100 = __ldg(b + 1), c010 = __ldg(b + g.nx), c110 = __ldg(b + g.nx + 1);
  const float2 c001 = __ldg(b + plane), c101 = __ldg(b + plane + 1), c011 = __ldg(b + plane + g.nx),
               c111 = __ldg(b + plane + g.nx + 1);
  if(c000.y == 0.0f || c100.y == 0.0f || c010.y == 0.0f || c110.y == 0.0f || c001.y == 0.0f || c101.y == 0.0f ||
     c011.y == 0.0f || c111.y == 0.0f)
    return none;
  const float fx = __fsub_rn(gx, x0), fy = __fsub_rn(gy, y0), fz = __fsub_rn(gz, z0);
  const float3 c00 = lerp3_rn(voxel_gradient(g, i0, j0, k0, c000.x), voxel_gradient(g, i0 + 1, j0, k0, c100.x), fx);
  const float3 c10 = lerp3_rn(voxel_gradient(g, i0, j0 + 1, k0, c010.x),
                              voxel_gradient(g, i0 + 1, j0 + 1, k0, c110.x), fx);
  const float3 c01 = lerp3_rn(voxel_gradient(g, i0, j0, k0 + 1, c001.x),
                              voxel_gradient(g, i0 + 1, j0, k0 + 1, c101.x), fx);
  const float3 c11 = lerp3_rn(voxel_gradient(g, i0, j0 + 1, k0 + 1, c011.x),
                              voxel_gradient(g, i0 + 1, j0 + 1, k0 + 1, c111.x), fx);
  return unit_normal(lerp3_rn(lerp3_rn(c00, c10, fy), lerp3_rn(c01, c11, fy), fz));
}

// The march of the ray of pixel (x, y): the distance to the first zero crossing, 0 where there is none.  INTENSITY:
// also the intensity at the hit into inten (-1 = none), from the grid coordinates of org + t dir in the march's form
// (the plain instance ignores C and inten).  NORMALS: also the normal at the hit, from the same grid coordinates, into
// normal (left as it is where there is no hit).  The raycasts and the volume prior share it, so that their depths are
// the plain raycast's, bit for bit.
template<bool INTENSITY, bool NORMALS>
__device__ __forceinline__ float raycast_hit(const VolumeRaycastParams &P, const VolumeRaycastColour &C, int x, int y,
                                             float &inten, float4 &normal)
{
  const VolumeGrid &g = P.g;
  // the ray of back_project (point_cloud.cuh), rotated into the world; it starts at the camera centre
  const float vx = __fdiv_rn(__fsub_rn((float)x, P.cam.cx), P.cam.fx);
  const float vy = __fdiv_rn(__fsub_rn((float)y, P.cam.cy), P.cam.fy);
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), 1.0f);
  const float inv_len = __fdiv_rn(1.0f, __fsqrt_rn(dot));
  const float qx = __fmul_rn(vx, inv_len), qy = __fmul_rn(vy, inv_len), qz = __fmul_rn(1.0f, inv_len);
  const float *T = P.T_world_curr.m;
  const float dir[3] = {__fadd_rn(__fadd_rn(__fmul_rn(T[0], qx), __fmul_rn(T[1], qy)), __fmul_rn(T[2], qz)),
                        __fadd_rn(__fadd_rn(__fmul_rn(T[4], qx), __fmul_rn(T[5], qy)), __fmul_rn(T[6], qz)),
                        __fadd_rn(__fadd_rn(__fmul_rn(T[8], qx), __fmul_rn(T[9], qy)), __fmul_rn(T[10], qz))};
  const float org[3] = {T[3], T[7], T[11]};
  const float lo[3] = {g.ox, g.oy, g.oz};
  const int n[3] = {g.nx, g.ny, g.nz};
  // slab test against the box of the voxel centres
  float t0 = 0.0f, t1 = __int_as_float(0x7f800000);
  bool inside = true;
#pragma unroll
  for(int a = 0; a < 3; ++a)
  {
    const float hi = voxel_coord(lo[a], n[a] - 1, g.voxel);
    if(dir[a] == 0.0f)
    {
      inside = inside && org[a] >= lo[a] && org[a] <= hi;
      continue;
    }
    const float ta = __fdiv_rn(__fsub_rn(lo[a], org[a]), dir[a]);
    const float tb = __fdiv_rn(__fsub_rn(hi, org[a]), dir[a]);
    t0 = fmaxf(t0, fminf(ta, tb));
    t1 = fminf(t1, fmaxf(ta, tb));
  }
  float out = 0.0f;
  if(inside && t0 <= t1)
  {
    // a segment inside the box is at most nx + ny + nz voxels long: the bound only stops a ray whose steps
    // vanish against t0 (a camera very far away)
    const int k_max = g.nx + g.ny + g.nz;
    const float s = g.voxel;
    bool prev_known = false;
    float t_prev = 0.0f, f_prev = 0.0f;
    for(int k = 0; k <= k_max; ++k)
    {
      const float t = __fadd_rn(t0, __fmul_rn((float)k, s));   // never accumulated
      if(!(t <= t1))
        break;
      const float gx = __fdiv_rn(__fsub_rn(__fadd_rn(org[0], __fmul_rn(t, dir[0])), g.ox), s);
      const float gy = __fdiv_rn(__fsub_rn(__fadd_rn(org[1], __fmul_rn(t, dir[1])), g.oy), s);
      const float gz = __fdiv_rn(__fsub_rn(__fadd_rn(org[2], __fmul_rn(t, dir[2])), g.oz), s);
      float f = 0.0f;
      const bool known = sample_records(g, g.vox, gx, gy, gz, f);
      if(known && prev_known && f_prev > 0.0f && f <= 0.0f)
      {
        out = __fadd_rn(t_prev, __fdiv_rn(__fmul_rn(s, f_prev), __fsub_rn(f_prev, f)));
        if(INTENSITY || NORMALS)
        {
          const float hx = __fdiv_rn(__fsub_rn(__fadd_rn(org[0], __fmul_rn(out, dir[0])), g.ox), s);
          const float hy = __fdiv_rn(__fsub_rn(__fadd_rn(org[1], __fmul_rn(out, dir[1])), g.oy), s);
          const float hz = __fdiv_rn(__fsub_rn(__fadd_rn(org[2], __fmul_rn(out, dir[2])), g.oz), s);
          if(INTENSITY && !sample_records(g, C.col, hx, hy, hz, inten))
            inten = -1.0f;
          if(NORMALS)
            normal = sample_normal(g, hx, hy, hz);
        }
        break;
      }
      prev_known = known;
      t_prev = t;
      f_prev = f;
    }
  }
  return out;
}

// The colour fields are a parameter of their own: past 128 B a parameter is read through a pointer, which slows the
// plain rays by about 5 %.
template<bool INTENSITY>
__global__ void __launch_bounds__(256) volume_raycast_kernel(const VolumeRaycastParams P, const VolumeRaycastColour C)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if(x >= P.width || y >= P.height)
    return;
  float inten = -1.0f;
  float4 unused;
  P.depth[(size_t)y * P.depth_stride + x] = raycast_hit<INTENSITY, false>(P, C, x, y, inten, unused);
  if(INTENSITY)
    C.intensity[(size_t)y * C.intensity_stride + x] = inten;
}

// The plain rays plus the normal at each hit, one 16-byte store per pixel; the normal outputs are a parameter of
// their own, like the colour fields.
__global__ void __launch_bounds__(256) volume_raycast_normals_kernel(const VolumeRaycastParams P,
                                                                     const VolumeRaycastNormals N)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if(x >= P.width || y >= P.height)
    return;
  const VolumeRaycastColour none = {};
  float unused;
  float4 normal = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  P.depth[(size_t)y * P.depth_stride + x] = raycast_hit<false, true>(P, none, x, y, unused, normal);
  N.normals[(size_t)y * N.normals_stride + x] = normal;
}

// One ray per pixel of the seeds' image; a BORDER pixel is not marched.  A hit within [min_depth, max_depth] becomes
// the seed (d, sigma_sq, 10, 10) in one 16-byte store; every other seed is left as it is.
__global__ void __launch_bounds__(256) volume_prior_kernel(const VolumeRaycastParams P, const VolumePriorSeeds S)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if(x >= P.width || y >= P.height)
    return;
  if(S.conv[(size_t)y * S.conv_stride + x] == RMD_BORDER)
    return;
  const VolumeRaycastColour none = {};
  float unused;
  float4 unused_normal;
  const float d = raycast_hit<false, false>(P, none, x, y, unused, unused_normal);
  if(!(d > 0.0f && d >= S.min_depth && d <= S.max_depth))
    return;
  // a = b = 10: inlier ratio 0.5, so the seed cannot be CONVERGED before new frames confirm it (as prior_apply_kernel)
  S.seed[(size_t)y * S.seed_stride + x] = make_float4(d, S.sigma_sq, 10.0f, 10.0f);
}

// ------------------------------------------------------------------------------------------------- brick store
// One CTA per brick, one thread per brick voxel (x fastest): the window index of voxel l of brick q, or -1 when the
// voxel does not move (DESIGN.md 4.8).  A candidate brick lies within 8 voxels of the window, so that 8 b - W fits.
__device__ __forceinline__ long long store_moving_voxel(const VolumeStoreParams &P, const VolumeStoreBrick &B, int l)
{
  const int n[3] = {P.g.nx, P.g.ny, P.g.nz};
  const int loc[3] = {l & 7, (l >> 3) & 7, l >> 6};
  int w[3];
  bool inside = true;
  for(int a = 0; a < 3; ++a)
  {
    w[a] = (int)(B.b[a] * 8 - P.W[a]) + loc[a];
    if(w[a] < 0 || w[a] >= n[a])
      return -1;
    inside = inside && w[a] >= P.lo[a] && w[a] < P.hi[a];
  }
  if(inside)
    return -1;
  return ((long long)w[2] * P.g.ny + w[1]) * P.g.nx + w[0];
}

__global__ void __launch_bounds__(512) volume_store_flag_kernel(const VolumeStoreParams P)
{
  const VolumeStoreBrick B = P.bricks[blockIdx.x];
  const long long w = store_moving_voxel(P, B, threadIdx.x);
  const int seen = w >= 0 && P.g.vox[w].y > 0.0f;
  const int any = __syncthreads_or(seen);
  if(threadIdx.x == 0)
    P.flags[blockIdx.x] = any;
}

template<bool INTENSITY>
__global__ void __launch_bounds__(512) volume_store_evict_kernel(const VolumeStoreParams P)
{
  const VolumeStoreBrick B = P.bricks[blockIdx.x];
  const long long w = store_moving_voxel(P, B, threadIdx.x);
  const size_t dst = (size_t)B.slot * VOLUME_STORE_VOXELS + threadIdx.x;
  if(w >= 0)
  {
    P.pool[dst] = P.g.vox[w];
    if(INTENSITY)
      P.pool_col[dst] = P.col[w];
  }
  else if(B.fresh)
  {
    P.pool[dst] = make_float2(0.0f, 0.0f);
    if(INTENSITY)
      P.pool_col[dst] = make_float2(0.0f, 0.0f);
  }
}

template<bool INTENSITY>
__global__ void __launch_bounds__(512) volume_store_restore_kernel(const VolumeStoreParams P)
{
  const VolumeStoreBrick B = P.bricks[blockIdx.x];
  const long long w = store_moving_voxel(P, B, threadIdx.x);
  if(w < 0)
    return;
  const size_t src = (size_t)B.slot * VOLUME_STORE_VOXELS + threadIdx.x;
  P.g.vox[w] = P.pool[src];
  if(INTENSITY)
    P.col[w] = P.pool_col[src];
}

} // namespace

cudaError_t launch_volume_integrate(const VolumeIntegrateParams &P, cudaStream_t stream)
{
  const unsigned int n = (unsigned int)P.g.nx * (unsigned int)P.g.ny * (unsigned int)P.g.nz;
  if(P.col)
    volume_integrate_kernel<true><<<(n + 255u) / 256u, 256, 0, stream>>>(P);
  else
    volume_integrate_kernel<false><<<(n + 255u) / 256u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_volume_surface_count(const VolumeSurfaceParams &P, cudaStream_t stream)
{
  volume_surface_count_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  cudaError_t err = cudaGetLastError();
  if(err != cudaSuccess) return err;
  volume_surface_scan_kernel<<<1, VOLUME_SCAN_BLOCK, 0, stream>>>(P.b);
  return cudaGetLastError();
}

cudaError_t launch_volume_surface_write(const VolumeSurfaceParams &P, cudaStream_t stream)
{
  if(P.keys)
    volume_surface_write_kernel<true, false, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  else if(P.intensity)
    volume_surface_write_kernel<false, true, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  else if(P.normals)
    volume_surface_write_kernel<false, false, true><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  else
    volume_surface_write_kernel<false, false, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_volume_mesh_count(const VolumeMeshParams &P, cudaStream_t stream)
{
  volume_mesh_count_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  cudaError_t err = cudaGetLastError();
  if(err != cudaSuccess) return err;
  volume_surface_scan_kernel<<<1, VOLUME_SCAN_BLOCK, 0, stream>>>(P.b);
  return cudaGetLastError();
}

cudaError_t launch_volume_mesh_write(const VolumeMeshParams &P, cudaStream_t stream)
{
  volume_mesh_write_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_volume_raycast(const VolumeRaycastParams &P, const VolumeRaycastColour &C, cudaStream_t stream)
{
  const dim3 block(32, 8);
  const dim3 grid((P.width + block.x - 1) / block.x, (P.height + block.y - 1) / block.y);
  if(C.col)
    volume_raycast_kernel<true><<<grid, block, 0, stream>>>(P, C);
  else
    volume_raycast_kernel<false><<<grid, block, 0, stream>>>(P, C);
  return cudaGetLastError();
}

cudaError_t launch_volume_raycast_normals(const VolumeRaycastParams &P, const VolumeRaycastNormals &N,
                                          cudaStream_t stream)
{
  const dim3 block(32, 8);
  const dim3 grid((P.width + block.x - 1) / block.x, (P.height + block.y - 1) / block.y);
  volume_raycast_normals_kernel<<<grid, block, 0, stream>>>(P, N);
  return cudaGetLastError();
}

cudaError_t launch_volume_prior(const VolumeRaycastParams &P, const VolumePriorSeeds &S, cudaStream_t stream)
{
  const dim3 block(32, 8);
  const dim3 grid((P.width + block.x - 1) / block.x, (P.height + block.y - 1) / block.y);
  volume_prior_kernel<<<grid, block, 0, stream>>>(P, S);
  return cudaGetLastError();
}

cudaError_t launch_volume_shift(const VolumeShiftParams &P, cudaStream_t stream)
{
  const unsigned int n = (unsigned int)P.g.nx * (unsigned int)P.g.ny * (unsigned int)P.g.nz;
  if(P.col)
    volume_shift_kernel<true><<<(n + 255u) / 256u, 256, 0, stream>>>(P);
  else
    volume_shift_kernel<false><<<(n + 255u) / 256u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_volume_spill_count(const VolumeSurfaceParams &P, const VolumeSpillBox &K, cudaStream_t stream)
{
  volume_spill_count_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  cudaError_t err = cudaGetLastError();
  if(err != cudaSuccess) return err;
  volume_surface_scan_kernel<<<1, VOLUME_SCAN_BLOCK, 0, stream>>>(P.b);
  return cudaGetLastError();
}

cudaError_t launch_volume_spill_write(const VolumeSurfaceParams &P, const VolumeSpillBox &K, cudaStream_t stream)
{
  if(P.intensity)
    volume_spill_write_kernel<true, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  else if(P.normals)
    volume_spill_write_kernel<false, true><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  else
    volume_spill_write_kernel<false, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  return cudaGetLastError();
}

cudaError_t launch_volume_spill_mesh_count(const VolumeSurfaceParams &P, const VolumeSpillBox &K, cudaStream_t stream)
{
  volume_spill_mesh_count_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  cudaError_t err = cudaGetLastError();
  if(err != cudaSuccess) return err;
  volume_surface_scan_kernel<<<1, VOLUME_SCAN_BLOCK, 0, stream>>>(P.b);
  return cudaGetLastError();
}

cudaError_t launch_volume_spill_mesh_write(const VolumeSurfaceParams &P, const VolumeSpillBox &K, cudaStream_t stream)
{
  if(P.intensity)
    volume_spill_mesh_write_kernel<true, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  else if(P.normals)
    volume_spill_mesh_write_kernel<false, true><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  else
    volume_spill_mesh_write_kernel<false, false><<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  return cudaGetLastError();
}

cudaError_t launch_volume_spill_tri_count(const VolumeMeshParams &P, const VolumeSpillBox &K, cudaStream_t stream)
{
  volume_spill_tri_count_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  cudaError_t err = cudaGetLastError();
  if(err != cudaSuccess) return err;
  volume_surface_scan_kernel<<<1, VOLUME_SCAN_BLOCK, 0, stream>>>(P.b);
  return cudaGetLastError();
}

cudaError_t launch_volume_spill_tri_write(const VolumeMeshParams &P, const VolumeSpillBox &K, cudaStream_t stream)
{
  volume_spill_tri_write_kernel<<<P.b.n_blocks, VOLUME_SURF_BLOCK, 0, stream>>>(P, K);
  return cudaGetLastError();
}

cudaError_t launch_volume_store_flag(const VolumeStoreParams &P, unsigned int n, cudaStream_t stream)
{
  if(n)
    volume_store_flag_kernel<<<n, VOLUME_STORE_VOXELS, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_volume_store_evict(const VolumeStoreParams &P, unsigned int n, cudaStream_t stream)
{
  if(n && P.col)
    volume_store_evict_kernel<true><<<n, VOLUME_STORE_VOXELS, 0, stream>>>(P);
  else if(n)
    volume_store_evict_kernel<false><<<n, VOLUME_STORE_VOXELS, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_volume_store_restore(const VolumeStoreParams &P, unsigned int n, cudaStream_t stream)
{
  if(n && P.col)
    volume_store_restore_kernel<true><<<n, VOLUME_STORE_VOXELS, 0, stream>>>(P);
  else if(n)
    volume_store_restore_kernel<false><<<n, VOLUME_STORE_VOXELS, 0, stream>>>(P);
  return cudaGetLastError();
}

} // namespace rmdb
