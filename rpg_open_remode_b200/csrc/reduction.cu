// reduction.cu -- single-launch, deterministic image reductions.
//
// Replaces the reference's two-launch shared-memory tree
// (src/reduction_kernels.cu:59-159 driven by src/reduction.cu:81-184, fixed
// 4x4 grid of 16x16 blocks) with one kernel: rows are strided over CTAs,
// columns over threads (coalesced), per-thread accumulation, warp-shuffle
// reduction, one partial per CTA, and the last CTA to finish (atomic ticket)
// folds the partials in a fixed order.  Float sums accumulate in double and
// round once to float, so the result lies within 1/2 ulp + n 2^-53 sum|x| of
// the exact sum (the reference's test compares with a double-accumulated
// cv::sum within 4 ulp, test/reduction_test.cpp:69).
#include "reduction.cuh"

#include <math.h>

namespace rmdb
{

namespace
{

struct Slot  // one 16-byte partial
{
  double a, b;
};

struct SumF32
{
  typedef float In;
  __device__ static Slot identity() { return Slot{0.0, 0.0}; }
  __device__ Slot take(Slot s, float v) const { s.a += (double)v; return s; }
  __device__ static Slot merge(Slot x, Slot y) { return Slot{x.a + y.a, 0.0}; }
};

struct SumI32
{
  typedef int In;
  __device__ static Slot identity() { return Slot{__longlong_as_double(0LL), 0.0}; }
  __device__ Slot take(Slot s, int v) const
  {
    s.a = __longlong_as_double(__double_as_longlong(s.a) + (long long)v);
    return s;
  }
  __device__ static Slot merge(Slot x, Slot y)
  {
    return Slot{__longlong_as_double(__double_as_longlong(x.a) + __double_as_longlong(y.a)), 0.0};
  }
};

struct CountEqI32
{
  typedef int In;
  int value;
  __device__ static Slot identity() { return SumI32::identity(); }
  __device__ Slot take(Slot s, int v) const
  {
    s.a = __longlong_as_double(__double_as_longlong(s.a) + (long long)(v == value));
    return s;
  }
  __device__ static Slot merge(Slot x, Slot y) { return SumI32::merge(x, y); }
};

// fmin / fmax drop NaN operands, so NaN entries are ignored; an image without a non-NaN entry keeps the identity
// (+inf, -inf), which also makes all-+inf and all--inf images come out as (inf, inf) and (-inf, -inf)
struct MinMaxF32
{
  typedef float In;
  __device__ static Slot identity() { return Slot{(double)INFINITY, -(double)INFINITY}; }
  __device__ Slot take(Slot s, float v) const
  {
    s.a = fmin(s.a, (double)v);
    s.b = fmax(s.b, (double)v);
    return s;
  }
  __device__ static Slot merge(Slot x, Slot y) { return Slot{fmin(x.a, y.a), fmax(x.b, y.b)}; }
};

template<typename Op>
__device__ Slot block_fold(Slot acc, Slot *warp_slots)
{
#pragma unroll
  for(int off = 16; off > 0; off >>= 1)
  {
    Slot other;
    other.a = __shfl_down_sync(0xffffffffu, acc.a, off);
    other.b = __shfl_down_sync(0xffffffffu, acc.b, off);
    acc = Op::merge(acc, other);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if(lane == 0) warp_slots[warp] = acc;
  __syncthreads();
  if(warp == 0)
  {
    acc = (lane < (int)(blockDim.x >> 5)) ? warp_slots[lane] : Op::identity();
#pragma unroll
    for(int off = 16; off > 0; off >>= 1)
    {
      Slot other;
      other.a = __shfl_down_sync(0xffffffffu, acc.a, off);
      other.b = __shfl_down_sync(0xffffffffu, acc.b, off);
      acc = Op::merge(acc, other);
    }
  }
  __syncthreads();
  return acc;  // valid in thread 0
}

template<typename Op>
__global__ void __launch_bounds__(256) reduce_kernel(
    const typename Op::In *__restrict__ img, size_t stride, size_t w, size_t h, Op op,
    Slot *partials, unsigned int *ticket, Slot *result)
{
  __shared__ Slot warp_slots[8];
  __shared__ bool is_last;

  Slot acc = Op::identity();
  for(size_t y = blockIdx.x; y < h; y += gridDim.x)
  {
    const typename Op::In *row = img + y * stride;
    for(size_t x = threadIdx.x; x < w; x += blockDim.x)
      acc = op.take(acc, row[x]);
  }
  acc = block_fold<Op>(acc, warp_slots);

  if(threadIdx.x == 0)
  {
    partials[blockIdx.x] = acc;
    __threadfence();
    const unsigned int t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if(!is_last)
    return;

  __threadfence();
  acc = Op::identity();
  const volatile Slot *vp = partials;
  for(unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x)
  {
    Slot s;
    s.a = vp[i].a;
    s.b = vp[i].b;
    acc = Op::merge(acc, s);
  }
  acc = block_fold<Op>(acc, warp_slots);
  if(threadIdx.x == 0)
  {
    *result = acc;
    *ticket = 0u;  // ready for the next launch on this stream
  }
}

template<typename Op>
cudaError_t launch(const typename Op::In *img, size_t stride, size_t w, size_t h, Op op,
                   const ReduceScratch &s, cudaStream_t stream)
{
  if(w == 0 || h == 0)
    return cudaErrorInvalidValue;
  int blocks = (int)(h < (size_t)s.max_blocks ? h : (size_t)s.max_blocks);
  if(blocks < 1) blocks = 1;
  reduce_kernel<Op><<<blocks, 256, 0, stream>>>(
      img, stride, w, h, op, reinterpret_cast<Slot*>(s.partials), s.ticket,
      reinterpret_cast<Slot*>(s.result));
  return cudaGetLastError();
}

} // namespace

cudaError_t launch_sum_f32(const float *img, size_t stride, size_t w, size_t h,
                           const ReduceScratch &s, cudaStream_t stream)
{
  return launch<SumF32>(img, stride, w, h, SumF32(), s, stream);
}

cudaError_t launch_sum_i32(const int *img, size_t stride, size_t w, size_t h,
                           const ReduceScratch &s, cudaStream_t stream)
{
  return launch<SumI32>(img, stride, w, h, SumI32(), s, stream);
}

cudaError_t launch_count_eq_i32(const int *img, size_t stride, size_t w, size_t h, int value,
                                const ReduceScratch &s, cudaStream_t stream)
{
  CountEqI32 op;
  op.value = value;
  return launch<CountEqI32>(img, stride, w, h, op, s, stream);
}

cudaError_t launch_min_max_f32(const float *img, size_t stride, size_t w, size_t h,
                               const ReduceScratch &s, cudaStream_t stream)
{
  return launch<MinMaxF32>(img, stride, w, h, MinMaxF32(), s, stream);
}

} // namespace rmdb
