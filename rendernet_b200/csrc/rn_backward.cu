// rn_backward.cu -- CUDA-core kernels of the BACKWARD (input-gradient) pass of the forward rendering path (SURVEY §8 f-4):
// what inverse rendering differentiates through the frozen network (Reconstruct_RenderNet_Face.py:383-412: tf.gradients of an
// image loss w.r.t. shape / texture / pose).  The dense contractions of the backward pass (data gradients of every stride-1
// convolution and transposed convolution) run on the tensor cores through the same implicit-GEMM kernel as the forward pass
// (rendernet_b200/backward.py: mirrored taps, transposed packed filters); this file holds what is not a GEMM:
//   * activation derivatives (PReLU tools/layer_util.py:27-45, sigmoid RenderNet_Shader.py:127-130),
//   * data gradients of the two thin strided 3-D convolutions e_conv1 / e_conv2 (RenderNet_Shader.py:36-43),
//   * the backward of the trilinear resampler (tools/resampling_voxel_grid.py:381-614 + tools/model_util.py:41-49) with
//     respect to the voxel grid (scatter-add of the 8 corner weights) and to the 3x4 inverse sampling matrix (derivative of
//     the corner weights w.r.t. the sample coordinates), from which the host derives d/d(azimuth, elevation, scale);
//   * the Texture net's 5-channel version of it (geometry + decoded texture sampled at one set of points), and the texture
//     decoder's fp32 PReLU and fully_connected data gradients (RenderNet_Texture_Face_Normal.py:34-46);
//   * the image objectives of inverse rendering: face reconstruction over TensorFlow's Phong composite, and the Shader pose /
//     light fit over the demo's NumPy composite (rendernet_b200/shader_fit.py).
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>

#include "../../include/rendernet_b200.h"
#include "rn_phong.cuh"

namespace rn {
extern std::atomic<long long> g_launch_count;
#define RN_COUNT_LAUNCH() rn::g_launch_count.fetch_add(1, std::memory_order_relaxed)

namespace {
__device__ __forceinline__ void st16(uint16_t* __restrict__ p, long long i, float v, int fmt, long long plane) {
  if (fmt == 1) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    p[i] = *reinterpret_cast<const uint16_t*>(&h);
  } else {
    const __half h = __float2half_rn(v);
    p[i] = *reinterpret_cast<const uint16_t*>(&h);
    if (fmt == 2) {
      const __half l = __float2half_rn(v - __half2float(h));
      p[i + plane] = *reinterpret_cast<const uint16_t*>(&l);
    }
  }
}
__device__ __forceinline__ float ld16(const uint16_t* __restrict__ p, long long i, int fmt, long long plane) {
  const uint16_t u = p[i];
  if (fmt == 1) return __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&u));
  float v = __half2float(*reinterpret_cast<const __half*>(&u));
  if (fmt == 2) {
    const uint16_t l = p[i + plane];
    v += __half2float(*reinterpret_cast<const __half*>(&l));
  }
  return v;
}
inline int grid_for(long long n, int block, int cap = 132 * 32) {
  long long g = (n + block - 1) / block;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}
void same_pad(int n_in, int k, int s, int* n_out, int* pb) {
  *n_out = (n_in + s - 1) / s;
  int total = (*n_out - 1) * s + k - n_in;
  if (total < 0) total = 0;
  *pb = total / 2;
}
}  // namespace

// ------------------------------------------------------------------------------------------ activations
// dL/d(pre-activation) of y = prelu(pre): g * (pre > 0 ? 1 : alpha[c]).  The sign of `pre` is recovered from the stored
// post-activation y (alpha >= 0: sign(y) == sign(pre); y == 0 counts as the negative branch, whose slope is alpha -- which
// is what d/dpre of max(0,pre) + alpha*min(0,pre) gives for pre < 0 and, for alpha = 0, also makes pre = 0 consistent).
__global__ void prelu_backward_kernel(const uint16_t* __restrict__ g, const uint16_t* __restrict__ y,
                                      const float* __restrict__ alpha, uint16_t* __restrict__ out, long long n, int C,
                                      int fmt) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gv = ld16(g, i, fmt, n), yv = ld16(y, i, fmt, n);
    st16(out, i, yv > 0.f ? gv : gv * __ldg(alpha + (i % C)), fmt, n);
  }
}

// Network output: img = sigmoid(logits) fp32 [npix, C]; g = dL/dimg fp32.  out = scale * g * img * (1 - img), written as a
// 16-bit tensor with Cpad >= C channels (zero padded: the data-gradient GEMM of the last up-conv needs K % 16 == 0).
__global__ void sigmoid_backward_kernel(const float* __restrict__ g, const float* __restrict__ img, uint16_t* __restrict__ out,
                                        long long npix, int C, int Cpad, float scale, int fmt) {
  const long long total = npix * Cpad;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / Cpad;
    const int c = static_cast<int>(i % Cpad);
    float v = 0.f;
    if (c < C) {
      const float s = img[p * C + c];
      v = scale * g[p * C + c] * s * (1.f - s);
    }
    st16(out, i, v, fmt, total);
  }
}

// ------------------------------------------------------------------------------------------ thin conv3d, data gradient
// Forward (tf.nn.conv3d SAME, tools/layer_util.py:228-265): y[o] = sum_k x[o*s + k - pb] w[k][ci][co].
// Data gradient: dx[i][ci] = sum over (k, o) with o*s + k - pb == i of g[o][co] w[k][ci][co].  One thread per input voxel,
// all CIN accumulators in registers, the filter ([tap][ci][co] fp32) in shared memory.  g: 16-bit [B,Ho,Wo,Do,COUT];
// dx: 16-bit and/or fp32 [B,H,W,D,CIN].
template <int CIN, int COUT, int K>
__global__ void __launch_bounds__(256) conv3d_bwd_data_kernel(const uint16_t* __restrict__ g, const float* __restrict__ w,
                                                              uint16_t* __restrict__ dx16, float* __restrict__ dx32, int B,
                                                              int H, int W, int D, int Ho, int Wo, int Do, int sy, int sx,
                                                              int sz, int py, int px, int pz, float out_scale, int fmt) {
  __shared__ float ws[K * K * K * CIN * COUT];
  for (int i = threadIdx.x; i < K * K * K * CIN * COUT; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const long long total = static_cast<long long>(B) * H * W * D;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int iz = static_cast<int>(idx % D);
  const int ix = static_cast<int>((idx / D) % W);
  const int iy = static_cast<int>((idx / (static_cast<long long>(D) * W)) % H);
  const int b = static_cast<int>(idx / (static_cast<long long>(D) * W * H));
  const long long gplane = static_cast<long long>(B) * Ho * Wo * Do * COUT;
  float acc[CIN];
#pragma unroll
  for (int c = 0; c < CIN; ++c) acc[c] = 0.f;
  for (int ky = 0; ky < K; ++ky) {
    const int ny = iy + py - ky;
    if (ny < 0 || ny % sy != 0) continue;
    const int oy = ny / sy;
    if (oy >= Ho) continue;
    for (int kx = 0; kx < K; ++kx) {
      const int nx = ix + px - kx;
      if (nx < 0 || nx % sx != 0) continue;
      const int ox = nx / sx;
      if (ox >= Wo) continue;
      for (int kz = 0; kz < K; ++kz) {
        const int nz = iz + pz - kz;
        if (nz < 0 || nz % sz != 0) continue;
        const int oz = nz / sz;
        if (oz >= Do) continue;
        const long long gi = (((static_cast<long long>(b) * Ho + oy) * Wo + ox) * Do + oz) * COUT;
        const float* wt = ws + ((ky * K + kx) * K + kz) * CIN * COUT;
#pragma unroll
        for (int co = 0; co < COUT; ++co) {
          const float gv = ld16(g, gi + co, fmt, gplane);
#pragma unroll
          for (int ci = 0; ci < CIN; ++ci) acc[ci] = fmaf(gv, wt[ci * COUT + co], acc[ci]);
        }
      }
    }
  }
#pragma unroll
  for (int ci = 0; ci < CIN; ++ci) {
    const long long o = idx * CIN + ci;
    if (dx16 != nullptr) st16(dx16, o, acc[ci], fmt, total * CIN);
    if (dx32 != nullptr) dx32[o] = acc[ci] * out_scale;
  }
}

// ------------------------------------------------------------------------------------------ fixed-order twins: helpers
// The resampler backward's scatter-add in fixed point (the twins run under torch.use_deterministic_algorithms, DESIGN §8b).
// Per batch item and channel, m = max |G| (an integer max of the fp32 bit patterns: order-free, and NaN sorts above Inf) fixes a
// power of two 2^k with m 2^k < 2^(62 - L), 2^L >= new_size^3.  Every corner weight is <= 1 and each sample point adds to each of
// its 8 corners once, so a corner takes at most new_size^3 contributions, each rounded to an integer of magnitude <= 2^(62 - L):
// the int64 sum stays within 2^62 for every pose.  Integer addition is associative, so the sum does not depend on the order of
// the atomics; one contribution is rounded by at most 2^-k / 2 <= 2^(L - 62) m, 2^-41 m at new_size = 128.
constexpr unsigned FX_NONFINITE = 0x7f800000u;                       // |G| bit patterns at or above this are Inf / NaN

__host__ __device__ inline int fx_exponent(float max_abs, int lg_points) {
  if (!(max_abs > 0.f) || !(max_abs <= 3.402823466e38f)) return 0;    // 0, or non-finite (handled by the caller)
  int e;
  frexpf(max_abs, &e);                                                 // max_abs < 2^e (subnormals included)
  return 62 - lg_points - e;
}

__device__ __forceinline__ double fx_scale(unsigned amax_bits, int lg_points) {
  return amax_bits >= FX_NONFINITE ? 0.0 : ldexp(1.0, fx_exponent(__uint_as_float(amax_bits), lg_points));
}

// one contribution: the fp32 product w g of the atomic kernel, scaled in double and rounded once; two's complement wraps, so
// unsigned addition is int64 addition
template <bool FX>
__device__ __forceinline__ void scatter_add(float* __restrict__ dst, unsigned long long* __restrict__ acc, size_t i, float v,
                                            double scale) {
  if constexpr (FX) atomicAdd(acc + i, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(v) * scale)));
  else atomicAdd(dst + i, v);
}

// amax[b * C + c] = max over the item's points of |G[b, point, c]|'s bit pattern (amax zeroed by the caller); blockIdx.y = item.
template <int C>
__global__ void __launch_bounds__(256) absmax_bits_kernel(const float* __restrict__ g, unsigned* __restrict__ amax,
                                                          long long points) {
  __shared__ unsigned red[8][C];
  const unsigned* gb = reinterpret_cast<const unsigned*>(g) + static_cast<size_t>(blockIdx.y) * points * C;
  unsigned m[C];
#pragma unroll
  for (int c = 0; c < C; ++c) m[c] = 0u;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < points;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
#pragma unroll
    for (int c = 0; c < C; ++c) m[c] = max(m[c], gb[p * C + c] & 0x7fffffffu);
  }
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    unsigned v = m[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) red[wib][c] = v;
  }
  __syncthreads();
  if (threadIdx.x < C) {
    unsigned v = 0u;
    for (int w = 0; w < 8; ++w) v = max(v, red[w][threadIdx.x]);
    atomicMax(amax + blockIdx.y * C + threadIdx.x, v);
  }
}

// out[b][i] = acc[b][i] 2^-k as fp32, k from amax[b * C_amax + c0 + i % Cout]; NaN for the whole item when any of its C_amax
// channels holds a non-finite G.  blockIdx.y = item.
__global__ void __launch_bounds__(256) fx_finalize_kernel(const unsigned long long* __restrict__ acc, const unsigned* __restrict__ amax,
                                                          int C_amax, int c0, int lg_points, float* __restrict__ out,
                                                          long long per_item, int Cout) {
  const unsigned* am = amax + blockIdx.y * C_amax;
  bool bad = false;
  for (int c = 0; c < C_amax; ++c) bad |= am[c] >= FX_NONFINITE;
  const size_t base = static_cast<size_t>(blockIdx.y) * per_item;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < per_item;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % Cout);
    const double inv = ldexp(1.0, -fx_exponent(__uint_as_float(am[c0 + c]), lg_points));
    out[base + i] = bad ? __int_as_float(0x7fffffff)
                        : __double2float_rn(__ll2double_rn(static_cast<long long>(acc[base + i])) * inv);
  }
}

// The fixed-order second stage of every twin: per item b and entry j < width, the sum over the item's nblk block partials
// part[(b * nblk + k) * width + j] in double.  One warp per (b, j): lane l adds k = l, l + 32, ... in order, then a fixed
// butterfly.  Entries j < nd go to out_d[b * nd + j] (double), the rest to out_f[b * (width - nd) + j - nd] (fp32; may be NULL).
// amax (may be NULL): the item's sums become NaN when any of its namax channels holds a non-finite G.
__global__ void __launch_bounds__(256) slot_sum_kernel(const double* __restrict__ part, int B, int nblk, int width, int nd,
                                                       double* __restrict__ out_d, float* __restrict__ out_f,
                                                       const unsigned* __restrict__ amax, int namax) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= B * width) return;                                          // whole warps leave together
  const int b = w / width, j = w % width;
  double s = 0.0;
  for (int k = lane; k < nblk; k += 32) s += part[(static_cast<size_t>(b) * nblk + k) * width + j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane != 0) return;
  if (amax != nullptr)
    for (int c = 0; c < namax; ++c)
      if (amax[b * namax + c] >= FX_NONFINITE) s = __longlong_as_double(0x7ff8000000000000LL);
  if (j < nd) out_d[b * nd + j] = s;
  else if (out_f != nullptr) out_f[b * (width - nd) + j - nd] = static_cast<float>(s);
}

// ------------------------------------------------------------------------------------------ resampler backward
// Forward (rn_resample_f32, transform = 1): N[b,p,q,r,c] = sum_corners w_k(x,y,z) V[b, corner_k, c] with
// (x,y,z) = Minv[b] . (r, new-1-p, q, 1), zero outside [0, size-1)^3.  Given G = dL/dN:
//   dL/dV[b, corner_k, c] += w_k G[b,p,q,r,c]                                                        (scatter-add)
//   dL/dMinv[b][a][j]     += sum_c G * (dN/d coord_a) * (r, new-1-p, q, 1)[j],   dN/dx = sum_k (dw_k/dx) V[corner_k], ...
// The floor() inside the weights is piecewise constant, so the derivative is the one of the trilinear patch the point
// lies in (what tf.gradients produces for tools/resampling_voxel_grid.py:465-485).  One warp per output row; the 12 matrix
// partial sums are reduced in the warp, then in the block, then one atomicAdd per block and entry.
// FX (the fixed-order twin): dvox and dminv are unused; the scatter adds fixed-point integers to acc [B,size^3,C] (scale from amax,
// see scatter_add) and each block writes its 12 partial sums to slots[blockIdx.x][12] (a block's rows lie in one item).
template <int C, bool FX>
__global__ void __launch_bounds__(256) resample_backward_kernel(const float* __restrict__ vox, const float* __restrict__ minv,
                                                                const float* __restrict__ gout, float* __restrict__ dvox,
                                                                float* __restrict__ dminv, int B, int size, int nsz,
                                                                int transform, unsigned long long* __restrict__ acc,
                                                                const unsigned* __restrict__ amax, int lg_points,
                                                                double* __restrict__ slots) {
  __shared__ float red[8][12];
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int rows = B * nsz * nsz;
  float dm[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) dm[i] = 0.f;
  int b = 0;
  if (warp_global < rows) {
    b = warp_global / (nsz * nsz);
    const int o1 = (warp_global / nsz) % nsz;
    const int o2 = warp_global % nsz;
    const float* M = minv + b * 12;
    const float m00 = __ldg(M + 0), m01 = __ldg(M + 1), m02 = __ldg(M + 2), m03 = __ldg(M + 3);
    const float m10 = __ldg(M + 4), m11 = __ldg(M + 5), m12 = __ldg(M + 6), m13 = __ldg(M + 7);
    const float m20 = __ldg(M + 8), m21 = __ldg(M + 9), m22 = __ldg(M + 10), m23 = __ldg(M + 11);
    const float gy = transform ? static_cast<float>(nsz - 1 - o1) : static_cast<float>(o2);
    const float gz = transform ? static_cast<float>(o2) : static_cast<float>(o1);
    const float lim = static_cast<float>(size - 1);
    const float* vb = vox + static_cast<size_t>(b) * size * size * size * C;
    float* dvb = dvox != nullptr ? dvox + static_cast<size_t>(b) * size * size * size * C : nullptr;
    unsigned long long* avb = FX && acc != nullptr ? acc + static_cast<size_t>(b) * size * size * size * C : nullptr;
    double sc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) sc[c] = FX ? fx_scale(__ldg(amax + b * C + c), lg_points) : 0.0;
    const float* grow = gout + static_cast<size_t>(warp_global) * nsz * C;
    for (int r = lane; r < nsz; r += 32) {
      const float gx = static_cast<float>(r);
      // same coordinate arithmetic as the forward kernels (rn_ops.cu sample_coord): identical in/out decisions
      const float x = __fadd_rn(__fmaf_rn(m02, gz, __fmaf_rn(m01, gy, __fmul_rn(m00, gx))), m03);
      const float y = __fadd_rn(__fmaf_rn(m12, gz, __fmaf_rn(m11, gy, __fmul_rn(m10, gx))), m13);
      const float z = __fadd_rn(__fmaf_rn(m22, gz, __fmaf_rn(m21, gy, __fmul_rn(m20, gx))), m23);
      if (!(x >= 0.f && x < lim && y >= 0.f && y < lim && z >= 0.f && z < lim)) continue;
      const float x0f = floorf(x), y0f = floorf(y), z0f = floorf(z);
      const int x0 = static_cast<int>(x0f), y0 = static_cast<int>(y0f), z0 = static_cast<int>(z0f);
      const float ax = (x0f + 1.f) - x, bx = x - x0f, ay = (y0f + 1.f) - y, by = y - y0f, az = (z0f + 1.f) - z, bz = z - z0f;
      const size_t i000 = ((static_cast<size_t>(z0) * size + y0) * size + x0) * C;
      const size_t sy = static_cast<size_t>(size) * C, sz = static_cast<size_t>(size) * size * C;
      float dvx = 0.f, dvy = 0.f, dvz = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float gv = grow[static_cast<size_t>(r) * C + c];
        if (gv == 0.f) continue;
        const float Ia = __ldg(vb + i000 + c), Ib = __ldg(vb + i000 + sy + c);
        const float Ic = __ldg(vb + i000 + C + c), Id = __ldg(vb + i000 + sy + C + c);
        const float Ie = __ldg(vb + i000 + sz + c), If = __ldg(vb + i000 + sz + sy + c);
        const float Ig = __ldg(vb + i000 + sz + C + c), Ih = __ldg(vb + i000 + sz + sy + C + c);
        // corners a:(x0,y0,z0) b:(x0,y1,z0) c:(x1,y0,z0) d:(x1,y1,z0) e..h: z1   (tools/resampling_voxel_grid.py:440-449)
        dvx += gv * (ay * az * (Ic - Ia) + by * az * (Id - Ib) + ay * bz * (Ig - Ie) + by * bz * (Ih - If));
        dvy += gv * (ax * az * (Ib - Ia) + bx * az * (Id - Ic) + ax * bz * (If - Ie) + bx * bz * (Ih - Ig));
        dvz += gv * (ax * ay * (Ie - Ia) + ax * by * (If - Ib) + bx * ay * (Ig - Ic) + bx * by * (Ih - Id));
        if (FX ? avb != nullptr : dvb != nullptr) {
          scatter_add<FX>(dvb, avb, i000 + c, ax * ay * az * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + sy + c, ax * by * az * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + C + c, bx * ay * az * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + sy + C + c, bx * by * az * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + sz + c, ax * ay * bz * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + sz + sy + c, ax * by * bz * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + sz + C + c, bx * ay * bz * gv, sc[c]);
          scatter_add<FX>(dvb, avb, i000 + sz + sy + C + c, bx * by * bz * gv, sc[c]);
        }
      }
      dm[0] += dvx * gx; dm[1] += dvx * gy; dm[2] += dvx * gz; dm[3] += dvx;
      dm[4] += dvy * gx; dm[5] += dvy * gy; dm[6] += dvy * gz; dm[7] += dvy;
      dm[8] += dvz * gx; dm[9] += dvz * gy; dm[10] += dvz * gz; dm[11] += dvz;
    }
  }
  if (FX ? slots == nullptr : dminv == nullptr) return;
  // rows of one block belong to one batch item when nsz*nsz % 8 == 0 (checked by the host): reduce within the block
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    float v = dm[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[wib][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    float v = 0.f;
    for (int wv = 0; wv < 8; ++wv) v += red[wv][threadIdx.x];
    const int first_row = (blockIdx.x * blockDim.x) >> 5;
    if constexpr (FX) slots[static_cast<size_t>(blockIdx.x) * 12 + threadIdx.x] = v;
    else if (first_row < rows && v != 0.f) atomicAdd(dminv + (first_row / (nsz * nsz)) * 12 + threadIdx.x, v);
  }
}

// Texture net input chain (resample5_conv1_kernel in rn_ops.cu; RenderNet_Texture_Face_Normal.py:155-179 and
// Reconstruct_RenderNet_Face.py:367-378): the geometry grid (C = 1) and the texture volume (C = 4) are sampled at the SAME
// points and concatenated, G = dL/d(concat) [B,N,N,N,5].  Each sample coordinate is computed once, with the forward kernel's
// sample_coord arithmetic and in/out test; channel 0 scatters into dvox, channels 1..4 into dtex (float4 corner gathers), and
// dM^-1 collects all five channels.  Per corner the five channels are first contracted to s_k = G0 V_k + G1..4 . T_k, so
// d/dx = sum_k (dw_k/dx) s_k.  Same warp-per-row layout and block reduction as resample_backward_kernel.  G covers the window
// of rows [wy0, wy0+wh) x columns [wx0, wx0+ww) (all depths; the whole grid: 0, 0, nsz, nsz), [B,wh,ww,nsz,5]: only the
// points of that window scatter.  FX (the fixed-order twin, whole grid): as resample_backward_kernel's, with acc_vox [B,size^3],
// acc_tex [B,size^3,4] and one scale per item and channel of G (amax [B,5]).
template <bool FX>
__global__ void __launch_bounds__(256) resample5_backward_kernel(const float* __restrict__ vox, const float* __restrict__ tex,
                                                                 const float* __restrict__ minv, const float* __restrict__ gout,
                                                                 float* __restrict__ dvox, float* __restrict__ dtex,
                                                                 float* __restrict__ dminv, int B, int size, int nsz, int wy0,
                                                                 int wx0, int wh, int ww, unsigned long long* __restrict__ acc_vox,
                                                                 unsigned long long* __restrict__ acc_tex,
                                                                 const unsigned* __restrict__ amax, int lg_points,
                                                                 double* __restrict__ slots) {
  __shared__ float red[8][12];
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int rows = B * wh * ww;
  float dm[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) dm[i] = 0.f;
  if (warp_global < rows) {
    const int b = warp_global / (wh * ww);
    const int o1 = wy0 + (warp_global / ww) % wh;
    const int o2 = wx0 + warp_global % ww;
    const float* M = minv + b * 12;
    const float m00 = __ldg(M + 0), m01 = __ldg(M + 1), m02 = __ldg(M + 2), m03 = __ldg(M + 3);
    const float m10 = __ldg(M + 4), m11 = __ldg(M + 5), m12 = __ldg(M + 6), m13 = __ldg(M + 7);
    const float m20 = __ldg(M + 8), m21 = __ldg(M + 9), m22 = __ldg(M + 10), m23 = __ldg(M + 11);
    const float gy = static_cast<float>(nsz - 1 - o1), gz = static_cast<float>(o2);    // axis transform, as the forward
    const float lim = static_cast<float>(size - 1);
    const size_t vol = static_cast<size_t>(size) * size * size;
    const float* vb = vox + static_cast<size_t>(b) * vol;
    const float4* tb = reinterpret_cast<const float4*>(tex) + static_cast<size_t>(b) * vol;
    float* dvb = dvox != nullptr ? dvox + static_cast<size_t>(b) * vol : nullptr;
    float* dtb = dtex != nullptr ? dtex + static_cast<size_t>(b) * vol * 4 : nullptr;
    unsigned long long* avb = FX && acc_vox != nullptr ? acc_vox + static_cast<size_t>(b) * vol : nullptr;
    unsigned long long* atb = FX && acc_tex != nullptr ? acc_tex + static_cast<size_t>(b) * vol * 4 : nullptr;
    double sc[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) sc[c] = FX ? fx_scale(__ldg(amax + b * 5 + c), lg_points) : 0.0;
    const size_t sy = static_cast<size_t>(size), sz = static_cast<size_t>(size) * size;
    const float* grow = gout + static_cast<size_t>(warp_global) * nsz * 5;
    for (int r = lane; r < nsz; r += 32) {
      const float gx = static_cast<float>(r);
      const float x = __fadd_rn(__fmaf_rn(m02, gz, __fmaf_rn(m01, gy, __fmul_rn(m00, gx))), m03);
      const float y = __fadd_rn(__fmaf_rn(m12, gz, __fmaf_rn(m11, gy, __fmul_rn(m10, gx))), m13);
      const float z = __fadd_rn(__fmaf_rn(m22, gz, __fmaf_rn(m21, gy, __fmul_rn(m20, gx))), m23);
      if (!(x >= 0.f && x < lim && y >= 0.f && y < lim && z >= 0.f && z < lim)) continue;
      const float* gp = grow + static_cast<size_t>(r) * 5;
      const float g0 = gp[0], g1 = gp[1], g2 = gp[2], g3 = gp[3], g4 = gp[4];
      if (g0 == 0.f && g1 == 0.f && g2 == 0.f && g3 == 0.f && g4 == 0.f) continue;
      const float x0f = floorf(x), y0f = floorf(y), z0f = floorf(z);
      const int x0 = static_cast<int>(x0f), y0 = static_cast<int>(y0f), z0 = static_cast<int>(z0f);
      const float ax = (x0f + 1.f) - x, bx = x - x0f, ay = (y0f + 1.f) - y, by = y - y0f, az = (z0f + 1.f) - z, bz = z - z0f;
      const size_t c000 = (static_cast<size_t>(z0) * size + y0) * size + x0;
      // corners a:(x0,y0,z0) b:(x0,y1,z0) c:(x1,y0,z0) d:(x1,y1,z0) e..h: z1   (tools/resampling_voxel_grid.py:440-449)
      const size_t off[8] = {c000, c000 + sy, c000 + 1, c000 + sy + 1, c000 + sz, c000 + sz + sy, c000 + sz + 1, c000 + sz + sy + 1};
      const float wk[8] = {ax * ay * az, ax * by * az, bx * ay * az, bx * by * az, ax * ay * bz, ax * by * bz, bx * ay * bz, bx * by * bz};
      float s[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float4 t = __ldg(tb + off[k]);
        s[k] = g0 * __ldg(vb + off[k]) + g1 * t.x + g2 * t.y + g3 * t.z + g4 * t.w;
      }
      const float dvx = ay * az * (s[2] - s[0]) + by * az * (s[3] - s[1]) + ay * bz * (s[6] - s[4]) + by * bz * (s[7] - s[5]);
      const float dvy = ax * az * (s[1] - s[0]) + bx * az * (s[3] - s[2]) + ax * bz * (s[5] - s[4]) + bx * bz * (s[7] - s[6]);
      const float dvz = ax * ay * (s[4] - s[0]) + ax * by * (s[5] - s[1]) + bx * ay * (s[6] - s[2]) + bx * by * (s[7] - s[3]);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if ((FX ? avb != nullptr : dvb != nullptr) && g0 != 0.f) scatter_add<FX>(dvb, avb, off[k], wk[k] * g0, sc[0]);
        if (FX ? atb != nullptr : dtb != nullptr) {
          const size_t d = off[k] * 4;
          scatter_add<FX>(dtb, atb, d + 0, wk[k] * g1, sc[1]); scatter_add<FX>(dtb, atb, d + 1, wk[k] * g2, sc[2]);
          scatter_add<FX>(dtb, atb, d + 2, wk[k] * g3, sc[3]); scatter_add<FX>(dtb, atb, d + 3, wk[k] * g4, sc[4]);
        }
      }
      dm[0] += dvx * gx; dm[1] += dvx * gy; dm[2] += dvx * gz; dm[3] += dvx;
      dm[4] += dvy * gx; dm[5] += dvy * gy; dm[6] += dvy * gz; dm[7] += dvy;
      dm[8] += dvz * gx; dm[9] += dvz * gy; dm[10] += dvz * gz; dm[11] += dvz;
    }
  }
  if (FX ? slots == nullptr : dminv == nullptr) return;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    float v = dm[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[wib][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    float v = 0.f;
    for (int wv = 0; wv < 8; ++wv) v += red[wv][threadIdx.x];
    const int first_row = (blockIdx.x * blockDim.x) >> 5;
    if constexpr (FX) slots[static_cast<size_t>(blockIdx.x) * 12 + threadIdx.x] = v;
    else if (first_row < rows && v != 0.f) atomicAdd(dminv + (first_row / (wh * ww)) * 12 + threadIdx.x, v);
  }
}

// ------------------------------------------------------------------------------------------ texture decoder, backward
// fp32 PReLU derivative (decoder layers, tools/layer_util.py:27-45): out = g * (z > 0 ? 1 : alpha[c]) with z the
// PRE-activation (the decoder's slopes may be negative, so the output's sign does not tell the branch).
__global__ void prelu_backward_f32_kernel(const float* __restrict__ g, const float* __restrict__ z, const float* __restrict__ alpha,
                                          float* __restrict__ out, long long n, int C) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gv = g[i];
    out[i] = z[i] > 0.f ? gv : gv * __ldg(alpha + (i % C));
  }
}

// Data gradient of fully_connected (tools/layer_util.py:311-343, y = x W + b, W TF [K,N]): dx[b][k] = sum_n g[b][n] W[k][n].
// Bandwidth-bound (W is 104 MB at K = 199, N = 2^17): W is read once for the whole batch.  Stage 1: one CTA per FCB_NC-wide
// chunk of n stages that chunk of g for every batch item in shared memory; warp w takes rows k = w, w+8, ..., each lane reads
// 16 W values (float4, coalesced) and accumulates BMAX dot products, reduced across the warp; lane b writes the chunk's partial
// sum part[chunk][b][k].  Stage 2 sums the partials over the chunks in a fixed order: no float atomics, bit-reproducible.
constexpr int FCB_NC = 512;
template <int BMAX>
__global__ void __launch_bounds__(256) fc_bwd_data_partial_kernel(const float* __restrict__ g, const float* __restrict__ w,
                                                                  float* __restrict__ part, int B, int K, int N) {
  extern __shared__ __align__(16) float gs[];            // [B][FCB_NC]
  const int chunk = blockIdx.x;
  const int n0 = chunk * FCB_NC;
  for (int i = threadIdx.x; i < B * FCB_NC; i += blockDim.x) {
    const int b = i / FCB_NC, n = n0 + (i - b * FCB_NC);
    gs[i] = n < N ? g[static_cast<size_t>(b) * N + n] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int k = wid; k < K; k += 8) {
    const float* wr = w + static_cast<size_t>(k) * N + n0;
    float acc[BMAX];
#pragma unroll
    for (int b = 0; b < BMAX; ++b) acc[b] = 0.f;
#pragma unroll
    for (int i = 0; i < FCB_NC / 128; ++i) {
      const int j = 4 * lane + 128 * i;
      float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n0 + j + 3 < N) wv = __ldg(reinterpret_cast<const float4*>(wr + j));
      else {
        if (n0 + j < N) wv.x = __ldg(wr + j);
        if (n0 + j + 1 < N) wv.y = __ldg(wr + j + 1);
        if (n0 + j + 2 < N) wv.z = __ldg(wr + j + 2);
      }
#pragma unroll
      for (int b = 0; b < BMAX; ++b) {
        if (b < B) {
          const float4 gv = *reinterpret_cast<const float4*>(gs + b * FCB_NC + j);
          acc[b] = fmaf(gv.x, wv.x, fmaf(gv.y, wv.y, fmaf(gv.z, wv.z, fmaf(gv.w, wv.w, acc[b]))));
        }
      }
    }
    float mine = 0.f;
#pragma unroll
    for (int b = 0; b < BMAX; ++b) {
      if (b < B) {
        float v = acc[b];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == b) mine = v;
      }
    }
    if (lane < B) part[(static_cast<size_t>(chunk) * B + lane) * K + k] = mine;
  }
}

__global__ void fc_bwd_data_reduce_kernel(const float* __restrict__ part, float* __restrict__ dx, int nchunks, int BK) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BK) return;
  float s = 0.f;
  for (int c = 0; c < nchunks; ++c) s += part[static_cast<size_t>(c) * BK + i];
  dx[i] = s;
}

// ------------------------------------------------------------------------------------------ shading-parameter gradients
// The SP instantiations of the three Phong kernels below (rn_*_params) also sum, per item, dL/d light_col (3) and dL/d ambient
// (phong_param_backward, rn_phong.cuh) and read the ambient term per item from ambient_b[b].  block_sum4 reduces the four terms
// over the block (the result in thread 0) and store_param_grads writes them: one atomic per block and component (d_col [B,3],
// d_amb [B], each may be NULL), or FX: to pslots[b][blockIdx.x][3] (colour) and pslots[3 B nblk + b nblk + blockIdx.x]
// (ambient), summed in block order by slot_sum_kernel.  Every thread of the block calls block_sum4.
__device__ __forceinline__ void block_sum4(float* v) {
  __shared__ float red4[8][4];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float x = v[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    if (lane == 0) red4[wib][i] = x;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) v[i] = 0.f;
    for (int w = 0; w < 8; ++w)
      for (int i = 0; i < 4; ++i) v[i] += red4[w][i];
  }
}

template <bool FX>
__device__ __forceinline__ void store_param_grads(const float* v, int b, float* d_col, float* d_amb, double* pslots) {
  if constexpr (FX) {
    double* sl = pslots + (static_cast<size_t>(b) * gridDim.x + blockIdx.x) * 3;
    for (int i = 0; i < 3; ++i) sl[i] = v[i];
    pslots[3 * static_cast<size_t>(gridDim.y) * gridDim.x + static_cast<size_t>(b) * gridDim.x + blockIdx.x] = v[3];
  } else {
    if (d_col != nullptr)
      for (int i = 0; i < 3; ++i) atomicAdd(d_col + 3 * b + i, v[i]);
    if (d_amb != nullptr) atomicAdd(d_amb + b, v[3]);
  }
}

// ------------------------------------------------------------------------------------------ face reconstruction objective
// Reconstruct_RenderNet_Face.py:372-383 over TensorFlow's Phong composite (tools/Phong_shading.py:24-113 tf_mask /
// tf_mask_white / tf_phong_shading / tf_phong_composite -- NOT the NumPy composite of phong_pixel):
//   shade = tf_phong_pixel(n, L = l / |l|, col, ambient, k_d, black, with_mask)     (rn_phong.cuh: the image rn_phong_shade renders)
//   loss[b] = mean_{h,w,c} (target - albedo_c shade_c)^2
// and its gradient in one pass: with g_c = dL/d(compos_c) = 2 (compos_c - target_c) / (3 HW), compos = albedo shade in fp32,
// d_albedo_c = g_c shade_c and dL/d(shade_c) = g_c albedo_c, the latter through tf_phong_pixel_backward on the terms the forward
// call recorded.  g is formed in double and rounded once: it is the fp32 value autograd of a float64 MSE on rn_phong_shade's
// compos hands rn_phong_shade_backward, so the fused and the composed objectives give the same image gradients.  TF-1's gradient
// conventions: tf.maximum(x, y) passes to x where x >= y; clip_by_value(x, lo, hi) passes where lo <= x <= hi; d|x|/dx = x/|x|.
// At n = (0.5, 0.5, 0.5) u = 0/0 and d are NaN: the forward shades the pixel as unlit, only the mask term reaches d_normal and
// the pixel adds nothing to d_light.  Where |n| = 0 the mask term is 0.  One thread per pixel; blockIdx.y = batch item.  loss is
// accumulated in double (one atomic per block); dL/dL is reduced over the block and mapped through the normalisation
// (I - L L^T) / |l| before one atomic per block and component.  FX (the fixed-order twin): the block's loss and d_light terms go
// to slots[b][blockIdx.x][4] instead, summed in block order by slot_sum_kernel; the per-pixel code is the same.  SP: see
// block_sum4 (pslots is used by FX only, d_col / d_amb by the atomic kernel only).
template <bool FX, bool SP>
__global__ void __launch_bounds__(256) phong_recon_loss_grad_kernel(const float* __restrict__ albedo, const float* __restrict__ normal,
                                                                    const float* __restrict__ target, const float* __restrict__ light_dir,
                                                                    const float* __restrict__ light_col, float ambient, float k_diffuse,
                                                                    int black, int with_mask, double* __restrict__ loss,
                                                                    float* __restrict__ d_albedo, float* __restrict__ d_normal,
                                                                    float* __restrict__ d_light, int HW, double* __restrict__ slots,
                                                                    const float* __restrict__ ambient_b, float* __restrict__ d_col,
                                                                    float* __restrict__ d_amb, double* __restrict__ pslots) {
  __shared__ float red[8][4];
  const int b = blockIdx.y;
  if constexpr (SP) ambient = __ldg(ambient_b + b);
  float pg[4] = {0.f, 0.f, 0.f, 0.f};                                  // SP: dL/d col (3), dL/d ambient
  const float l0 = __ldg(light_dir + 3 * b), l1 = __ldg(light_dir + 3 * b + 1), l2 = __ldg(light_dir + 3 * b + 2);
  const float lnorm = sqrtf(l0 * l0 + l1 * l1 + l2 * l2);
  const float L[3] = {l0 / lnorm, l1 / lnorm, l2 / lnorm};
  const float col[3] = {__ldg(light_col + 3 * b), __ldg(light_col + 3 * b + 1), __ldg(light_col + 3 * b + 2)};
  const double inv_n = 1.0 / (3.0 * static_cast<double>(HW));         // d mean / d compos
  float part[4] = {0.f, 0.f, 0.f, 0.f};                                // loss, dL/dL (3)
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < HW) {
    const size_t o = (static_cast<size_t>(b) * HW + p) * 3;
    const float n[3] = {normal[o], normal[o + 1], normal[o + 2]};
    float shade[3], ds[3], dn[3];
    TfPhongTerms t;
    tf_phong_pixel(n[0], n[1], n[2], L, col, ambient, k_diffuse, black, with_mask, shade, &t);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float a = albedo[o + c];
      const float compos = __fmul_rn(a, shade[c]);                     // the fp32 compos rn_phong_shade returns
      const float r = __fsub_rn(compos, target[o + c]);
      part[0] += r * r;
      const float dpred = static_cast<float>(2.0 * __dmul_rn(inv_n, __dsub_rn(compos, target[o + c])));
      d_albedo[o + c] = dpred * shade[c];
      ds[c] = dpred * a;
    }
    tf_phong_pixel_backward(n, L, t, col, ambient, k_diffuse, black, with_mask, ds, dn, part + 1);
    if constexpr (SP) phong_param_backward(t.d, t.m, t.pre, t.x, k_diffuse, with_mask, ds, pg, pg + 3);
#pragma unroll
    for (int i = 0; i < 3; ++i) d_normal[o + i] = dn[i];
  }
  if constexpr (SP) {
    if (FX ? pslots != nullptr : (d_col != nullptr || d_amb != nullptr)) {
      block_sum4(pg);
      if (threadIdx.x == 0) store_param_grads<FX>(pg, b, d_col, d_amb, pslots);
    }
  }
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float v = part[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) red[wib][i] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    for (int w = 0; w < 8; ++w)
      for (int i = 0; i < 4; ++i) t[i] += red[w][i];
    const float ldt = L[0] * t[1] + L[1] * t[2] + L[2] * t[3];           // d (l/|l|) = (dL - L (L.dL)) / |l|
    if constexpr (FX) {
      double* sl = slots + (static_cast<size_t>(b) * gridDim.x + blockIdx.x) * 4;
      sl[0] = static_cast<double>(t[0]) / (3.0 * HW);
      for (int i = 0; i < 3; ++i) sl[1 + i] = (t[1 + i] - L[i] * ldt) / lnorm;
    } else {
      atomicAdd(loss + b, static_cast<double>(t[0]) / (3.0 * HW));
      if (d_light != nullptr)
        for (int i = 0; i < 3; ++i) atomicAdd(d_light + 3 * b + i, (t[1 + i] - L[i] * ldt) / lnorm);
    }
  }
}

// ------------------------------------------------------------------------------------------ Shader pose / light fit objective
// The demo's NumPy composite (RenderNet_demo.py:54-58, tools/Phong_shading.py:138-228) against a target image:
//   out = phong_pixel(img, l, col, ambient, k_d, white, with_mask)     (rn_phong.cuh: the image rn_phong_composite renders)
//   loss[b] += mean_{h,w,c} (target - out)^2                           (double)
// and its gradients in the same pass, with the conventions of phong_recon_loss_grad_kernel: max(x, 0) passes where x >= 0, a
// clip where lo <= x <= hi.  Three paths reach img: the normalisation d = (img - 0.5) . L / |img - 0.5| (dd/dv = (L - d u) / |v|,
// u = v / |v|), and the soft mask m = sigmoid(255 |img| - 150) (black) / sigmoid(255 |1 - img| - 80) (white), whose derivative
// m (1 - m) 255 (+-a / |a|) is evaluated in double from the fp32 pixel (the argument multiplies |a|'s rounding by 255).  dL/dL
// = dd u is reduced over the block and mapped through the light's normalisation (I - L L^T) / |l|.  At img = (0.5, 0.5, 0.5)
// d is 0 * inf = NaN; phong_pixel's fmaxf turns it into 0 (the pixel is shaded as if unlit) and the gradient passes nothing
// through the normal there (only the mask term reaches d_img; nothing reaches d_light).  Where |a| = 0 the mask term is 0.
// FX: slots[b][blockIdx.x][4] as phong_recon_loss_grad_kernel's.  SP: as phong_recon_loss_grad_kernel's.
template <bool FX, bool SP>
__global__ void __launch_bounds__(256) phong_composite_loss_grad_kernel(const float* __restrict__ img, const float* __restrict__ target,
                                                                        const float* __restrict__ light_dir,
                                                                        const float* __restrict__ light_col, float ambient,
                                                                        float k_diffuse, int white, int with_mask,
                                                                        double* __restrict__ loss, float* __restrict__ d_img,
                                                                        float* __restrict__ d_light, int HW, double* __restrict__ slots,
                                                                        const float* __restrict__ ambient_b, float* __restrict__ d_col,
                                                                        float* __restrict__ d_amb, double* __restrict__ pslots) {
  __shared__ double red_loss[8];
  __shared__ float red[8][3];
  const int b = blockIdx.y;
  if constexpr (SP) ambient = __ldg(ambient_b + b);
  float pg[4] = {0.f, 0.f, 0.f, 0.f};                                 // SP: dL/d col (3), dL/d ambient
  const float l0 = __ldg(light_dir + 3 * b), l1 = __ldg(light_dir + 3 * b + 1), l2 = __ldg(light_dir + 3 * b + 2);
  const float col[3] = {__ldg(light_col + 3 * b), __ldg(light_col + 3 * b + 1), __ldg(light_col + 3 * b + 2)};
  const float inv_n = 2.f / (3.f * static_cast<float>(HW));          // d mean / d out, times the 2 of the square
  double lsum = 0.0;
  float dl[3] = {0.f, 0.f, 0.f};                                      // dL/dL (the normalised light)
  PhongTerms t;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;               // < HW for thread 0 of every block
  if (p < HW) {
    const size_t o = (static_cast<size_t>(b) * HW + p) * 3;
    const float r = img[o], g = img[o + 1], bl = img[o + 2];
    float out[3];
    phong_pixel(r, g, bl, l0, l1, l2, col, ambient, k_diffuse, white, with_mask, out, &t);
    float dndl = 0.f, dm = 0.f, dout[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float res = out[c] - target[o + c];
      if constexpr (SP) dout[c] = inv_n * res;
      lsum += static_cast<double>(res) * res;
      const float dx = (t.x[c] >= 0.f && t.x[c] <= 1.f) ? inv_n * res : 0.f;      // clip(compos, 0, 1)
      if (with_mask) dm += dx * (ambient + t.diff[c] - 1.f);
      const float ddiff = with_mask ? dx * t.mask : dx;
      const float dpre = (t.pre[c] >= 0.f && t.pre[c] <= 1.f) ? ddiff : 0.f;      // clip(diffuse, 0, 1)
      dndl += dpre * k_diffuse * col[c];
    }
    const float dd = t.d >= 0.f ? dndl : 0.f;                        // max(d, 0); false for the NaN of img = 0.5
    float di[3] = {0.f, 0.f, 0.f};
    if (dd != 0.f) {
      const float u[3] = {(r - 0.5f) * t.inv, (g - 0.5f) * t.inv, (bl - 0.5f) * t.inv};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        di[i] = dd * (t.L[i] - t.d * u[i]) * t.inv;
        dl[i] = dd * u[i];
      }
    }
    if (with_mask && dm != 0.f) {
      const double a[3] = {white ? 1.0 - r : static_cast<double>(r), white ? 1.0 - g : static_cast<double>(g),
                           white ? 1.0 - bl : static_cast<double>(bl)};
      const double nrm = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
      if (nrm > 0.0) {
        const double md = 1.0 / (1.0 + exp(-(255.0 * nrm - (white ? 80.0 : 150.0))));
        const double ds = static_cast<double>(dm) * md * (1.0 - md) * (white ? -255.0 : 255.0) / nrm;
#pragma unroll
        for (int i = 0; i < 3; ++i) di[i] += static_cast<float>(ds * a[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) d_img[o + i] = di[i];
    if constexpr (SP) phong_param_backward(t.d, t.mask, t.pre, t.x, k_diffuse, with_mask, dout, pg, pg + 3);
  }
  if constexpr (SP) {
    if (FX ? pslots != nullptr : (d_col != nullptr || d_amb != nullptr)) {
      block_sum4(pg);
      if (threadIdx.x == 0) store_param_grads<FX>(pg, b, d_col, d_amb, pslots);
    }
  }
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, off);
  if (lane == 0) red_loss[wib] = lsum;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float v = dl[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) red[wib][i] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    float v[3] = {0.f, 0.f, 0.f};
    for (int w = 0; w < 8; ++w) {
      s += red_loss[w];
      for (int i = 0; i < 3; ++i) v[i] += red[w][i];
    }
    if constexpr (FX) {
      double* sl = slots + (static_cast<size_t>(b) * gridDim.x + blockIdx.x) * 4;
      sl[0] = s / (3.0 * HW);
      const float ldv = t.L[0] * v[0] + t.L[1] * v[1] + t.L[2] * v[2];
      for (int i = 0; i < 3; ++i) sl[1 + i] = (v[i] - t.L[i] * ldv) * t.linv;
    } else {
      atomicAdd(loss + b, s / (3.0 * HW));
      if (d_light != nullptr) {                                        // d (l/|l|) = (dL - L (L.dL)) / |l|
        const float ldv = t.L[0] * v[0] + t.L[1] * v[1] + t.L[2] * v[2];
        for (int i = 0; i < 3; ++i) atomicAdd(d_light + 3 * b + i, (v[i] - t.L[i] * ldv) * t.linv);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ Phong composite, any loss
// The vector-Jacobian product of rn_phong_shade (phong_shade_kernel, rn_ops.cu) for an upstream gradient g = dL/d(compos):
//   compos_c = albedo_c shade_c (albedo NULL: compos = shade)  ->  d_albedo_c = g_c shade_c,  dL/d(shade_c) = g_c albedo_c
// and dL/d(shade) through the composite's own pixel function: tf_phong_pixel_backward (TF) or phong_pixel_backward (NumPy), each
// fed the terms its forward recorded in this thread, so the shading differentiated is rn_phong_shade's bit for bit.  dL/dL is
// reduced over the block and mapped through the forward's normalisation of the light: (I - L L^T) / |l| with the TF composite's
// division by |l|, or times the NumPy composite's reciprocal 1 / |l|; one atomic per block and component.  One thread per pixel,
// blockIdx.y = batch item.  FX: the block's three d_light terms go to slots[b][blockIdx.x][3] (summed by slot_sum_kernel).
// SP: as phong_recon_loss_grad_kernel's.
template <bool TF, bool FX, bool SP>
__global__ void __launch_bounds__(256) phong_shade_backward_kernel(const float* __restrict__ normal, const float* __restrict__ albedo,
                                                                   const float* __restrict__ light_dir,
                                                                   const float* __restrict__ light_col, float ambient,
                                                                   float k_diffuse, int white, int with_mask,
                                                                   const float* __restrict__ g_compos, float* __restrict__ d_normal,
                                                                   float* __restrict__ d_albedo, float* __restrict__ d_light, int HW,
                                                                   double* __restrict__ slots, const float* __restrict__ ambient_b,
                                                                   float* __restrict__ d_col, float* __restrict__ d_amb,
                                                                   double* __restrict__ pslots) {
  __shared__ float red[8][3];
  const int b = blockIdx.y;
  if constexpr (SP) ambient = __ldg(ambient_b + b);
  float pg[4] = {0.f, 0.f, 0.f, 0.f};                                 // SP: dL/d col (3), dL/d ambient
  const float l0 = __ldg(light_dir + 3 * b), l1 = __ldg(light_dir + 3 * b + 1), l2 = __ldg(light_dir + 3 * b + 2);
  const float col[3] = {__ldg(light_col + 3 * b), __ldg(light_col + 3 * b + 1), __ldg(light_col + 3 * b + 2)};
  float L[3], lscale;                                                 // the normalised light; 1/|l| (NumPy) or |l| (TF)
  if constexpr (TF) {
    lscale = sqrtf(l0 * l0 + l1 * l1 + l2 * l2);                      // as phong_shade_kernel normalises it
    L[0] = l0 / lscale; L[1] = l1 / lscale; L[2] = l2 / lscale;
  } else {
    lscale = 1.0f / sqrtf(l0 * l0 + l1 * l1 + l2 * l2);               // as phong_pixel normalises it
    L[0] = l0 * lscale; L[1] = l1 * lscale; L[2] = l2 * lscale;
  }
  float dl[3] = {0.f, 0.f, 0.f};
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < HW) {
    const size_t o = (static_cast<size_t>(b) * HW + p) * 3;
    const float n[3] = {normal[o], normal[o + 1], normal[o + 2]};
    float s[3], ds[3], dn[3];
    const float g[3] = {g_compos[o], g_compos[o + 1], g_compos[o + 2]};
    if constexpr (TF) {
      TfPhongTerms t;
      tf_phong_pixel(n[0], n[1], n[2], L, col, ambient, k_diffuse, !white, with_mask, s, &t);
      if (albedo != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) ds[c] = g[c] * albedo[o + c];
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) ds[c] = g[c];
      }
      tf_phong_pixel_backward(n, L, t, col, ambient, k_diffuse, !white, with_mask, ds, dn, dl);
      if constexpr (SP) phong_param_backward(t.d, t.m, t.pre, t.x, k_diffuse, with_mask, ds, pg, pg + 3);
    } else {
      PhongTerms t;
      phong_pixel(n[0], n[1], n[2], l0, l1, l2, col, ambient, k_diffuse, white, with_mask, s, &t);
      if (albedo != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) ds[c] = g[c] * albedo[o + c];
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) ds[c] = g[c];
      }
      phong_pixel_backward(n[0], n[1], n[2], t, col, ambient, k_diffuse, white, with_mask, ds, dn, dl);
      if constexpr (SP) phong_param_backward(t.d, t.mask, t.pre, t.x, k_diffuse, with_mask, ds, pg, pg + 3);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) d_normal[o + i] = dn[i];
    if (albedo != nullptr && d_albedo != nullptr) {
#pragma unroll
      for (int c = 0; c < 3; ++c) d_albedo[o + c] = g[c] * s[c];
    }
  }
  if constexpr (SP) {
    if (FX ? pslots != nullptr : (d_col != nullptr || d_amb != nullptr)) {
      block_sum4(pg);
      if (threadIdx.x == 0) store_param_grads<FX>(pg, b, d_col, d_amb, pslots);
    }
  }
  if (FX ? slots == nullptr : d_light == nullptr) return;             // the same in every thread: the barrier below stays whole
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float v = dl[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) red[wib][i] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float v[3] = {0.f, 0.f, 0.f};
    for (int w = 0; w < 8; ++w)
      for (int i = 0; i < 3; ++i) v[i] += red[w][i];
    const float ldv = L[0] * v[0] + L[1] * v[1] + L[2] * v[2];       // d (l/|l|) = (dL - L (L.dL)) / |l|
    for (int i = 0; i < 3; ++i) {
      const float dli = TF ? (v[i] - L[i] * ldv) / lscale : (v[i] - L[i] * ldv) * lscale;
      if constexpr (FX) slots[(static_cast<size_t>(b) * gridDim.x + blockIdx.x) * 3 + i] = dli;
      else atomicAdd(d_light + 3 * b + i, dli);
    }
  }
}

}  // namespace rn

using namespace rn;

extern "C" int rn_prelu_backward_16(const void* g, const void* y, const float* alpha, void* out, long long n, int C, int fmt,
                                    void* stream) {
  if (!g || !y || !alpha || !out || n < 0 || C < 1 || fmt < 0 || fmt > 2) return -1;
  if (n == 0) return 0;
  prelu_backward_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(g), static_cast<const uint16_t*>(y), alpha, static_cast<uint16_t*>(out), n, C, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_sigmoid_backward(const float* g, const float* img, void* out16, long long npix, int C, int Cpad, float scale,
                                   int fmt, void* stream) {
  if (!g || !img || !out16 || npix < 1 || C < 1 || Cpad < C || fmt < 0 || fmt > 2) return -1;
  sigmoid_backward_kernel<<<grid_for(npix * Cpad, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      g, img, static_cast<uint16_t*>(out16), npix, C, Cpad, scale, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_conv3d_backward_data_direct(const void* g16, const float* w, void* dx16, float* dx32, int B, int H, int W,
                                              int D, int Cin, int Cout, int k, int sy, int sx, int sz, float out_scale, int fmt,
                                              void* stream) {
  if (!g16 || !w || (!dx16 && !dx32) || B < 1 || fmt < 0 || fmt > 2) return -1;
  int Ho, Wo, Do, py, px, pz;
  same_pad(H, k, sy, &Ho, &py);
  same_pad(W, k, sx, &Wo, &px);
  same_pad(D, k, sz, &Do, &pz);
  const long long total = static_cast<long long>(B) * H * W * D;
  const long long blocks = (total + 255) / 256;
  if (blocks > 0x7fffffffLL) return -3;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint16_t* g = static_cast<const uint16_t*>(g16);
  uint16_t* d16 = static_cast<uint16_t*>(dx16);
#define RN_BWD(CI, CO, KK)                                                                                                   \
  conv3d_bwd_data_kernel<CI, CO, KK><<<static_cast<int>(blocks), 256, 0, st>>>(g, w, d16, dx32, B, H, W, D, Ho, Wo, Do, sy, \
                                                                                  sx, sz, py, px, pz, out_scale, fmt)
  if (Cin == 1 && Cout == 8 && k == 5) RN_BWD(1, 8, 5);
  else if (Cin == 5 && Cout == 8 && k == 5) RN_BWD(5, 8, 5);
  else if (Cin == 8 && Cout == 16 && k == 3) RN_BWD(8, 16, 3);
  else return -2;
#undef RN_BWD
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_resample_backward_f32(const float* vox, const float* minv, const float* gout, float* dvox, float* dminv, int B,
                                        int C, int size, int new_size, int transform, void* stream) {
  if (!vox || !minv || !gout || (!dvox && !dminv) || B < 1 || size < 2 || new_size < 1) return -1;
  if ((new_size * new_size) % 8 != 0) return -2;      // a block's 8 rows must belong to one batch item
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = static_cast<long long>(B) * new_size * new_size;
  const int grid = static_cast<int>((rows * 32 + 255) / 256);
  switch (C) {
    case 1:
      resample_backward_kernel<1, false><<<grid, 256, 0, st>>>(vox, minv, gout, dvox, dminv, B, size, new_size, transform, nullptr,
                                                               nullptr, 0, nullptr);
      break;
    case 4:
      resample_backward_kernel<4, false><<<grid, 256, 0, st>>>(vox, minv, gout, dvox, dminv, B, size, new_size, transform, nullptr,
                                                               nullptr, 0, nullptr);
      break;
    default: return -3;
  }
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

static int resample5_backward_launch(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox,
                                     float* dtex, float* dminv, int B, int size, int new_size, int y0, int x0, int ph, int pw,
                                     void* stream) {
  if ((reinterpret_cast<uintptr_t>(tex) & 15) != 0 || (reinterpret_cast<uintptr_t>(dtex) & 15) != 0) return -3;
  const long long rows = static_cast<long long>(B) * ph * pw;
  resample5_backward_kernel<false><<<static_cast<int>((rows * 32 + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      vox, tex, minv, gout, dvox, dtex, dminv, B, size, new_size, y0, x0, ph, pw, nullptr, nullptr, nullptr, 0, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_resample5_backward_f32(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox,
                                         float* dtex, float* dminv, int B, int size, int new_size, void* stream) {
  if (!vox || !tex || !minv || !gout || (!dvox && !dtex && !dminv) || B < 1 || size < 2 || new_size < 1) return -1;
  if ((new_size * new_size) % 8 != 0) return -2;      // a block's 8 rows must belong to one batch item
  return resample5_backward_launch(vox, tex, minv, gout, dvox, dtex, dminv, B, size, new_size, 0, 0, new_size, new_size, stream);
}

extern "C" int rn_resample5_backward_window_f32(const float* vox, const float* tex, const float* minv, const float* gout,
                                                float* dvox, float* dtex, float* dminv, int B, int size, int new_size, int y0,
                                                int x0, int ph, int pw, void* stream) {
  if (!vox || !tex || !minv || !gout || (!dvox && !dtex && !dminv) || B < 1 || size < 2 || new_size < 16) return -1;
  // same window rule as rn_ops.cu's window_ok; ph * pw % 8 == 0 keeps a block's 8 rows in one batch item
  if (ph < 16 || pw < 16 || ph % 16 != 0 || pw % 16 != 0 || y0 < 0 || x0 < 0 || y0 > new_size - ph || x0 > new_size - pw)
    return -2;
  return resample5_backward_launch(vox, tex, minv, gout, dvox, dtex, dminv, B, size, new_size, y0, x0, ph, pw, stream);
}

extern "C" int rn_prelu_backward_f32(const float* g, const float* z, const float* alpha, float* out, long long n, int C,
                                     void* stream) {
  if (!g || !z || !alpha || !out || n < 0 || C < 1) return -1;
  if (n == 0) return 0;
  prelu_backward_f32_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(g, z, alpha, out, n, C);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" long long rn_fully_connected_backward_workspace(int B, int K, int N) {
  if (B < 1 || K < 1 || N < 1) return -1;
  return static_cast<long long>((N + FCB_NC - 1) / FCB_NC) * B * K;
}

extern "C" int rn_fully_connected_backward_data(const float* g, const float* w, float* work, float* dx, int B, int K, int N,
                                                void* stream) {
  if (!g || !w || !work || !dx || B < 1 || K < 1 || N < 1) return -1;
  if (B > 32) return -2;
  if ((reinterpret_cast<uintptr_t>(w) & 15) != 0 || N % 4 != 0) return -3;   // float4 rows
  const int nchunks = (N + FCB_NC - 1) / FCB_NC;
  const int smem = B * FCB_NC * static_cast<int>(sizeof(float));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B <= 8) {
    fc_bwd_data_partial_kernel<8><<<nchunks, 256, smem, st>>>(g, w, work, B, K, N);
  } else {
    cudaError_t e = cudaFuncSetAttribute(fc_bwd_data_partial_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    fc_bwd_data_partial_kernel<32><<<nchunks, 256, smem, st>>>(g, w, work, B, K, N);
  }
  RN_COUNT_LAUNCH();
  fc_bwd_data_reduce_kernel<<<(B * K + 255) / 256, 256, 0, st>>>(work, dx, nchunks, B * K);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_phong_recon_loss_grad(const float* albedo, const float* normal, const float* target, const float* light_dir,
                                        const float* light_col, float ambient, float k_diffuse, int black_background,
                                        int with_mask, double* loss, float* d_albedo, float* d_normal, float* d_light_dir, int B,
                                        int H, int W, void* stream) {
  if (!albedo || !normal || !target || !light_dir || !light_col || !loss || !d_albedo || !d_normal || B < 1 || H < 1 || W < 1)
    return -1;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  phong_recon_loss_grad_kernel<false, false><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      albedo, normal, target, light_dir, light_col, ambient, k_diffuse, black_background, with_mask, loss, d_albedo, d_normal,
      d_light_dir, HW, nullptr, nullptr, nullptr, nullptr, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_phong_composite_loss_grad(const float* img, const float* target, const float* light_dir, const float* light_col,
                                            float ambient, float k_diffuse, int background_white, int with_mask, double* loss,
                                            float* d_img, float* d_light_dir, int B, int H, int W, void* stream) {
  if (!img || !target || !light_dir || !light_col || !loss || !d_img || B < 1 || H < 1 || W < 1) return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 256 || B > 65535) return -2;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  phong_composite_loss_grad_kernel<false, false><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      img, target, light_dir, light_col, ambient, k_diffuse, background_white, with_mask, loss, d_img, d_light_dir, HW, nullptr,
      nullptr, nullptr, nullptr, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_phong_shade_backward(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                                       float ambient, float k_diffuse, int composite, int background_white, int with_mask,
                                       const float* g_compos, float* d_normal, float* d_albedo, float* d_light_dir, int B, int H,
                                       int W, void* stream) {
  if (!normal || !light_dir || !light_col || !g_compos || !d_normal || B < 1 || H < 1 || W < 1) return -1;
  if (composite != RN_PHONG_NUMPY && composite != RN_PHONG_TF) return -1;
  if (B > 65535 || static_cast<long long>(H) * W > 0x7fffffffLL - 255) return -2;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  const int white = background_white != 0, mask = with_mask != 0;
  if (composite == RN_PHONG_TF)
    phong_shade_backward_kernel<true, false, false><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        normal, albedo, light_dir, light_col, ambient, k_diffuse, white, mask, g_compos, d_normal, d_albedo, d_light_dir, HW,
        nullptr, nullptr, nullptr, nullptr, nullptr);
  else
    phong_shade_backward_kernel<false, false, false><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        normal, albedo, light_dir, light_col, ambient, k_diffuse, white, mask, g_compos, d_normal, d_albedo, d_light_dir, HW,
        nullptr, nullptr, nullptr, nullptr, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------ fixed-order twins (entry points)
namespace rn {
// the second stage of every twin (also launched by rn_train.cu's rn_image_loss_grad_items_fixed)
int launch_slot_sum(const double* part, int B, int nblk, int width, int nd, double* out_d, float* out_f, const unsigned* amax,
                    int namax, cudaStream_t st) {
  const long long threads = static_cast<long long>(B) * width * 32;
  slot_sum_kernel<<<static_cast<int>((threads + 255) / 256), 256, 0, st>>>(part, B, nblk, width, nd, out_d, out_f, amax, namax);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}
}  // namespace rn

namespace {
int lg_points(int new_size) {                                          // smallest L with 2^L >= new_size^3
  const long long n = static_cast<long long>(new_size) * new_size * new_size;
  int L = 0;
  while ((1LL << L) < n) ++L;
  return L;
}
long long up8(long long bytes) { return (bytes + 7) / 8 * 8; }
// workspace of the resampler twins: [acc int64 B*size^3*nacc][slots double B*(new^2/8)*12][amax uint32 B*C]
long long resample_fixed_bytes(int B, int C, int size, int new_size, int nacc) {
  const long long vol = static_cast<long long>(size) * size * size;
  return 8LL * B * vol * nacc + 8LL * B * (static_cast<long long>(new_size) * new_size / 8) * 12 + up8(4LL * B * C);
}
int resample_fixed_check(const float* vox, const float* minv, const float* gout, int B, int size, int new_size) {
  if (!vox || !minv || !gout || B < 1 || size < 2 || new_size < 1) return -1;
  if ((new_size * new_size) % 8 != 0) return -2;                       // a block's 8 rows must belong to one batch item
  if (new_size > 1024 || size > 1024) return -2;                       // new_size^3 < 2^31 sample points, 2^L fits int64
  return 0;
}
int grid_items(long long per_item) {                                   // blocks per item of the twins' elementwise stages
  return grid_for(per_item, 256 * 4, 132 * 4);
}
}  // namespace

extern "C" int rn_fixed_point_exponent(float max_abs, int new_size) {
  if (new_size < 1 || new_size > 1024) return -1000;
  return fx_exponent(max_abs, lg_points(new_size));
}

extern "C" long long rn_resample_backward_fixed_workspace(int B, int C, int size, int new_size, int want_dvox) {
  if (B < 1 || (C != 1 && C != 4) || size < 2 || new_size < 1) return -1;
  return resample_fixed_bytes(B, C, size, new_size, want_dvox ? C : 0);
}

extern "C" int rn_resample_backward_fixed_f32(const float* vox, const float* minv, const float* gout, float* dvox, float* dminv,
                                              int B, int C, int size, int new_size, int transform, void* work, long long work_bytes,
                                              void* stream) {
  if (int rc = resample_fixed_check(vox, minv, gout, B, size, new_size)) return rc;
  if (!dvox && !dminv) return -1;
  if (C != 1 && C != 4) return -3;
  if (!work || work_bytes < resample_fixed_bytes(B, C, size, new_size, dvox ? C : 0)) return -4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long vol = static_cast<long long>(size) * size * size, nbpi = static_cast<long long>(new_size) * new_size / 8;
  unsigned long long* acc = dvox ? static_cast<unsigned long long*>(work) : nullptr;
  double* slots = reinterpret_cast<double*>(static_cast<char*>(work) + 8LL * B * vol * (dvox ? C : 0));
  unsigned* amax = reinterpret_cast<unsigned*>(slots + B * nbpi * 12);
  const int L = lg_points(new_size);
  cudaError_t e = cudaMemsetAsync(amax, 0, 4ULL * B * C, st);
  if (e == cudaSuccess && acc) e = cudaMemsetAsync(acc, 0, 8ULL * B * vol * C, st);
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long points = static_cast<long long>(new_size) * new_size * new_size;
  const dim3 mgrid(grid_items(points), B);
  const int grid = static_cast<int>(B * nbpi);
  double* sl = dminv ? slots : nullptr;
  if (C == 1) {
    absmax_bits_kernel<1><<<mgrid, 256, 0, st>>>(gout, amax, points);
    resample_backward_kernel<1, true><<<grid, 256, 0, st>>>(vox, minv, gout, nullptr, nullptr, B, size, new_size, transform, acc,
                                                            amax, L, sl);
  } else {
    absmax_bits_kernel<4><<<mgrid, 256, 0, st>>>(gout, amax, points);
    resample_backward_kernel<4, true><<<grid, 256, 0, st>>>(vox, minv, gout, nullptr, nullptr, B, size, new_size, transform, acc,
                                                            amax, L, sl);
  }
  RN_COUNT_LAUNCH();
  RN_COUNT_LAUNCH();
  if (dvox) {
    fx_finalize_kernel<<<dim3(grid_items(vol * C), B), 256, 0, st>>>(acc, amax, C, 0, L, dvox, vol * C, C);
    RN_COUNT_LAUNCH();
  }
  if (dminv) return launch_slot_sum(slots, B, static_cast<int>(nbpi), 12, 0, nullptr, dminv, amax, C, st);
  return static_cast<int>(cudaGetLastError());
}

extern "C" long long rn_resample5_backward_fixed_workspace(int B, int size, int new_size, int want_dvox, int want_dtex) {
  if (B < 1 || size < 2 || new_size < 1) return -1;
  return resample_fixed_bytes(B, 5, size, new_size, (want_dvox ? 1 : 0) + (want_dtex ? 4 : 0));
}

extern "C" int rn_resample5_backward_fixed_f32(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox,
                                               float* dtex, float* dminv, int B, int size, int new_size, void* work,
                                               long long work_bytes, void* stream) {
  if (int rc = resample_fixed_check(vox, minv, gout, B, size, new_size)) return rc;
  if (!tex || (!dvox && !dtex && !dminv)) return -1;
  if ((reinterpret_cast<uintptr_t>(tex) & 15) != 0) return -3;
  const int nacc = (dvox ? 1 : 0) + (dtex ? 4 : 0);
  if (!work || work_bytes < resample_fixed_bytes(B, 5, size, new_size, nacc)) return -4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long vol = static_cast<long long>(size) * size * size, nbpi = static_cast<long long>(new_size) * new_size / 8;
  unsigned long long* acc_vox = dvox ? static_cast<unsigned long long*>(work) : nullptr;
  unsigned long long* acc_tex = dtex ? static_cast<unsigned long long*>(work) + (dvox ? B * vol : 0) : nullptr;
  double* slots = reinterpret_cast<double*>(static_cast<char*>(work) + 8LL * B * vol * nacc);
  unsigned* amax = reinterpret_cast<unsigned*>(slots + B * nbpi * 12);
  const int L = lg_points(new_size);
  cudaError_t e = cudaMemsetAsync(amax, 0, 4ULL * B * 5, st);
  if (e == cudaSuccess && nacc) e = cudaMemsetAsync(work, 0, 8ULL * B * vol * nacc, st);
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long points = static_cast<long long>(new_size) * new_size * new_size;
  absmax_bits_kernel<5><<<dim3(grid_items(points), B), 256, 0, st>>>(gout, amax, points);
  RN_COUNT_LAUNCH();
  resample5_backward_kernel<true><<<static_cast<int>(B * nbpi), 256, 0, st>>>(
      vox, tex, minv, gout, nullptr, nullptr, nullptr, B, size, new_size, 0, 0, new_size, new_size, acc_vox, acc_tex, amax, L,
      dminv ? slots : nullptr);
  RN_COUNT_LAUNCH();
  if (dvox) {
    fx_finalize_kernel<<<dim3(grid_items(vol), B), 256, 0, st>>>(acc_vox, amax, 5, 0, L, dvox, vol, 1);
    RN_COUNT_LAUNCH();
  }
  if (dtex) {
    fx_finalize_kernel<<<dim3(grid_items(vol * 4), B), 256, 0, st>>>(acc_tex, amax, 5, 1, L, dtex, vol * 4, 4);
    RN_COUNT_LAUNCH();
  }
  if (dminv) return launch_slot_sum(slots, B, static_cast<int>(nbpi), 12, 0, nullptr, dminv, amax, 5, st);
  return static_cast<int>(cudaGetLastError());
}

// the three Phong twins: one slot row of 4 doubles per (item, 256-pixel block)
extern "C" long long rn_phong_recon_loss_grad_fixed_workspace(int B, int H, int W) {
  if (B < 1 || H < 1 || W < 1) return -1;
  return 8LL * B * ((static_cast<long long>(H) * W + 255) / 256) * 4;
}
extern "C" long long rn_phong_composite_loss_grad_fixed_workspace(int B, int H, int W) {
  return rn_phong_recon_loss_grad_fixed_workspace(B, H, W);
}
extern "C" long long rn_phong_shade_backward_fixed_workspace(int B, int H, int W) {
  return rn_phong_recon_loss_grad_fixed_workspace(B, H, W);
}

extern "C" int rn_phong_recon_loss_grad_fixed(const float* albedo, const float* normal, const float* target, const float* light_dir,
                                              const float* light_col, float ambient, float k_diffuse, int black_background,
                                              int with_mask, double* loss, float* d_albedo, float* d_normal, float* d_light_dir,
                                              int B, int H, int W, void* work, long long work_bytes, void* stream) {
  if (!albedo || !normal || !target || !light_dir || !light_col || !loss || !d_albedo || !d_normal || B < 1 || H < 1 || W < 1)
    return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 255 || B > 65535) return -2;
  if (!work || work_bytes < rn_phong_recon_loss_grad_fixed_workspace(B, H, W)) return -4;
  const int HW = H * W, nblk = (HW + 255) / 256;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  phong_recon_loss_grad_kernel<true, false><<<dim3(nblk, B), 256, 0, st>>>(
      albedo, normal, target, light_dir, light_col, ambient, k_diffuse, black_background, with_mask, nullptr, d_albedo, d_normal,
      nullptr, HW, static_cast<double*>(work), nullptr, nullptr, nullptr, nullptr);
  RN_COUNT_LAUNCH();
  return launch_slot_sum(static_cast<double*>(work), B, nblk, 4, 1, loss, d_light_dir, nullptr, 0, st);
}

extern "C" int rn_phong_composite_loss_grad_fixed(const float* img, const float* target, const float* light_dir,
                                                  const float* light_col, float ambient, float k_diffuse, int background_white,
                                                  int with_mask, double* loss, float* d_img, float* d_light_dir, int B, int H, int W,
                                                  void* work, long long work_bytes, void* stream) {
  if (!img || !target || !light_dir || !light_col || !loss || !d_img || B < 1 || H < 1 || W < 1) return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 256 || B > 65535) return -2;
  if (!work || work_bytes < rn_phong_composite_loss_grad_fixed_workspace(B, H, W)) return -4;
  const int HW = H * W, nblk = (HW + 255) / 256;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  phong_composite_loss_grad_kernel<true, false><<<dim3(nblk, B), 256, 0, st>>>(
      img, target, light_dir, light_col, ambient, k_diffuse, background_white, with_mask, nullptr, d_img, nullptr, HW,
      static_cast<double*>(work), nullptr, nullptr, nullptr, nullptr);
  RN_COUNT_LAUNCH();
  return launch_slot_sum(static_cast<double*>(work), B, nblk, 4, 1, loss, d_light_dir, nullptr, 0, st);
}

extern "C" int rn_phong_shade_backward_fixed(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                                             float ambient, float k_diffuse, int composite, int background_white, int with_mask,
                                             const float* g_compos, float* d_normal, float* d_albedo, float* d_light_dir, int B,
                                             int H, int W, void* work, long long work_bytes, void* stream) {
  if (!normal || !light_dir || !light_col || !g_compos || !d_normal || B < 1 || H < 1 || W < 1) return -1;
  if (composite != RN_PHONG_NUMPY && composite != RN_PHONG_TF) return -1;
  if (B > 65535 || static_cast<long long>(H) * W > 0x7fffffffLL - 255) return -2;
  if (d_light_dir && (!work || work_bytes < rn_phong_shade_backward_fixed_workspace(B, H, W))) return -4;
  const int HW = H * W, nblk = (HW + 255) / 256;
  const dim3 grid(nblk, B);
  const int white = background_white != 0, mask = with_mask != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* slots = d_light_dir ? static_cast<double*>(work) : nullptr;
  if (composite == RN_PHONG_TF)
    phong_shade_backward_kernel<true, true, false><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, ambient, k_diffuse,
                                                                         white, mask, g_compos, d_normal, d_albedo, nullptr, HW, slots,
                                                                         nullptr, nullptr, nullptr, nullptr);
  else
    phong_shade_backward_kernel<false, true, false><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, ambient, k_diffuse,
                                                                          white, mask, g_compos, d_normal, d_albedo, nullptr, HW,
                                                                          slots, nullptr, nullptr, nullptr, nullptr);
  RN_COUNT_LAUNCH();
  if (d_light_dir) return launch_slot_sum(slots, B, nblk, 3, 0, nullptr, d_light_dir, nullptr, 0, st);
  return static_cast<int>(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------ shading-parameter entries
// The SP instantiations: each is its scalar-ambient entry with ambient read per item from a device array [B] and the
// gradients of light_col [B,3] and ambient [B] (either may be NULL).  The atomic entries accumulate into them (zero them
// first); the twins overwrite them.  Twin workspace: slots of 4 doubles per (item, 256-pixel block) for the loss and d_light_dir
// terms, then 3 for the colour and 1 for the ambient term.
namespace {
long long phong_params_fixed_bytes(int B, int H, int W) {
  if (B < 1 || H < 1 || W < 1) return -1;
  return 8LL * B * ((static_cast<long long>(H) * W + 255) / 256) * 8;
}
// the colour and ambient sums of a twin (pslots = work + 4 B nblk doubles)
int param_slot_sums(const double* pslots, int B, int nblk, float* d_col, float* d_amb, cudaStream_t st) {
  int rc = 0;
  if (d_col) rc = launch_slot_sum(pslots, B, nblk, 3, 0, nullptr, d_col, nullptr, 0, st);
  if (rc == 0 && d_amb) rc = launch_slot_sum(pslots + 3LL * B * nblk, B, nblk, 1, 0, nullptr, d_amb, nullptr, 0, st);
  return rc;
}
}  // namespace

extern "C" int rn_phong_recon_loss_grad_params(const float* albedo, const float* normal, const float* target,
                                               const float* light_dir, const float* light_col, const float* ambient,
                                               float k_diffuse, int black_background, int with_mask, double* loss,
                                               float* d_albedo, float* d_normal, float* d_light_dir, float* d_light_col,
                                               float* d_ambient, int B, int H, int W, void* stream) {
  if (!albedo || !normal || !target || !light_dir || !light_col || !ambient || !loss || !d_albedo || !d_normal || B < 1 || H < 1 ||
      W < 1)
    return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 255 || B > 65535) return -2;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  phong_recon_loss_grad_kernel<false, true><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      albedo, normal, target, light_dir, light_col, 0.f, k_diffuse, black_background, with_mask, loss, d_albedo, d_normal,
      d_light_dir, HW, nullptr, ambient, d_light_col, d_ambient, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_phong_composite_loss_grad_params(const float* img, const float* target, const float* light_dir,
                                                   const float* light_col, const float* ambient, float k_diffuse,
                                                   int background_white, int with_mask, double* loss, float* d_img,
                                                   float* d_light_dir, float* d_light_col, float* d_ambient, int B, int H, int W,
                                                   void* stream) {
  if (!img || !target || !light_dir || !light_col || !ambient || !loss || !d_img || B < 1 || H < 1 || W < 1) return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 256 || B > 65535) return -2;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  phong_composite_loss_grad_kernel<false, true><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      img, target, light_dir, light_col, 0.f, k_diffuse, background_white, with_mask, loss, d_img, d_light_dir, HW, nullptr,
      ambient, d_light_col, d_ambient, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_phong_shade_backward_params(const float* normal, const float* albedo, const float* light_dir,
                                              const float* light_col, const float* ambient, float k_diffuse, int composite,
                                              int background_white, int with_mask, const float* g_compos, float* d_normal,
                                              float* d_albedo, float* d_light_dir, float* d_light_col, float* d_ambient, int B,
                                              int H, int W, void* stream) {
  if (!normal || !light_dir || !light_col || !ambient || !g_compos || !d_normal || B < 1 || H < 1 || W < 1) return -1;
  if (composite != RN_PHONG_NUMPY && composite != RN_PHONG_TF) return -1;
  if (B > 65535 || static_cast<long long>(H) * W > 0x7fffffffLL - 255) return -2;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  const int white = background_white != 0, mask = with_mask != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (composite == RN_PHONG_TF)
    phong_shade_backward_kernel<true, false, true><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, 0.f, k_diffuse,
                                                                         white, mask, g_compos, d_normal, d_albedo, d_light_dir,
                                                                         HW, nullptr, ambient, d_light_col, d_ambient, nullptr);
  else
    phong_shade_backward_kernel<false, false, true><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, 0.f, k_diffuse,
                                                                          white, mask, g_compos, d_normal, d_albedo, d_light_dir,
                                                                          HW, nullptr, ambient, d_light_col, d_ambient, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" long long rn_phong_recon_loss_grad_params_fixed_workspace(int B, int H, int W) {
  return phong_params_fixed_bytes(B, H, W);
}
extern "C" long long rn_phong_composite_loss_grad_params_fixed_workspace(int B, int H, int W) {
  return phong_params_fixed_bytes(B, H, W);
}
extern "C" long long rn_phong_shade_backward_params_fixed_workspace(int B, int H, int W) {
  return phong_params_fixed_bytes(B, H, W);
}

extern "C" int rn_phong_recon_loss_grad_params_fixed(const float* albedo, const float* normal, const float* target,
                                                     const float* light_dir, const float* light_col, const float* ambient,
                                                     float k_diffuse, int black_background, int with_mask, double* loss,
                                                     float* d_albedo, float* d_normal, float* d_light_dir, float* d_light_col,
                                                     float* d_ambient, int B, int H, int W, void* work, long long work_bytes,
                                                     void* stream) {
  if (!albedo || !normal || !target || !light_dir || !light_col || !ambient || !loss || !d_albedo || !d_normal || B < 1 || H < 1 ||
      W < 1)
    return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 255 || B > 65535) return -2;
  if (!work || work_bytes < phong_params_fixed_bytes(B, H, W)) return -4;
  const int HW = H * W, nblk = (HW + 255) / 256;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* slots = static_cast<double*>(work);
  double* pslots = (d_light_col || d_ambient) ? slots + 4LL * B * nblk : nullptr;
  phong_recon_loss_grad_kernel<true, true><<<dim3(nblk, B), 256, 0, st>>>(
      albedo, normal, target, light_dir, light_col, 0.f, k_diffuse, black_background, with_mask, nullptr, d_albedo, d_normal,
      nullptr, HW, slots, ambient, nullptr, nullptr, pslots);
  RN_COUNT_LAUNCH();
  int rc = launch_slot_sum(slots, B, nblk, 4, 1, loss, d_light_dir, nullptr, 0, st);
  return rc ? rc : param_slot_sums(pslots, B, nblk, d_light_col, d_ambient, st);
}

extern "C" int rn_phong_composite_loss_grad_params_fixed(const float* img, const float* target, const float* light_dir,
                                                         const float* light_col, const float* ambient, float k_diffuse,
                                                         int background_white, int with_mask, double* loss, float* d_img,
                                                         float* d_light_dir, float* d_light_col, float* d_ambient, int B, int H,
                                                         int W, void* work, long long work_bytes, void* stream) {
  if (!img || !target || !light_dir || !light_col || !ambient || !loss || !d_img || B < 1 || H < 1 || W < 1) return -1;
  if (static_cast<long long>(H) * W > 0x7fffffffLL - 256 || B > 65535) return -2;
  if (!work || work_bytes < phong_params_fixed_bytes(B, H, W)) return -4;
  const int HW = H * W, nblk = (HW + 255) / 256;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* slots = static_cast<double*>(work);
  double* pslots = (d_light_col || d_ambient) ? slots + 4LL * B * nblk : nullptr;
  phong_composite_loss_grad_kernel<true, true><<<dim3(nblk, B), 256, 0, st>>>(
      img, target, light_dir, light_col, 0.f, k_diffuse, background_white, with_mask, nullptr, d_img, nullptr, HW, slots, ambient,
      nullptr, nullptr, pslots);
  RN_COUNT_LAUNCH();
  int rc = launch_slot_sum(slots, B, nblk, 4, 1, loss, d_light_dir, nullptr, 0, st);
  return rc ? rc : param_slot_sums(pslots, B, nblk, d_light_col, d_ambient, st);
}

extern "C" int rn_phong_shade_backward_params_fixed(const float* normal, const float* albedo, const float* light_dir,
                                                    const float* light_col, const float* ambient, float k_diffuse, int composite,
                                                    int background_white, int with_mask, const float* g_compos, float* d_normal,
                                                    float* d_albedo, float* d_light_dir, float* d_light_col, float* d_ambient,
                                                    int B, int H, int W, void* work, long long work_bytes, void* stream) {
  if (!normal || !light_dir || !light_col || !ambient || !g_compos || !d_normal || B < 1 || H < 1 || W < 1) return -1;
  if (composite != RN_PHONG_NUMPY && composite != RN_PHONG_TF) return -1;
  if (B > 65535 || static_cast<long long>(H) * W > 0x7fffffffLL - 255) return -2;
  const bool any = d_light_dir || d_light_col || d_ambient;
  if (any && (!work || work_bytes < phong_params_fixed_bytes(B, H, W))) return -4;
  const int HW = H * W, nblk = (HW + 255) / 256;
  const dim3 grid(nblk, B);
  const int white = background_white != 0, mask = with_mask != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* slots = d_light_dir ? static_cast<double*>(work) : nullptr;
  double* pslots = (d_light_col || d_ambient) ? static_cast<double*>(work) + 4LL * B * nblk : nullptr;
  if (composite == RN_PHONG_TF)
    phong_shade_backward_kernel<true, true, true><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, 0.f, k_diffuse, white,
                                                                        mask, g_compos, d_normal, d_albedo, nullptr, HW, slots,
                                                                        ambient, nullptr, nullptr, pslots);
  else
    phong_shade_backward_kernel<false, true, true><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, 0.f, k_diffuse,
                                                                         white, mask, g_compos, d_normal, d_albedo, nullptr, HW,
                                                                         slots, ambient, nullptr, nullptr, pslots);
  RN_COUNT_LAUNCH();
  int rc = d_light_dir ? launch_slot_sum(slots, B, nblk, 3, 0, nullptr, d_light_dir, nullptr, 0, st) : 0;
  rc = rc ? rc : param_slot_sums(pslots, B, nblk, d_light_col, d_ambient, st);
  return rc ? rc : static_cast<int>(cudaGetLastError());
}
