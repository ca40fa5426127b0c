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
//     decoder's fp32 PReLU and fully_connected data gradients (RenderNet_Texture_Face_Normal.py:34-46).
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>

#include "../../include/rendernet_b200.h"

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

// ------------------------------------------------------------------------------------------ resampler backward
// Forward (rn_resample_f32, transform = 1): N[b,p,q,r,c] = sum_corners w_k(x,y,z) V[b, corner_k, c] with
// (x,y,z) = Minv[b] . (r, new-1-p, q, 1), zero outside [0, size-1)^3.  Given G = dL/dN:
//   dL/dV[b, corner_k, c] += w_k G[b,p,q,r,c]                                                        (scatter-add)
//   dL/dMinv[b][a][j]     += sum_c G * (dN/d coord_a) * (r, new-1-p, q, 1)[j],   dN/dx = sum_k (dw_k/dx) V[corner_k], ...
// The floor() inside the weights is piecewise constant, so the derivative is the one of the trilinear patch the point
// lies in (what tf.gradients produces for tools/resampling_voxel_grid.py:465-485).  One warp per output row; the 12 matrix
// partial sums are reduced in the warp, then in the block, then one atomicAdd per block and entry.
template <int C>
__global__ void __launch_bounds__(256) resample_backward_kernel(const float* __restrict__ vox, const float* __restrict__ minv,
                                                                const float* __restrict__ gout, float* __restrict__ dvox,
                                                                float* __restrict__ dminv, int B, int size, int nsz,
                                                                int transform) {
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
        if (dvb != nullptr) {
          atomicAdd(dvb + i000 + c, ax * ay * az * gv);
          atomicAdd(dvb + i000 + sy + c, ax * by * az * gv);
          atomicAdd(dvb + i000 + C + c, bx * ay * az * gv);
          atomicAdd(dvb + i000 + sy + C + c, bx * by * az * gv);
          atomicAdd(dvb + i000 + sz + c, ax * ay * bz * gv);
          atomicAdd(dvb + i000 + sz + sy + c, ax * by * bz * gv);
          atomicAdd(dvb + i000 + sz + C + c, bx * ay * bz * gv);
          atomicAdd(dvb + i000 + sz + sy + C + c, bx * by * bz * gv);
        }
      }
      dm[0] += dvx * gx; dm[1] += dvx * gy; dm[2] += dvx * gz; dm[3] += dvx;
      dm[4] += dvy * gx; dm[5] += dvy * gy; dm[6] += dvy * gz; dm[7] += dvy;
      dm[8] += dvz * gx; dm[9] += dvz * gy; dm[10] += dvz * gz; dm[11] += dvz;
    }
  }
  if (dminv == nullptr) return;
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
    if (first_row < rows && v != 0.f) atomicAdd(dminv + (first_row / (nsz * nsz)) * 12 + threadIdx.x, v);
  }
}

// Texture net input chain (resample5_conv1_kernel in rn_ops.cu; RenderNet_Texture_Face_Normal.py:155-179 and
// Reconstruct_RenderNet_Face.py:367-378): the geometry grid (C = 1) and the texture volume (C = 4) are sampled at the SAME
// points and concatenated, G = dL/d(concat) [B,N,N,N,5].  Each sample coordinate is computed once, with the forward kernel's
// sample_coord arithmetic and in/out test; channel 0 scatters into dvox, channels 1..4 into dtex (float4 corner gathers), and
// dM^-1 collects all five channels.  Per corner the five channels are first contracted to s_k = G0 V_k + G1..4 . T_k, so
// d/dx = sum_k (dw_k/dx) s_k.  Same warp-per-row layout and block reduction as resample_backward_kernel.
__global__ void __launch_bounds__(256) resample5_backward_kernel(const float* __restrict__ vox, const float* __restrict__ tex,
                                                                 const float* __restrict__ minv, const float* __restrict__ gout,
                                                                 float* __restrict__ dvox, float* __restrict__ dtex,
                                                                 float* __restrict__ dminv, int B, int size, int nsz) {
  __shared__ float red[8][12];
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int rows = B * nsz * nsz;
  float dm[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) dm[i] = 0.f;
  if (warp_global < rows) {
    const int b = warp_global / (nsz * nsz);
    const int o1 = (warp_global / nsz) % nsz;
    const int o2 = warp_global % nsz;
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
        if (dvb != nullptr && g0 != 0.f) atomicAdd(dvb + off[k], wk[k] * g0);
        if (dtb != nullptr) {
          float* d = dtb + off[k] * 4;
          atomicAdd(d + 0, wk[k] * g1); atomicAdd(d + 1, wk[k] * g2);
          atomicAdd(d + 2, wk[k] * g3); atomicAdd(d + 3, wk[k] * g4);
        }
      }
      dm[0] += dvx * gx; dm[1] += dvx * gy; dm[2] += dvx * gz; dm[3] += dvx;
      dm[4] += dvy * gx; dm[5] += dvy * gy; dm[6] += dvy * gz; dm[7] += dvy;
      dm[8] += dvz * gx; dm[9] += dvz * gy; dm[10] += dvz * gz; dm[11] += dvz;
    }
  }
  if (dminv == nullptr) return;
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
    if (first_row < rows && v != 0.f) atomicAdd(dminv + (first_row / (nsz * nsz)) * 12 + threadIdx.x, v);
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

// ------------------------------------------------------------------------------------------ face reconstruction objective
// Reconstruct_RenderNet_Face.py:372-383 over TensorFlow's Phong composite (tools/Phong_shading.py:24-113 tf_mask /
// tf_mask_white / tf_phong_shading / tf_phong_composite -- NOT the NumPy composite of phong_pixel):
//   L = l / |l|;  u = (n - 0.5) / |n - 0.5|;  dif_c = clip(k_d * max(u.L, 0) * col_c, 0, 1)
//   m = sigmoid(255 |n| - 80) (black background) or sigmoid(255 (sqrt 3 - |n|) - 80) (white)
//   shade_c = clip(m (ambient + dif_c) + 1 - m, 0, 1)   (with_mask; else clip(ambient + dif_c, 0, 1))
//   loss[b] = mean_{h,w,c} (target - albedo_c shade_c)^2
// and its gradient, in one pass, with TF-1's gradient conventions: tf.maximum(x, y) passes to x where x >= y;
// clip_by_value(x, lo, hi) passes where lo <= x <= hi; d|x|/dx = x/|x|.  One thread per pixel; blockIdx.y = batch item.  loss
// is accumulated in double (one atomic per block); dL/dL is reduced over the block and mapped through the normalisation
// (I - L L^T) / |l| before one atomic per block and component.
__global__ void __launch_bounds__(256) phong_recon_loss_grad_kernel(const float* __restrict__ albedo, const float* __restrict__ normal,
                                                                    const float* __restrict__ target, const float* __restrict__ light_dir,
                                                                    const float* __restrict__ light_col, float ambient, float k_diffuse,
                                                                    int black, int with_mask, double* __restrict__ loss,
                                                                    float* __restrict__ d_albedo, float* __restrict__ d_normal,
                                                                    float* __restrict__ d_light, int HW) {
  __shared__ float red[8][4];
  const int b = blockIdx.y;
  const float l0 = __ldg(light_dir + 3 * b), l1 = __ldg(light_dir + 3 * b + 1), l2 = __ldg(light_dir + 3 * b + 2);
  const float lnorm = sqrtf(l0 * l0 + l1 * l1 + l2 * l2);
  const float L[3] = {l0 / lnorm, l1 / lnorm, l2 / lnorm};
  const float col[3] = {__ldg(light_col + 3 * b), __ldg(light_col + 3 * b + 1), __ldg(light_col + 3 * b + 2)};
  const float inv_n = 2.f / (3.f * static_cast<float>(HW));          // d mean / d pred, times the 2 of the square
  float part[4] = {0.f, 0.f, 0.f, 0.f};                                // loss, dL/dL (3)
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < HW) {
    const size_t o = (static_cast<size_t>(b) * HW + p) * 3;
    const float n[3] = {normal[o], normal[o + 1], normal[o + 2]};
    const float v[3] = {n[0] - 0.5f, n[1] - 0.5f, n[2] - 0.5f};
    const float vn = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float u[3] = {v[0] / vn, v[1] / vn, v[2] / vn};
    const float d = u[0] * L[0] + u[1] * L[1] + u[2] * L[2];
    const float dmax = fmaxf(d, 0.f);
    // The mask's argument 255 |n| - 80 multiplies |n|'s rounding by 255 and its derivative by another 255: evaluated in fp32 it
    // alone moves the shading by ~1e-5.  It is a handful of operations per pixel, so it runs in double.
    float m = 1.f;
    double md = 1.0, nnd = 1.0;
    if (with_mask) {
      nnd = sqrt(static_cast<double>(n[0]) * n[0] + static_cast<double>(n[1]) * n[1] + static_cast<double>(n[2]) * n[2]);
      const double s = black ? 255.0 * nnd - 80.0 : 255.0 * (1.7320508075688772 - nnd) - 80.0;
      md = 1.0 / (1.0 + exp(-s));
      m = static_cast<float>(md);
    }
    float ddmax = 0.f, dm = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float pre = k_diffuse * dmax * col[c];
      const float dif = fminf(fmaxf(pre, 0.f), 1.f);
      const float x = with_mask ? m * (ambient + dif) + (1.f - m) : ambient + dif;
      const float shade = fminf(fmaxf(x, 0.f), 1.f);
      const float a = albedo[o + c];
      const float r = a * shade - target[o + c];
      part[0] += r * r;
      const float dpred = inv_n * r;
      d_albedo[o + c] = dpred * shade;
      const float dx = (x >= 0.f && x <= 1.f) ? dpred * a : 0.f;          // clip_by_value(compos, 0, 1)
      const float ddif = with_mask ? dx * m : dx;
      if (with_mask) dm += dx * (ambient + dif - 1.f);
      const float dpre = (pre >= 0.f && pre <= 1.f) ? ddif : 0.f;         // clip_by_value(diffuse, 0, 1)
      ddmax += dpre * k_diffuse * col[c];
    }
    const float dd = d >= 0.f ? ddmax : 0.f;                              // tf.maximum(d, 0): passes where d >= 0
    float du[3], dn[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      du[i] = dd * L[i];
      part[1 + i] += dd * u[i];
    }
    const float udu = u[0] * du[0] + u[1] * du[1] + u[2] * du[2];       // d (v/|v|) = (du - u (u.du)) / |v|
#pragma unroll
    for (int i = 0; i < 3; ++i) dn[i] = (du[i] - u[i] * udu) / vn;
    if (with_mask) {                                                      // sigmoid, then d|n|/dn = n/|n|
      const double ds = static_cast<double>(dm) * md * (1.0 - md) * (black ? 255.0 : -255.0) / nnd;
#pragma unroll
      for (int i = 0; i < 3; ++i) dn[i] += static_cast<float>(ds * n[i]);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) d_normal[o + i] = dn[i];
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
    atomicAdd(loss + b, static_cast<double>(t[0]) / (3.0 * HW));
    const float ldt = L[0] * t[1] + L[1] * t[2] + L[2] * t[3];           // d (l/|l|) = (dL - L (L.dL)) / |l|
    if (d_light != nullptr)
      for (int i = 0; i < 3; ++i) atomicAdd(d_light + 3 * b + i, (t[1 + i] - L[i] * ldt) / lnorm);
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
    case 1: resample_backward_kernel<1><<<grid, 256, 0, st>>>(vox, minv, gout, dvox, dminv, B, size, new_size, transform); break;
    case 4: resample_backward_kernel<4><<<grid, 256, 0, st>>>(vox, minv, gout, dvox, dminv, B, size, new_size, transform); break;
    default: return -3;
  }
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_resample5_backward_f32(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox,
                                         float* dtex, float* dminv, int B, int size, int new_size, void* stream) {
  if (!vox || !tex || !minv || !gout || (!dvox && !dtex && !dminv) || B < 1 || size < 2 || new_size < 1) return -1;
  if ((new_size * new_size) % 8 != 0) return -2;      // a block's 8 rows must belong to one batch item
  if ((reinterpret_cast<uintptr_t>(tex) & 15) != 0 || (reinterpret_cast<uintptr_t>(dtex) & 15) != 0) return -3;
  const long long rows = static_cast<long long>(B) * new_size * new_size;
  resample5_backward_kernel<<<static_cast<int>((rows * 32 + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      vox, tex, minv, gout, dvox, dtex, dminv, B, size, new_size);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
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
  phong_recon_loss_grad_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      albedo, normal, target, light_dir, light_col, ambient, k_diffuse, black_background, with_mask, loss, d_albedo, d_normal,
      d_light_dir, HW);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}
