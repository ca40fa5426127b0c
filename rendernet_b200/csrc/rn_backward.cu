// rn_backward.cu -- CUDA-core kernels of the BACKWARD (input-gradient) pass of the forward rendering path (SURVEY §8 f-4):
// what inverse rendering differentiates through the frozen network (Reconstruct_RenderNet_Face.py:383-412: tf.gradients of an
// image loss w.r.t. shape / texture / pose).  The dense contractions of the backward pass (data gradients of every stride-1
// convolution and transposed convolution) run on the tensor cores through the same implicit-GEMM kernel as the forward pass
// (rendernet_b200/backward.py: mirrored taps, transposed packed filters); this file holds what is not a GEMM:
//   * activation derivatives (PReLU tools/layer_util.py:27-45, sigmoid RenderNet_Shader.py:127-130),
//   * data gradients of the two thin strided 3-D convolutions e_conv1 / e_conv2 (RenderNet_Shader.py:36-43),
//   * the backward of the trilinear resampler (tools/resampling_voxel_grid.py:381-614 + tools/model_util.py:41-49) with
//     respect to the voxel grid (scatter-add of the 8 corner weights) and to the 3x4 inverse sampling matrix (derivative of
//     the corner weights w.r.t. the sample coordinates), from which the host derives d/d(azimuth, elevation, scale).
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
