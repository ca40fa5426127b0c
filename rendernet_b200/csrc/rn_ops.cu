// rn_ops.cu -- the non-tensor-core kernels of the RenderNet forward path and the reference-shaped C-ABI
// wrappers over the implicit-GEMM kernel (rn_igemm.cu).
//   * fused rotate + trilinear resample + axis transform  (tools/resampling_voxel_grid.py:381-614,
//     tools/model_util.py:41-49)                                               -> HBM-bound gather
//   * weight packing / casts
//   * thin 3-D convolutions e_conv1 / e_conv2 on CUDA cores (RenderNet_Shader.py:36-43)
//   * Phong composite + uint8 quantisation (tools/Phong_shading.py:138-228, RenderNet_demo.py:54-58)
#include <cstdio>
#include <cstring>
#include <vector>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "../../include/rendernet_b200.h"

#include <atomic>
#include "rn_igemm.cuh"
#include "rn_phong.cuh"
namespace rn {
extern std::atomic<long long> g_launch_count;
#define RN_COUNT_LAUNCH() rn::g_launch_count.fetch_add(1, std::memory_order_relaxed)

// 16-bit storage in the three formats of the C ABI (RN_FMT_*): fp16, bf16, or an fp16 hi/lo pair whose LO plane lives
// `plane` elements after the HI plane (hi = fp16(v), lo = fp16(v - hi)).
__device__ __forceinline__ void store16(uint16_t* __restrict__ p, long long i, float v, int fmt, long long plane) {
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
// two values -> one packed 32-bit word of the HI plane (and of the LO plane for fmt 2)
__device__ __forceinline__ void pack16x2(float v0, float v1, int fmt, uint32_t* hi, uint32_t* lo) {
  if (fmt == 1) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1);
    *hi = *reinterpret_cast<const uint32_t*>(&h);
    *lo = 0u;
  } else {
    const __half2 h = __floats2half2_rn(v0, v1);
    *hi = *reinterpret_cast<const uint32_t*>(&h);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    *lo = *reinterpret_cast<const uint32_t*>(&l);
  }
}
__device__ __forceinline__ float load16(const uint16_t* __restrict__ p, long long i, int fmt, long long plane) {
  const uint16_t u = p[i];
  if (fmt == 1) return __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&u));
  float v = __half2float(*reinterpret_cast<const __half*>(&u));
  if (fmt == 2) {
    const uint16_t l = p[i + plane];
    v += __half2float(*reinterpret_cast<const __half*>(&l));
  }
  return v;
}

// ------------------------------------------------------------------------------------------ resampler
// One row of p_src = Minv . (gx, gy, gz, 1) (tools/resampling_voxel_grid.py:605) in the arithmetic of a float32 matmul that
// accumulates over k = 0..3 with fused multiply-adds -- what NumPy/OpenBLAS (and therefore the oracle) computes: verified
// bit for bit against np.matmul on all 128^3 grid points for five poses.  The order matters: axis-aligned poses put sample
// points exactly ON the clamp discontinuity at 0 / size-1, where one ulp decides between a voxel value and zero.
__device__ __forceinline__ float sample_coord(float m0, float m1, float m2, float m3, float gx, float gy, float gz) {
  return __fadd_rn(__fmaf_rn(m2, gz, __fmaf_rn(m1, gy, __fmul_rn(m0, gx))), m3);
}

// One warp per output row (innermost output axis); each lane owns 4 consecutive points per iteration so
// C=1 rows are written with one 16-byte store per lane (512 B per warp instruction).  The rows are those of the window
// o1 in [wy0, wy0+wh), o2 in [wx0, wx0+ww) of the nsz^2 output rows per item (the whole grid: 0, 0, nsz, nsz), written
// densely: out is [B,wh,ww,nsz,C].
template <int C>
__global__ void __launch_bounds__(256) resample_kernel(const float* __restrict__ vox, const float* __restrict__ minv,
                                                       float* __restrict__ out, int B, int size, int nsz,
                                                       int transform, int wy0, int wx0, int wh, int ww) {
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int rows = B * wh * ww;
  if (warp_global >= rows) return;
  const int b = warp_global / (wh * ww);
  const int o1 = wy0 + (warp_global / ww) % wh;
  const int o2 = wx0 + warp_global % ww;
  const float* M = minv + b * 12;
  const float m00 = __ldg(M + 0), m01 = __ldg(M + 1), m02 = __ldg(M + 2), m03 = __ldg(M + 3);
  const float m10 = __ldg(M + 4), m11 = __ldg(M + 5), m12 = __ldg(M + 6), m13 = __ldg(M + 7);
  const float m20 = __ldg(M + 8), m21 = __ldg(M + 9), m22 = __ldg(M + 10), m23 = __ldg(M + 11);
  // grid point (gx, gy, gz) = (k, j, i) (:500-512); with the axis transform N[b,p,q,r] = T[b,q,nsz-1-p,r]
  const float gy = transform ? static_cast<float>(nsz - 1 - o1) : static_cast<float>(o2);
  const float gz = transform ? static_cast<float>(o2) : static_cast<float>(o1);
  const float lim = static_cast<float>(size - 1);
  const float* vb = vox + static_cast<size_t>(b) * size * size * size * C;
  float* orow = out + static_cast<size_t>(warp_global) * nsz * C;

  for (int r0 = lane * 4; r0 < nsz; r0 += 128) {
    float res[4][C];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float gx = static_cast<float>(r0 + u);
      const float x = sample_coord(m00, m01, m02, m03, gx, gy, gz);
      const float y = sample_coord(m10, m11, m12, m13, gx, gy, gz);
      const float z = sample_coord(m20, m21, m22, m23, gx, gy, gz);
#pragma unroll
      for (int c = 0; c < C; ++c) res[u][c] = 0.f;
      // clamp-then-weight rule (:410-485): both clamped corners coincide outside [0,size-1) -> weights cancel
      if (x >= 0.f && x < lim && y >= 0.f && y < lim && z >= 0.f && z < lim && (r0 + u) < nsz) {
        const float x0f = floorf(x), y0f = floorf(y), z0f = floorf(z);
        const int x0 = static_cast<int>(x0f), y0 = static_cast<int>(y0f), z0 = static_cast<int>(z0f);
        const float x1f = x0f + 1.f, y1f = y0f + 1.f, z1f = z0f + 1.f;
        const float ax = __fsub_rn(x1f, x), bxw = __fsub_rn(x, x0f);
        const float ay = __fsub_rn(y1f, y), byw = __fsub_rn(y, y0f);
        const float az = __fsub_rn(z1f, z), bzw = __fsub_rn(z, z0f);
        const float wa = __fmul_rn(__fmul_rn(ax, ay), az), wb = __fmul_rn(__fmul_rn(ax, byw), az);
        const float wc = __fmul_rn(__fmul_rn(bxw, ay), az), wd = __fmul_rn(__fmul_rn(bxw, byw), az);
        const float we = __fmul_rn(__fmul_rn(ax, ay), bzw), wf = __fmul_rn(__fmul_rn(ax, byw), bzw);
        const float wg = __fmul_rn(__fmul_rn(bxw, ay), bzw), wh = __fmul_rn(__fmul_rn(bxw, byw), bzw);
        const size_t i000 = ((static_cast<size_t>(z0) * size + y0) * size + x0) * C;  // flat = z*W*H + y*W + x
        const size_t sy = static_cast<size_t>(size) * C, sz = static_cast<size_t>(size) * size * C;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          const float Ia = __ldg(vb + i000 + c), Ib = __ldg(vb + i000 + sy + c);
          const float Ic = __ldg(vb + i000 + C + c), Id = __ldg(vb + i000 + sy + C + c);
          const float Ie = __ldg(vb + i000 + sz + c), If = __ldg(vb + i000 + sz + sy + c);
          const float Ig = __ldg(vb + i000 + sz + C + c), Ih = __ldg(vb + i000 + sz + sy + C + c);
          float s = __fmul_rn(wa, Ia);                       // add_n order a..h (:485)
          s = __fadd_rn(s, __fmul_rn(wb, Ib));
          s = __fadd_rn(s, __fmul_rn(wc, Ic));
          s = __fadd_rn(s, __fmul_rn(wd, Id));
          s = __fadd_rn(s, __fmul_rn(we, Ie));
          s = __fadd_rn(s, __fmul_rn(wf, If));
          s = __fadd_rn(s, __fmul_rn(wg, Ig));
          s = __fadd_rn(s, __fmul_rn(wh, Ih));
          res[u][c] = s;
        }
      }
    }
    if constexpr (C == 1) {
      if (r0 + 3 < nsz) {
        *reinterpret_cast<float4*>(orow + r0) = make_float4(res[0][0], res[1][0], res[2][0], res[3][0]);
      } else {
        for (int u = 0; u < 4 && r0 + u < nsz; ++u) orow[r0 + u] = res[u][0];
      }
    } else {
      for (int u = 0; u < 4 && r0 + u < nsz; ++u) {
        if constexpr (C == 4) {
          *reinterpret_cast<float4*>(orow + static_cast<size_t>(r0 + u) * 4) =
              make_float4(res[u][0], res[u][1], res[u][2], res[u][3]);
        } else {
#pragma unroll
          for (int c = 0; c < C; ++c) orow[static_cast<size_t>(r0 + u) * C + c] = res[u][c];
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ tf_interpolate
// tools/resampling_voxel_grid.py:381-486 at caller-supplied sample coordinates, operation for operation: BOTH corners of
// every axis are clamped to [0, size-1] (:410-422) and the weights come from the CLAMPED corners (:465-482), so a point
// outside the cube gets two coincident corners whose weights cancel up to fp32 rounding (the reference's <= 2e-4 |v|
// "noise", reproduced here bit for bit -- unlike resample_kernel, which writes exact zeros there).  One thread per point.
__global__ void __launch_bounds__(256) interpolate_kernel(const float* __restrict__ vox, const float* __restrict__ xs,
                                                          const float* __restrict__ ys, const float* __restrict__ zs,
                                                          float* __restrict__ out, long long n_total, long long n_per_item,
                                                          int C, int size) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n_total) return;
  const long long b = i / n_per_item;
  const float x = xs[i], y = ys[i], z = zs[i];
  const int mx = size - 1;
  int x0 = static_cast<int>(floorf(x)), y0 = static_cast<int>(floorf(y)), z0 = static_cast<int>(floorf(z));
  int x1 = x0 + 1, y1 = y0 + 1, z1 = z0 + 1;
  x0 = min(max(x0, 0), mx); x1 = min(max(x1, 0), mx);
  y0 = min(max(y0, 0), mx); y1 = min(max(y1, 0), mx);
  z0 = min(max(z0, 0), mx); z1 = min(max(z1, 0), mx);
  const float x0f = static_cast<float>(x0), x1f = static_cast<float>(x1), y0f = static_cast<float>(y0);
  const float y1f = static_cast<float>(y1), z0f = static_cast<float>(z0), z1f = static_cast<float>(z1);
  const float ax = __fsub_rn(x1f, x), bx = __fsub_rn(x, x0f), ay = __fsub_rn(y1f, y), by = __fsub_rn(y, y0f);
  const float az = __fsub_rn(z1f, z), bz = __fsub_rn(z, z0f);
  const float wa = __fmul_rn(__fmul_rn(ax, ay), az), wb = __fmul_rn(__fmul_rn(ax, by), az);
  const float wc = __fmul_rn(__fmul_rn(bx, ay), az), wd = __fmul_rn(__fmul_rn(bx, by), az);
  const float we = __fmul_rn(__fmul_rn(ax, ay), bz), wf = __fmul_rn(__fmul_rn(ax, by), bz);
  const float wg = __fmul_rn(__fmul_rn(bx, ay), bz), wh = __fmul_rn(__fmul_rn(bx, by), bz);
  const float* vb = vox + static_cast<size_t>(b) * size * size * size * C;
  auto at = [&](int zz, int yy, int xx) { return vb + ((static_cast<size_t>(zz) * size + yy) * size + xx) * C; };
  const float *pa = at(z0, y0, x0), *pb = at(z0, y1, x0), *pc = at(z0, y0, x1), *pd = at(z0, y1, x1);
  const float *pe = at(z1, y0, x0), *pf = at(z1, y1, x0), *pg = at(z1, y0, x1), *ph = at(z1, y1, x1);
  for (int c = 0; c < C; ++c) {
    float s = __fmul_rn(wa, __ldg(pa + c));                    // add_n order a..h (:485)
    s = __fadd_rn(s, __fmul_rn(wb, __ldg(pb + c)));
    s = __fadd_rn(s, __fmul_rn(wc, __ldg(pc + c)));
    s = __fadd_rn(s, __fmul_rn(wd, __ldg(pd + c)));
    s = __fadd_rn(s, __fmul_rn(we, __ldg(pe + c)));
    s = __fadd_rn(s, __fmul_rn(wf, __ldg(pf + c)));
    s = __fadd_rn(s, __fmul_rn(wg, __ldg(pg + c)));
    s = __fadd_rn(s, __fmul_rn(wh, __ldg(ph + c)));
    out[i * C + c] = s;
  }
}

// ------------------------------------------------------------------------------------------ packing / casts
struct TapSel { int n; int idx[64]; };

__global__ void pack_weights_kernel(const float* __restrict__ w, uint16_t* __restrict__ packed, int Cin, int Cout,
                                    int cout_pad, int transposed, TapSel sel, int fmt, long long plane) {
  const long long total = static_cast<long long>(sel.n) * cout_pad * Cin;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % Cin);
    const int co = static_cast<int>((i / Cin) % cout_pad);
    const int t = static_cast<int>(i / (static_cast<long long>(Cin) * cout_pad));
    float v = 0.f;
    if (co < Cout) {
      const long long base = static_cast<long long>(sel.idx[t]) * Cin * Cout;
      v = transposed ? w[base + static_cast<long long>(co) * Cin + ci] : w[base + static_cast<long long>(ci) * Cout + co];
    }
    store16(packed, i, v, fmt, plane);
  }
}

__global__ void cast_f32_to_16_kernel(const float* __restrict__ s, uint16_t* __restrict__ d, long long n,
                                      long long n_pad, int fmt) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_pad;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = i < n ? s[i] : 0.f;
    store16(d, i, v, fmt, n_pad);
  }
}

__global__ void cast_16_to_f32_kernel(const uint16_t* __restrict__ s, float* __restrict__ d, long long n, int fmt) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    d[i] = load16(s, i, fmt, n);
  }
}



// ------------------------------------------------------------------------------------------ banded conv3d filter
// Wb[tap=(ky,kx)][i][n'][k = zi_l*Cin + ci]: K block i of the processing order is block kb = order[i] of the band.
// Relative to the N tile's first output depth z0: zi = sz*z0 - pz + kb*(64/Cin) + zi_l, zo = z0 + zo_l
//   ->  kz = zi - (sz*zo - pz) = kb*(64/Cin) + zi_l - sz*zo_l;  entry = w[ky][kx][kz][ci][co] when 0 <= kz < 3, else 0.
// Row n' of a tile holds filter row n = zo_l*Cout + co.  Full blocks: n = n'.  Half blocks (they feed only columns
// [base, base+64) of the tile, base = 0 or 64; rn_igemm.cuh band_layout) keep the needed rows FIRST so that an N = 64 MMA finds
// them at the start of the operand: n = base + n' for n' < 64.  Unused rows are zero.   (BN = 128, KB = 64; sz = z stride)
__global__ void pack_banded_kernel(const float* __restrict__ w, uint16_t* __restrict__ packed, int Cin, int Cout,
                                   BandLayout L, int sz, int fmt, long long plane) {
  const int kblocks = L.kblocks;
  const long long total = 9LL * kblocks * 128 * 64;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % 64);
    const int np = static_cast<int>((i / 64) % 128);
    const int bi = static_cast<int>((i / (64 * 128)) % kblocks);
    const int tap = static_cast<int>(i / (64LL * 128 * kblocks));
    const int kb = L.order[bi], half = L.half[bi];
    int n = np;
    if (half != 0) n = np < 64 ? (half == 2 ? 64 : 0) + np : -1;
    float v = 0.f;
    if (n >= 0) {
      const int zi_l = k / Cin, ci = k % Cin, zo_l = n / Cout, co = n % Cout;
      const int kz = kb * (64 / Cin) + zi_l - sz * zo_l;
      if (kz >= 0 && kz <= 2) v = w[((static_cast<long long>(tap) * 3 + kz) * Cin + ci) * Cout + co];
    }
    store16(packed, i, v, fmt, plane);
  }
}

// ------------------------------------------------------------------------------------------ sliced conv3d filter
// Ws[plane][tap=(ky,kx)][r = zs*32 + co][ci] = w[ky][kx][kz = 2 - zs][ci][co]: one K-major [96 x 32] tile per (ky, kx) whose
// three 32-row slices are the kz = 2, 1, 0 filters: slice zs is what input depth j contributes to output depth j - 2 + zs
// (rn_conv3d_sliced.cu).  Cin = Cout = 32; the LO plane (fmt 2) follows the HI plane.
__global__ void pack_sliced_kernel(const float* __restrict__ w, uint16_t* __restrict__ packed, int fmt, long long plane) {
  const int total = 9 * 96 * 32;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int ci = i % 32, r = (i / 32) % 96, tap = i / (32 * 96);
    const int kz = 2 - r / 32, co = r % 32;
    store16(packed, i, w[((tap * 3 + kz) * 32 + ci) * 32 + co], fmt, plane);
  }
}

__global__ void expand_channels_kernel(const float* __restrict__ v, float* __restrict__ out, int C, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v[i % C];
}

// ------------------------------------------------------------------------------------------ elementwise
// y = act(x + bias[c]) + residual, 16-bit in/out, channel = innermost axis (standalone prelu / tf.add /
// sigmoid when they cannot be fused into a convolution epilogue; tools/layer_util.py:27-45,73,105).
__global__ void bias_act_kernel(const uint16_t* __restrict__ x, const float* __restrict__ bias,
                                const float* __restrict__ alpha, int act, const uint16_t* __restrict__ res,
                                uint16_t* __restrict__ out, float* __restrict__ out32, long long n, int C, int fmt) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    float v = load16(x, i, fmt, n);
    if (bias != nullptr) v += bias[c];
    if (act == 1) v = fmaxf(v, 0.f) + alpha[c] * fminf(v, 0.f);
    else if (act == 2) v = 1.f / (1.f + __expf(-v));
    if (res != nullptr) v += load16(res, i, fmt, n);
    if (out != nullptr) store16(out, i, v, fmt, n);
    if (out32 != nullptr) out32[i] = v;
  }
}

// ------------------------------------------------------------------------------------------ thin conv3d
// Direct SAME convolution, one thread per output voxel, all COUT accumulators in registers; the filter
// ([tap][ci][co] fp32, <= 14 KB) sits in shared memory and is read as warp-broadcast float4.
template <int CIN, int COUT, int K, bool X_F32>
__global__ void __launch_bounds__(256) conv3d_direct_kernel(const void* __restrict__ xv, const float* __restrict__ w,
                                                            const float* __restrict__ bias,
                                                            const float* __restrict__ alpha,
                                                            uint16_t* __restrict__ out, int B, int H, int W, int D,
                                                            int Ho, int Wo, int Do, int sy, int sx, int sz, int py,
                                                            int px, int pz, int fmt) {
  __shared__ __align__(16) float ws[K * K * K * CIN * COUT];
  for (int i = threadIdx.x; i < K * K * K * CIN * COUT; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const long long total = static_cast<long long>(B) * Ho * Wo * Do;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int oz = static_cast<int>(idx % Do);
  const int ox = static_cast<int>((idx / Do) % Wo);
  const int oy = static_cast<int>((idx / (static_cast<long long>(Do) * Wo)) % Ho);
  const int b = static_cast<int>(idx / (static_cast<long long>(Do) * Wo * Ho));
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  const int iy0 = oy * sy - py, ix0 = ox * sx - px, iz0 = oz * sz - pz;
  for (int ky = 0; ky < K; ++ky) {
    const int iy = iy0 + ky;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < K; ++kx) {
      const int ix = ix0 + kx;
      if (ix < 0 || ix >= W) continue;
      const size_t rowbase = ((static_cast<size_t>(b) * H + iy) * W + ix) * D;
#pragma unroll
      for (int kz = 0; kz < K; ++kz) {
        const int iz = iz0 + kz;
        if (iz < 0 || iz >= D) continue;
        float xin[CIN];
        if constexpr (X_F32) {
          const float* xp = static_cast<const float*>(xv) + (rowbase + iz) * CIN;
#pragma unroll
          for (int ci = 0; ci < CIN; ++ci) xin[ci] = __ldg(xp + ci);
        } else {
          static_assert(X_F32 || CIN % 8 == 0, "16-bit input needs CIN % 8 == 0");
          const uint4* xp = reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(xv) + (rowbase + iz) * CIN);
          const long long xplane8 = (static_cast<long long>(B) * H * W * D * CIN) >> 3;   // fmt 2: LO plane, in uint4 units
#pragma unroll
          for (int v = 0; v < CIN / 8; ++v) {
            const uint4 q = __ldg(xp + v);
            const uint32_t u[4] = {q.x, q.y, q.z, q.w};
            uint32_t ul[4] = {0u, 0u, 0u, 0u};
            if (fmt == 2) { const uint4 ql = __ldg(xp + v + xplane8); ul[0] = ql.x; ul[1] = ql.y; ul[2] = ql.z; ul[3] = ql.w; }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float2 f;
              if (fmt == 1) f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u[j]));
              else {
                f = __half22float2(*reinterpret_cast<const __half2*>(&u[j]));
                if (fmt == 2) { const float2 g = __half22float2(*reinterpret_cast<const __half2*>(&ul[j])); f.x += g.x; f.y += g.y; }
              }
              xin[v * 8 + 2 * j] = f.x;
              xin[v * 8 + 2 * j + 1] = f.y;
            }
          }
        }
        const float* wt = ws + ((ky * K + kx) * K + kz) * CIN * COUT;
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) {
#pragma unroll
          for (int c4 = 0; c4 < COUT; c4 += 4) {
            const float4 w4 = *reinterpret_cast<const float4*>(wt + ci * COUT + c4);
            acc[c4 + 0] = fmaf(xin[ci], w4.x, acc[c4 + 0]);
            acc[c4 + 1] = fmaf(xin[ci], w4.y, acc[c4 + 1]);
            acc[c4 + 2] = fmaf(xin[ci], w4.z, acc[c4 + 2]);
            acc[c4 + 3] = fmaf(xin[ci], w4.w, acc[c4 + 3]);
          }
        }
      }
    }
  }
  uint32_t pk[COUT / 2], pl[COUT / 2];
#pragma unroll
  for (int c = 0; c < COUT; c += 2) {
    float v0 = acc[c] + __ldg(bias + c), v1 = acc[c + 1] + __ldg(bias + c + 1);
    if (alpha != nullptr) {
      v0 = fmaxf(v0, 0.f) + __ldg(alpha + c) * fminf(v0, 0.f);
      v1 = fmaxf(v1, 0.f) + __ldg(alpha + c + 1) * fminf(v1, 0.f);
    }
    pack16x2(v0, v1, fmt, &pk[c / 2], &pl[c / 2]);
  }
  uint4* op = reinterpret_cast<uint4*>(out + static_cast<size_t>(idx) * COUT);
#pragma unroll
  for (int v = 0; v < COUT / 8; ++v) op[v] = make_uint4(pk[4 * v], pk[4 * v + 1], pk[4 * v + 2], pk[4 * v + 3]);
  if (fmt == 2) {
    uint4* ol = op + ((total * COUT) >> 3);      // LO plane
#pragma unroll
    for (int v = 0; v < COUT / 8; ++v) ol[v] = make_uint4(pl[4 * v], pl[4 * v + 1], pl[4 * v + 2], pl[4 * v + 3]);
  }
}


// ------------------------------------------------------------------------------------------ resampler (+) e_conv1
// SURVEY §8 f-1: rotate/resample (tools/resampling_voxel_grid.py:381-614) + axis transform (tools/model_util.py:41-49)
// + e_conv1 (5^3, stride 2, 1 -> 8, SAME = pad 1 before / 2 after; RenderNet_Shader.py:36-39) + bias + PReLU in one
// kernel: the 128^3 fp32 grid (8.4 MB per render) is never written.  One CTA = 8^3 outputs; it samples the 19^3 input
// points it needs into shared memory (same arithmetic, operation for operation, as resample_kernel), and if every one
// of them is exactly 0 -- outside the rotated cube or empty space, ~85-90 % of all tiles -- the outputs are
// PReLU(bias) and the 5^3 convolution is skipped.  Accumulation order per output = conv3d_direct_kernel's
// (ky, kx, kz), so results are bit-identical to the unfused pair.  The CTAs cover a window of rows [wy0, wy0+wh) x columns
// [wx0, wx0+ww) of the transformed grid (all depths; the whole grid: 0, 0, nsz, nsz): points outside it are SAME padding,
// as when the grid is sliced before the convolution (training on patches, RenderNet_Shader.py:150-156).
constexpr int RC_T = 8;                 // outputs per tile edge
constexpr int RC_IN = 2 * RC_T + 3;     // 19 input points per edge
constexpr int RC_ZP = 20;               // padded z row: even z at [0,10), odd z at [10,19) -> conflict-free stride-2 reads

__global__ void __launch_bounds__(256) resample_conv1_kernel(const float* __restrict__ vox,
                                                             const float* __restrict__ minv,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             const float* __restrict__ alpha, uint16_t* __restrict__ out,
                                                             int B, int size, int nsz, int fmt, int wy0, int wx0, int wh,
                                                             int ww) {
  __shared__ float tile[RC_IN * RC_IN * RC_ZP];
  __shared__ __align__(16) float ws[125 * 8];
  const int tid = threadIdx.x;
  const int Ho = wh >> 1, Wo = ww >> 1, Do = nsz >> 1;      // output extents of the window
  const int tpy = Ho / RC_T, tpx = Wo / RC_T, tpz = Do / RC_T;
  int bid = blockIdx.x;
  const int tz = bid % tpz; bid /= tpz;
  const int tx = bid % tpx; bid /= tpx;
  const int ty = bid % tpy;
  const int b = bid / tpy;
  for (int i = tid; i < 125 * 8; i += 256) ws[i] = __ldg(w + i);

  const float* M = minv + b * 12;
  const float m00 = __ldg(M + 0), m01 = __ldg(M + 1), m02 = __ldg(M + 2), m03 = __ldg(M + 3);
  const float m10 = __ldg(M + 4), m11 = __ldg(M + 5), m12 = __ldg(M + 6), m13 = __ldg(M + 7);
  const float m20 = __ldg(M + 8), m21 = __ldg(M + 9), m22 = __ldg(M + 10), m23 = __ldg(M + 11);
  const float lim = static_cast<float>(size - 1);
  const float* vb = vox + static_cast<size_t>(b) * size * size * size;
  const size_t sy = static_cast<size_t>(size), sz = static_cast<size_t>(size) * size;
  const int p0 = wy0 + 2 * ty * RC_T - 1, q0 = wx0 + 2 * tx * RC_T - 1, r0 = 2 * tz * RC_T - 1;

  // Tile-level rejection: the source coordinate is affine in (p,q,r), so over the tile's input box each of x,y,z is
  // bounded by its values at the box's 8 corners.  If one axis lies entirely outside [0, size-1) (with a margin far
  // above the fmaf rounding of the per-point evaluation) every sample is exactly 0 by the clamp rule and neither the
  // gather nor the convolution runs.
  int nonzero = 0;
  bool maybe_inside = true;
  {
    const float pl = static_cast<float>(max(p0, wy0)), ph = static_cast<float>(min(p0 + RC_IN - 1, wy0 + wh - 1));
    const float ql = static_cast<float>(max(q0, wx0)), qh = static_cast<float>(min(q0 + RC_IN - 1, wx0 + ww - 1));
    const float rl = static_cast<float>(max(r0, 0)), rh = static_cast<float>(min(r0 + RC_IN - 1, nsz - 1));
    const float gyl = static_cast<float>(nsz - 1) - ph, gyh = static_cast<float>(nsz - 1) - pl;   // gy = nsz-1-p
    const float mrow[3][4] = {{m00, m01, m02, m03}, {m10, m11, m12, m13}, {m20, m21, m22, m23}};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      // interval arithmetic: min/max of m0*gx + m1*gy + m2*gz + m3 over gx in [rl,rh], gy in [gyl,gyh], gz in [ql,qh]
      const float lo = fminf(mrow[a][0] * rl, mrow[a][0] * rh) + fminf(mrow[a][1] * gyl, mrow[a][1] * gyh) +
                       fminf(mrow[a][2] * ql, mrow[a][2] * qh) + mrow[a][3];
      const float hi = fmaxf(mrow[a][0] * rl, mrow[a][0] * rh) + fmaxf(mrow[a][1] * gyl, mrow[a][1] * gyh) +
                       fmaxf(mrow[a][2] * ql, mrow[a][2] * qh) + mrow[a][3];
      if (hi < -0.01f || lo > lim + 0.01f) maybe_inside = false;
    }
  }
  if (maybe_inside) {
    // i = (iy*19 + ix)*19 + iz walked with a stride of 256 = 13*19 + 9 without divisions
    int iz = tid % RC_IN, row = tid / RC_IN;
    for (int i = tid; i < RC_IN * RC_IN * RC_IN; i += 256) {
      const int iy = row / RC_IN, ix = row - iy * RC_IN;
      const int p = p0 + iy, q = q0 + ix, r = r0 + iz;
      float v = 0.f;
      if (p >= wy0 && p < wy0 + wh && q >= wx0 && q < wx0 + ww && r >= 0 && r < nsz) {   // SAME zeros at the window border
        // N[b,p,q,r] = T[b,q,nsz-1-p,r]; grid point (gx,gy,gz) = (r, nsz-1-p, q)
        const float gx = static_cast<float>(r), gy = static_cast<float>(nsz - 1 - p), gz = static_cast<float>(q);
        const float x = sample_coord(m00, m01, m02, m03, gx, gy, gz);
        const float y = sample_coord(m10, m11, m12, m13, gx, gy, gz);
        const float z = sample_coord(m20, m21, m22, m23, gx, gy, gz);
        if (x >= 0.f && x < lim && y >= 0.f && y < lim && z >= 0.f && z < lim) {
          const float x0f = floorf(x), y0f = floorf(y), z0f = floorf(z);
          const int x0 = static_cast<int>(x0f), y0 = static_cast<int>(y0f), z0 = static_cast<int>(z0f);
          const float x1f = x0f + 1.f, y1f = y0f + 1.f, z1f = z0f + 1.f;
          const float ax = __fsub_rn(x1f, x), bxw = __fsub_rn(x, x0f);
          const float ay = __fsub_rn(y1f, y), byw = __fsub_rn(y, y0f);
          const float az = __fsub_rn(z1f, z), bzw = __fsub_rn(z, z0f);
          const float wa = __fmul_rn(__fmul_rn(ax, ay), az), wb = __fmul_rn(__fmul_rn(ax, byw), az);
          const float wc = __fmul_rn(__fmul_rn(bxw, ay), az), wd = __fmul_rn(__fmul_rn(bxw, byw), az);
          const float we = __fmul_rn(__fmul_rn(ax, ay), bzw), wf = __fmul_rn(__fmul_rn(ax, byw), bzw);
          const float wg = __fmul_rn(__fmul_rn(bxw, ay), bzw), wh = __fmul_rn(__fmul_rn(bxw, byw), bzw);
          const float* c0 = vb + (static_cast<size_t>(z0) * size + y0) * size + x0;
          float s = __fmul_rn(wa, __ldg(c0));                       // add_n order a..h (:485)
          s = __fadd_rn(s, __fmul_rn(wb, __ldg(c0 + sy)));
          s = __fadd_rn(s, __fmul_rn(wc, __ldg(c0 + 1)));
          s = __fadd_rn(s, __fmul_rn(wd, __ldg(c0 + sy + 1)));
          s = __fadd_rn(s, __fmul_rn(we, __ldg(c0 + sz)));
          s = __fadd_rn(s, __fmul_rn(wf, __ldg(c0 + sz + sy)));
          s = __fadd_rn(s, __fmul_rn(wg, __ldg(c0 + sz + 1)));
          s = __fadd_rn(s, __fmul_rn(wh, __ldg(c0 + sz + sy + 1)));
          v = s;
        }
      }
      nonzero |= (v != 0.f);
      tile[row * RC_ZP + (iz & 1) * 10 + (iz >> 1)] = v;
      iz += 256 % RC_IN;
      row += 256 / RC_IN;
      if (iz >= RC_IN) { iz -= RC_IN; ++row; }
    }
  }
  const int any = __syncthreads_or(nonzero);

  const int oz = tid & 7, ox = (tid >> 3) & 7, oy = tid >> 6;   // second output: oy + 4
  float acc0[8], acc1[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc0[c] = acc1[c] = 0.f;
  if (any) {
    for (int ky = 0; ky < 5; ++ky) {
      for (int kx = 0; kx < 5; ++kx) {
        const float* t0 = tile + ((2 * oy + ky) * RC_IN + (2 * ox + kx)) * RC_ZP + oz;
        const float* t1 = t0 + 8 * RC_IN * RC_ZP;
        const float4* wt = reinterpret_cast<const float4*>(ws + (ky * 5 + kx) * 5 * 8);
#pragma unroll
        for (int kz = 0; kz < 5; ++kz) {
          const int zi = (kz & 1) * 10 + (kz >> 1);
          const float a0 = t0[zi], a1 = t1[zi];
          const float4 wlo = wt[2 * kz], whi = wt[2 * kz + 1];
          acc0[0] = fmaf(a0, wlo.x, acc0[0]); acc0[1] = fmaf(a0, wlo.y, acc0[1]);
          acc0[2] = fmaf(a0, wlo.z, acc0[2]); acc0[3] = fmaf(a0, wlo.w, acc0[3]);
          acc0[4] = fmaf(a0, whi.x, acc0[4]); acc0[5] = fmaf(a0, whi.y, acc0[5]);
          acc0[6] = fmaf(a0, whi.z, acc0[6]); acc0[7] = fmaf(a0, whi.w, acc0[7]);
          acc1[0] = fmaf(a1, wlo.x, acc1[0]); acc1[1] = fmaf(a1, wlo.y, acc1[1]);
          acc1[2] = fmaf(a1, wlo.z, acc1[2]); acc1[3] = fmaf(a1, wlo.w, acc1[3]);
          acc1[4] = fmaf(a1, whi.x, acc1[4]); acc1[5] = fmaf(a1, whi.y, acc1[5]);
          acc1[6] = fmaf(a1, whi.z, acc1[6]); acc1[7] = fmaf(a1, whi.w, acc1[7]);
        }
      }
    }
  }
  uint32_t pk0[4], pk1[4], pl0[4], pl1[4];
#pragma unroll
  for (int c = 0; c < 8; c += 2) {
    const float b0 = __ldg(bias + c), b1 = __ldg(bias + c + 1);
    float u0 = acc0[c] + b0, u1 = acc0[c + 1] + b1, v0 = acc1[c] + b0, v1 = acc1[c + 1] + b1;
    if (alpha != nullptr) {
      const float al0 = __ldg(alpha + c), al1 = __ldg(alpha + c + 1);
      u0 = fmaxf(u0, 0.f) + al0 * fminf(u0, 0.f);
      u1 = fmaxf(u1, 0.f) + al1 * fminf(u1, 0.f);
      v0 = fmaxf(v0, 0.f) + al0 * fminf(v0, 0.f);
      v1 = fmaxf(v1, 0.f) + al1 * fminf(v1, 0.f);
    }
    pack16x2(u0, u1, fmt, &pk0[c / 2], &pl0[c / 2]);
    pack16x2(v0, v1, fmt, &pk1[c / 2], &pl1[c / 2]);
  }
  const size_t o0 = (((static_cast<size_t>(b) * Ho + (ty * RC_T + oy)) * Wo + (tx * RC_T + ox)) * Do + (tz * RC_T + oz)) * 8;
  const size_t o1 = o0 + static_cast<size_t>(4) * Wo * Do * 8;
  *reinterpret_cast<uint4*>(out + o0) = make_uint4(pk0[0], pk0[1], pk0[2], pk0[3]);
  *reinterpret_cast<uint4*>(out + o1) = make_uint4(pk1[0], pk1[1], pk1[2], pk1[3]);
  if (fmt == 2) {    // LO plane of the fp16 hi/lo pair
    const size_t plane = static_cast<size_t>(B) * Ho * Wo * Do * 8;
    *reinterpret_cast<uint4*>(out + plane + o0) = make_uint4(pl0[0], pl0[1], pl0[2], pl0[3]);
    *reinterpret_cast<uint4*>(out + plane + o1) = make_uint4(pl1[0], pl1[1], pl1[2], pl1[3]);
  }
}


// ------------------------------------------------------------------------------------------ resampler x2 (+) concat (+) e_conv1, Texture net
// BASELINE config 4 (RenderNet_Texture_Face_Normal.py:155-179): the geometry grid (C = 1) and the decoded texture volume
// (C = 4) are resampled with the SAME pose, concatenated on the channel axis and fed to e_conv1 (5^3, stride 2, 5 -> 8).
// Unfused that is two gathers, a concat and a CUDA-core conv over a 128^3 x 5 fp32 grid (42 MB per render written and read
// back).  Fused exactly like resample_conv1_kernel: one CTA = 8^3 outputs, the 19^3 x 5 input points it needs are sampled
// into shared memory (one set of trilinear weights per point, five gathers per corner), tiles outside the rotated cube skip
// both the gather and the convolution, tiles that sampled only zeros skip the convolution.  Accumulation order per output =
// conv3d_direct_kernel<5,8,5>'s (ky, kx, kz, ci), so the result is bit-identical to the unfused chain.
constexpr int RC5_C = 5;
constexpr int RC5_TILE = RC_IN * RC_IN * RC_ZP;          // floats per channel plane of the input tile

__global__ void __launch_bounds__(256) resample5_conv1_kernel(const float* __restrict__ vox, const float* __restrict__ tex,
                                                              const float* __restrict__ minv, const float* __restrict__ w,
                                                              const float* __restrict__ bias, const float* __restrict__ alpha,
                                                              uint16_t* __restrict__ out, int B, int size, int nsz, int fmt,
                                                              int wy0, int wx0, int wh, int ww) {
  extern __shared__ __align__(16) float smem5[];
  float* tile = smem5;                                   // [5][19*19*20]
  float* ws = smem5 + RC5_C * RC5_TILE;                  // [125][5][8]
  const int tid = threadIdx.x;
  const int Ho = wh >> 1, Wo = ww >> 1, Do = nsz >> 1;
  const int tpy = Ho / RC_T, tpx = Wo / RC_T, tpz = Do / RC_T;
  int bid = blockIdx.x;
  const int tz = bid % tpz; bid /= tpz;
  const int tx = bid % tpx; bid /= tpx;
  const int ty = bid % tpy;
  const int b = bid / tpy;
  for (int i = tid; i < 125 * RC5_C * 8; i += 256) ws[i] = __ldg(w + i);

  const float* M = minv + b * 12;
  const float m00 = __ldg(M + 0), m01 = __ldg(M + 1), m02 = __ldg(M + 2), m03 = __ldg(M + 3);
  const float m10 = __ldg(M + 4), m11 = __ldg(M + 5), m12 = __ldg(M + 6), m13 = __ldg(M + 7);
  const float m20 = __ldg(M + 8), m21 = __ldg(M + 9), m22 = __ldg(M + 10), m23 = __ldg(M + 11);
  const float lim = static_cast<float>(size - 1);
  const size_t vol = static_cast<size_t>(size) * size * size;
  const float* vb = vox + static_cast<size_t>(b) * vol;
  const float* tb = tex + static_cast<size_t>(b) * vol * 4;
  const size_t sy = static_cast<size_t>(size), sz = static_cast<size_t>(size) * size;
  const int p0 = wy0 + 2 * ty * RC_T - 1, q0 = wx0 + 2 * tx * RC_T - 1, r0 = 2 * tz * RC_T - 1;

  int nonzero = 0;
  bool maybe_inside = true;
  {
    const float pl = static_cast<float>(max(p0, wy0)), ph = static_cast<float>(min(p0 + RC_IN - 1, wy0 + wh - 1));
    const float ql = static_cast<float>(max(q0, wx0)), qh = static_cast<float>(min(q0 + RC_IN - 1, wx0 + ww - 1));
    const float rl = static_cast<float>(max(r0, 0)), rh = static_cast<float>(min(r0 + RC_IN - 1, nsz - 1));
    const float gyl = static_cast<float>(nsz - 1) - ph, gyh = static_cast<float>(nsz - 1) - pl;
    const float mrow[3][4] = {{m00, m01, m02, m03}, {m10, m11, m12, m13}, {m20, m21, m22, m23}};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float lo = fminf(mrow[a][0] * rl, mrow[a][0] * rh) + fminf(mrow[a][1] * gyl, mrow[a][1] * gyh) +
                       fminf(mrow[a][2] * ql, mrow[a][2] * qh) + mrow[a][3];
      const float hi = fmaxf(mrow[a][0] * rl, mrow[a][0] * rh) + fmaxf(mrow[a][1] * gyl, mrow[a][1] * gyh) +
                       fmaxf(mrow[a][2] * ql, mrow[a][2] * qh) + mrow[a][3];
      if (hi < -0.01f || lo > lim + 0.01f) maybe_inside = false;
    }
  }
  if (maybe_inside) {
    int iz = tid % RC_IN, row = tid / RC_IN;
    for (int i = tid; i < RC_IN * RC_IN * RC_IN; i += 256) {
      const int iy = row / RC_IN, ix = row - iy * RC_IN;
      const int p = p0 + iy, q = q0 + ix, r = r0 + iz;
      float v[RC5_C] = {0.f, 0.f, 0.f, 0.f, 0.f};
      if (p >= wy0 && p < wy0 + wh && q >= wx0 && q < wx0 + ww && r >= 0 && r < nsz) {   // SAME zeros at the window border
        const float gx = static_cast<float>(r), gy = static_cast<float>(nsz - 1 - p), gz = static_cast<float>(q);
        const float x = sample_coord(m00, m01, m02, m03, gx, gy, gz);
        const float y = sample_coord(m10, m11, m12, m13, gx, gy, gz);
        const float z = sample_coord(m20, m21, m22, m23, gx, gy, gz);
        if (x >= 0.f && x < lim && y >= 0.f && y < lim && z >= 0.f && z < lim) {
          const float x0f = floorf(x), y0f = floorf(y), z0f = floorf(z);
          const int x0 = static_cast<int>(x0f), y0 = static_cast<int>(y0f), z0 = static_cast<int>(z0f);
          const float x1f = x0f + 1.f, y1f = y0f + 1.f, z1f = z0f + 1.f;
          const float ax = __fsub_rn(x1f, x), bxw = __fsub_rn(x, x0f);
          const float ay = __fsub_rn(y1f, y), byw = __fsub_rn(y, y0f);
          const float az = __fsub_rn(z1f, z), bzw = __fsub_rn(z, z0f);
          const float wgt[8] = {__fmul_rn(__fmul_rn(ax, ay), az), __fmul_rn(__fmul_rn(ax, byw), az),
                                __fmul_rn(__fmul_rn(bxw, ay), az), __fmul_rn(__fmul_rn(bxw, byw), az),
                                __fmul_rn(__fmul_rn(ax, ay), bzw), __fmul_rn(__fmul_rn(ax, byw), bzw),
                                __fmul_rn(__fmul_rn(bxw, ay), bzw), __fmul_rn(__fmul_rn(bxw, byw), bzw)};
          const size_t c000 = (static_cast<size_t>(z0) * size + y0) * size + x0;
          const size_t off[8] = {c000, c000 + sy, c000 + 1, c000 + sy + 1, c000 + sz, c000 + sz + sy, c000 + sz + 1,
                                 c000 + sz + sy + 1};                                   // corners a..h (:440-449)
          float s = __fmul_rn(wgt[0], __ldg(vb + off[0]));                              // add_n order a..h (:485)
#pragma unroll
          for (int k = 1; k < 8; ++k) s = __fadd_rn(s, __fmul_rn(wgt[k], __ldg(vb + off[k])));
          v[0] = s;
          float4 t4 = __ldg(reinterpret_cast<const float4*>(tb) + off[0]);
          float t0 = __fmul_rn(wgt[0], t4.x), t1 = __fmul_rn(wgt[0], t4.y), t2 = __fmul_rn(wgt[0], t4.z), t3 = __fmul_rn(wgt[0], t4.w);
#pragma unroll
          for (int k = 1; k < 8; ++k) {
            t4 = __ldg(reinterpret_cast<const float4*>(tb) + off[k]);
            t0 = __fadd_rn(t0, __fmul_rn(wgt[k], t4.x)); t1 = __fadd_rn(t1, __fmul_rn(wgt[k], t4.y));
            t2 = __fadd_rn(t2, __fmul_rn(wgt[k], t4.z)); t3 = __fadd_rn(t3, __fmul_rn(wgt[k], t4.w));
          }
          v[1] = t0; v[2] = t1; v[3] = t2; v[4] = t3;
        }
      }
      const int ti = row * RC_ZP + (iz & 1) * 10 + (iz >> 1);
#pragma unroll
      for (int c = 0; c < RC5_C; ++c) {
        nonzero |= (v[c] != 0.f);
        tile[c * RC5_TILE + ti] = v[c];
      }
      iz += 256 % RC_IN;
      row += 256 / RC_IN;
      if (iz >= RC_IN) { iz -= RC_IN; ++row; }
    }
  }
  const int any = __syncthreads_or(nonzero);

  const int oz = tid & 7, ox = (tid >> 3) & 7, oy = tid >> 6;   // second output: oy + 4
  float acc0[8], acc1[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc0[c] = acc1[c] = 0.f;
  if (any) {
    for (int ky = 0; ky < 5; ++ky) {
      for (int kx = 0; kx < 5; ++kx) {
        const float* t0 = tile + ((2 * oy + ky) * RC_IN + (2 * ox + kx)) * RC_ZP + oz;
        const float* t1 = t0 + 8 * RC_IN * RC_ZP;
        const float* wk = ws + (ky * 5 + kx) * 5 * RC5_C * 8;
#pragma unroll
        for (int kz = 0; kz < 5; ++kz) {
          const int zi = (kz & 1) * 10 + (kz >> 1);
#pragma unroll
          for (int c = 0; c < RC5_C; ++c) {
            const float a0 = t0[c * RC5_TILE + zi], a1 = t1[c * RC5_TILE + zi];
            const float4 wlo = *reinterpret_cast<const float4*>(wk + (kz * RC5_C + c) * 8);
            const float4 whi = *reinterpret_cast<const float4*>(wk + (kz * RC5_C + c) * 8 + 4);
            acc0[0] = fmaf(a0, wlo.x, acc0[0]); acc0[1] = fmaf(a0, wlo.y, acc0[1]);
            acc0[2] = fmaf(a0, wlo.z, acc0[2]); acc0[3] = fmaf(a0, wlo.w, acc0[3]);
            acc0[4] = fmaf(a0, whi.x, acc0[4]); acc0[5] = fmaf(a0, whi.y, acc0[5]);
            acc0[6] = fmaf(a0, whi.z, acc0[6]); acc0[7] = fmaf(a0, whi.w, acc0[7]);
            acc1[0] = fmaf(a1, wlo.x, acc1[0]); acc1[1] = fmaf(a1, wlo.y, acc1[1]);
            acc1[2] = fmaf(a1, wlo.z, acc1[2]); acc1[3] = fmaf(a1, wlo.w, acc1[3]);
            acc1[4] = fmaf(a1, whi.x, acc1[4]); acc1[5] = fmaf(a1, whi.y, acc1[5]);
            acc1[6] = fmaf(a1, whi.z, acc1[6]); acc1[7] = fmaf(a1, whi.w, acc1[7]);
          }
        }
      }
    }
  }
  uint32_t pk0[4], pk1[4], pl0[4], pl1[4];
#pragma unroll
  for (int c = 0; c < 8; c += 2) {
    const float b0 = __ldg(bias + c), b1 = __ldg(bias + c + 1);
    float u0 = acc0[c] + b0, u1 = acc0[c + 1] + b1, v0 = acc1[c] + b0, v1 = acc1[c + 1] + b1;
    if (alpha != nullptr) {
      const float al0 = __ldg(alpha + c), al1 = __ldg(alpha + c + 1);
      u0 = fmaxf(u0, 0.f) + al0 * fminf(u0, 0.f);
      u1 = fmaxf(u1, 0.f) + al1 * fminf(u1, 0.f);
      v0 = fmaxf(v0, 0.f) + al0 * fminf(v0, 0.f);
      v1 = fmaxf(v1, 0.f) + al1 * fminf(v1, 0.f);
    }
    pack16x2(u0, u1, fmt, &pk0[c / 2], &pl0[c / 2]);
    pack16x2(v0, v1, fmt, &pk1[c / 2], &pl1[c / 2]);
  }
  const size_t o0 = (((static_cast<size_t>(b) * Ho + (ty * RC_T + oy)) * Wo + (tx * RC_T + ox)) * Do + (tz * RC_T + oz)) * 8;
  const size_t o1 = o0 + static_cast<size_t>(4) * Wo * Do * 8;
  *reinterpret_cast<uint4*>(out + o0) = make_uint4(pk0[0], pk0[1], pk0[2], pk0[3]);
  *reinterpret_cast<uint4*>(out + o1) = make_uint4(pk1[0], pk1[1], pk1[2], pk1[3]);
  if (fmt == 2) {
    const size_t plane = static_cast<size_t>(B) * Ho * Wo * Do * 8;
    *reinterpret_cast<uint4*>(out + plane + o0) = make_uint4(pl0[0], pl0[1], pl0[2], pl0[3]);
    *reinterpret_cast<uint4*>(out + plane + o1) = make_uint4(pl1[0], pl1[1], pl1[2], pl1[3]);
  }
}


// ------------------------------------------------------------------------------------------ texture decoder (config 4)
// fully_connected (tools/layer_util.py:311-343): y[b][n] = act(sum_k x[b][k] w[k][n] + bias[n]); w is TF [in,out].
// One thread per output column, weights streamed once (coalesced across n), x staged in shared memory.
template <int BMAX>
__global__ void __launch_bounds__(256) fc_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                 const float* __restrict__ bias, const float* __restrict__ alpha,
                                                 uint16_t* __restrict__ out16, float* __restrict__ out32, int B, int K,
                                                 int N, int fmt) {
  extern __shared__ float xs[];  // [B][K]
  for (int i = threadIdx.x; i < B * K; i += blockDim.x) xs[i] = x[i];
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float acc[BMAX];
#pragma unroll
  for (int b = 0; b < BMAX; ++b) acc[b] = 0.f;
  for (int k = 0; k < K; ++k) {
    const float wv = __ldg(w + static_cast<size_t>(k) * N + n);
#pragma unroll
    for (int b = 0; b < BMAX; ++b)
      if (b < B) acc[b] = fmaf(xs[b * K + k], wv, acc[b]);
  }
  const float bv = bias != nullptr ? __ldg(bias + n) : 0.f;
  const float av = alpha != nullptr ? __ldg(alpha + n) : 1.f;
#pragma unroll
  for (int b = 0; b < BMAX; ++b) {
    if (b < B) {
      float v = acc[b] + bv;
      if (alpha != nullptr) v = fmaxf(v, 0.f) + av * fminf(v, 0.f);
      const size_t o = static_cast<size_t>(b) * N + n;
      if (out32 != nullptr) out32[o] = v;
      if (out16 != nullptr) store16(out16, o, v, fmt, static_cast<long long>(B) * N);
    }
  }
}

// Thin 3-D (transposed) convolution with tiny channel counts (<= 8), TF SAME, + bias + PReLU; fp32 or 16-bit in,
// 16-bit and/or fp32 out.  One thread per output voxel.  transposed: out[o] += x[i] w[k][co][ci], o = i*s + k - pb
// (tools/layer_util.py:269-309); forward: out[o] = sum x[o*s + k - pb] w[k][ci][co] (:228-265).
template <int CIN, int COUT>
__global__ void __launch_bounds__(256) conv3d_small_kernel(const void* __restrict__ xv, int x_is_f32,
                                                           const float* __restrict__ w, const float* __restrict__ bias,
                                                           const float* __restrict__ alpha, uint16_t* __restrict__ out16,
                                                           float* __restrict__ out32, int B, int H, int W, int D, int Ho,
                                                           int Wo, int Do, int K, int s, int pb, int transposed, int fmt) {
  extern __shared__ float wsm[];  // K^3 * CIN * COUT
  const int nw = K * K * K * CIN * COUT;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) wsm[i] = w[i];
  __syncthreads();
  const long long total = static_cast<long long>(B) * Ho * Wo * Do;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int oz = static_cast<int>(idx % Do);
  const int ox = static_cast<int>((idx / Do) % Wo);
  const int oy = static_cast<int>((idx / (static_cast<long long>(Do) * Wo)) % Ho);
  const int b = static_cast<int>(idx / (static_cast<long long>(Do) * Wo * Ho));
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  for (int ky = 0; ky < K; ++ky) {
    int iy;
    if (transposed) { const int n = oy + pb - ky; if (n < 0 || n % s != 0) continue; iy = n / s; }
    else iy = oy * s + ky - pb;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < K; ++kx) {
      int ix;
      if (transposed) { const int n = ox + pb - kx; if (n < 0 || n % s != 0) continue; ix = n / s; }
      else ix = ox * s + kx - pb;
      if (ix < 0 || ix >= W) continue;
      for (int kz = 0; kz < K; ++kz) {
        int iz;
        if (transposed) { const int n = oz + pb - kz; if (n < 0 || n % s != 0) continue; iz = n / s; }
        else iz = oz * s + kz - pb;
        if (iz < 0 || iz >= D) continue;
        const size_t xi = (((static_cast<size_t>(b) * H + iy) * W + ix) * D + iz) * CIN;
        float xin[CIN];
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) {
          if (x_is_f32) xin[ci] = __ldg(static_cast<const float*>(xv) + xi + ci);
          else xin[ci] = load16(static_cast<const uint16_t*>(xv), xi + ci, fmt, static_cast<long long>(B) * H * W * D * CIN);
        }
        const float* wt = wsm + ((ky * K + kx) * K + kz) * CIN * COUT;
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci)
#pragma unroll
          for (int co = 0; co < COUT; ++co)
            acc[co] = fmaf(xin[ci], transposed ? wt[co * CIN + ci] : wt[ci * COUT + co], acc[co]);
      }
    }
  }
#pragma unroll
  for (int co = 0; co < COUT; ++co) {
    float v = acc[co] + (bias != nullptr ? __ldg(bias + co) : 0.f);
    if (alpha != nullptr) v = fmaxf(v, 0.f) + __ldg(alpha + co) * fminf(v, 0.f);
    const size_t o = static_cast<size_t>(idx) * COUT + co;
    if (out32 != nullptr) out32[o] = v;
    if (out16 != nullptr) store16(out16, o, v, fmt, total * COUT);
  }
}

// The texture decoder's last layer (conv3d 4^3, 8 -> 4, stride 1, SAME = pad 1 before / 2 after, + bias + PReLU on a 64^3 grid;
// RenderNet_Texture_Face_Normal.py:44-45) is 0.54 GMAC per render: 3.4 ms per B=24 step in the generic one-thread-per-voxel
// kernel above, 20 % of the fast-precision Texture step.  Tiled version: one CTA = 8^3 outputs, the 11^3 x 8 input tile is staged
// channel-planar in shared memory (z rows padded to 12 floats), the filter too; each thread computes two outputs x 4 channels.
// Same (ky, kx, kz, ci) accumulation order as conv3d_small_kernel<8,4>: bit-identical results.
constexpr int T4_IN = 11, T4_ZP = 12, T4_PLANE = T4_IN * T4_IN * T4_ZP;
__global__ void __launch_bounds__(256) conv3d_k4_8to4_tiled_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                   const float* __restrict__ bias, const float* __restrict__ alpha,
                                                                   float* __restrict__ out, int B, int H, int W, int D) {
  extern __shared__ __align__(16) float sm4[];
  float* tile = sm4;                       // [8][11][11][12]
  float* ws = sm4 + 8 * T4_PLANE;          // [64 taps][8 ci][4 co]
  const int tid = threadIdx.x;
  const int tz = D / 8, tx = W / 8, ty = H / 8;
  int bid = blockIdx.x;
  const int bz = bid % tz; bid /= tz;
  const int bxx = bid % tx; bid /= tx;
  const int byy = bid % ty;
  const int b = bid / ty;
  for (int i = tid; i < 64 * 32; i += 256) ws[i] = __ldg(w + i);
  const int y0 = byy * 8 - 1, x0 = bxx * 8 - 1, z0 = bz * 8 - 1;       // SAME: pad-before 1
  for (int i = tid; i < T4_IN * T4_IN * T4_IN; i += 256) {
    const int iz = i % T4_IN, ix = (i / T4_IN) % T4_IN, iy = i / (T4_IN * T4_IN);
    const int gy = y0 + iy, gx = x0 + ix, gz = z0 + iz;
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W && gz >= 0 && gz < D) {
      const float4* px = reinterpret_cast<const float4*>(x + ((((static_cast<size_t>(b) * H + gy) * W + gx) * D + gz) * 8));
      lo = __ldg(px); hi = __ldg(px + 1);
    }
    const int o = (iy * T4_IN + ix) * T4_ZP + iz;
    tile[0 * T4_PLANE + o] = lo.x; tile[1 * T4_PLANE + o] = lo.y; tile[2 * T4_PLANE + o] = lo.z; tile[3 * T4_PLANE + o] = lo.w;
    tile[4 * T4_PLANE + o] = hi.x; tile[5 * T4_PLANE + o] = hi.y; tile[6 * T4_PLANE + o] = hi.z; tile[7 * T4_PLANE + o] = hi.w;
  }
  __syncthreads();
  const int oz = tid & 7, ox = (tid >> 3) & 7, oy = tid >> 6;            // second output: oy + 4
  float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
  for (int ky = 0; ky < 4; ++ky)
    for (int kx = 0; kx < 4; ++kx) {
      const float* t0 = tile + ((oy + ky) * T4_IN + (ox + kx)) * T4_ZP + oz;
      const float* t1 = t0 + 4 * T4_IN * T4_ZP;
      const float4* wk = reinterpret_cast<const float4*>(ws + (ky * 4 + kx) * 4 * 32);
#pragma unroll
      for (int kz = 0; kz < 4; ++kz)
#pragma unroll
        for (int ci = 0; ci < 8; ++ci) {
          const float u = t0[ci * T4_PLANE + kz], v = t1[ci * T4_PLANE + kz];
          const float4 w4 = wk[kz * 8 + ci];
          a0[0] = fmaf(u, w4.x, a0[0]); a0[1] = fmaf(u, w4.y, a0[1]); a0[2] = fmaf(u, w4.z, a0[2]); a0[3] = fmaf(u, w4.w, a0[3]);
          a1[0] = fmaf(v, w4.x, a1[0]); a1[1] = fmaf(v, w4.y, a1[1]); a1[2] = fmaf(v, w4.z, a1[2]); a1[3] = fmaf(v, w4.w, a1[3]);
        }
    }
  float r0[4], r1[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float bv = bias != nullptr ? __ldg(bias + c) : 0.f;
    r0[c] = a0[c] + bv; r1[c] = a1[c] + bv;
    if (alpha != nullptr) {
      const float al = __ldg(alpha + c);
      r0[c] = fmaxf(r0[c], 0.f) + al * fminf(r0[c], 0.f);
      r1[c] = fmaxf(r1[c], 0.f) + al * fminf(r1[c], 0.f);
    }
  }
  const size_t o0 = (((static_cast<size_t>(b) * H + (byy * 8 + oy)) * W + (bxx * 8 + ox)) * D + (bz * 8 + oz)) * 4;
  *reinterpret_cast<float4*>(out + o0) = make_float4(r0[0], r0[1], r0[2], r0[3]);
  *reinterpret_cast<float4*>(out + o0 + static_cast<size_t>(4) * W * D * 4) = make_float4(r1[0], r1[1], r1[2], r1[3]);
}

// channel concat of two fp32 channel-last tensors: out[..., 0:Ca] = a, out[..., Ca:Ca+Cb] = b
__global__ void concat_channels_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                                       long long n, int Ca, int Cb) {
  const int C = Ca + Cb;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n * C;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / C;
    const int c = static_cast<int>(i % C);
    out[i] = c < Ca ? a[p * Ca + c] : b[p * Cb + (c - Ca)];
  }
}


// ------------------------------------------------------------------------------------------ x-folded thin transposed conv
// Stride-1 SAME transposed conv (o = i + k - pb) with few channels, re-expressed over F-pixel groups:
// x = F*q + r, x' = F*q' + p.  Rows of the GEMM are pixel groups q, K = (p, ci) = F*Cin, N = (r, co) = F*Cout, taps are
// (ky, dq) with dq in {-1,0,1}:  Wf[ky][dq+1][r*Cout+co][p*Cin+ci] = w[ky][kx][co][ci], kx = pb - (F*dq + p - r), or 0
// when kx is outside the filter.  TMA then moves 128-byte rows and kw taps collapse into 3.
__global__ void pack_xfold_kernel(const float* __restrict__ w, uint16_t* __restrict__ packed, int kh, int kw, int Cin,
                                  int Cout, int F, int cout_pad, int fmt) {
  const int K = F * Cin, N = F * Cout, pb = (kw - 1) / 2;
  const long long total = static_cast<long long>(kh) * 3 * cout_pad * K;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const int n = static_cast<int>((i / K) % cout_pad);
    const int t = static_cast<int>(i / (static_cast<long long>(K) * cout_pad));
    const int ky = kh - 1 - t / 3, dq = t % 3 - 1;   // taps stored ky-reversed so that dy = pby - ky increases with t/3
    float v = 0.f;
    if (n < N) {
      const int p = k / Cin, ci = k % Cin, r = n / Cout, co = n % Cout;
      const int kx = pb - (F * dq + p - r);
      if (kx >= 0 && kx < kw) v = w[((static_cast<long long>(ky) * kw + kx) * Cout + co) * Cin + ci];
    }
    store16(packed, i, v, fmt, total);
  }
}


// ------------------------------------------------------------------------------------------ merged-phase transposed conv
// k = 4, stride 2, SAME (pb = 1): o = 2*i + k - 1.  Output (2y+ay, 2x+ax) reads input (y+dy, x+dx) through filter tap
// ky = ay + 1 - 2*dy (kx likewise) when that lies in [0,4): (ay,dy) in {(0,0)->1, (0,-1)->3, (1,1)->0, (1,0)->2}.
// Wm[(dy+1)*3 + (dx+1)][(ay*2+ax)*Cout + co][ci].
__global__ void pack_tconv_s2_merged_kernel(const float* __restrict__ w, uint16_t* __restrict__ packed, int Cin, int Cout,
                                            int fmt) {
  const int N = 4 * Cout;
  const long long total = 9LL * N * Cin;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % Cin);
    const int n = static_cast<int>((i / Cin) % N);
    const int t = static_cast<int>(i / (static_cast<long long>(Cin) * N));
    const int dy = t / 3 - 1, dx = t % 3 - 1;
    const int ay = n / (2 * Cout), ax = (n / Cout) % 2, co = n % Cout;
    const int ky = ay + 1 - 2 * dy, kx = ax + 1 - 2 * dx;
    float v = 0.f;
    if (ky >= 0 && ky < 4 && kx >= 0 && kx < 4) v = w[((static_cast<long long>(ky) * 4 + kx) * Cout + co) * Cin + ci];
    store16(packed, i, v, fmt, total);
  }
}

// ------------------------------------------------------------------------------------------ binvox RLE decode
// tools/binvox_rw.py:84-93 on the device (SURVEY §8 f-2): the payload is (value, count) byte pairs; the reference
// expands them with np.repeat, reshapes to dims (x, z, y order) and transposes (0, 2, 1).  Here the 6-12 KB payload is
// uploaded as is (plus the exclusive prefix sum of the counts, computed on the host over <= a few thousand runs) and
// each output voxel binary-searches its run: out[b][a][b'][c] = value(run containing flat index (a*d1 + c)*d2 + b').
__global__ void binvox_decode_kernel(const uint8_t* __restrict__ pairs, const int* __restrict__ run_start,
                                     const int* __restrict__ item_first_run, float* __restrict__ out, int n_items,
                                     int d0, int d1, int d2, int fix_coords) {
  const long long per = static_cast<long long>(d0) * d1 * d2;
  const long long total = per * n_items;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int item = static_cast<int>(i / per);
    const int o = static_cast<int>(i - item * per);
    int f = o;
    if (fix_coords) {       // output [a][b][c] (extents d0, d2, d1) reads stored [a][c][b]
      const int c = o % d1, b = (o / d1) % d2, a = o / (d1 * d2);
      f = (a * d1 + c) * d2 + b;
    }
    int lo = __ldg(item_first_run + item), hi = __ldg(item_first_run + item + 1);   // runs [lo, hi) of this item
    const int* rs = run_start;                                                     // starts are item-relative
    while (hi - lo > 1) {    // last run r with run_start[r] <= f (zero-length runs are skipped by construction)
      const int mid = (lo + hi) >> 1;
      if (__ldg(rs + mid) <= f) lo = mid; else hi = mid;
    }
    out[i] = __ldg(pairs + 2 * static_cast<size_t>(lo)) != 0 ? 1.f : 0.f;
  }
}

// ------------------------------------------------------------------------------------------ Phong
// The one Phong pass (rn_phong_shade; rn_phong_composite is its NumPy-composite, no-albedo case).  One thread per pixel,
// blockIdx.y = batch item.  shade = phong_pixel (TF = false) or tf_phong_pixel (TF = true); compos = albedo * shade, or shade
// itself without an albedo; each of shade_f32, compos_f32 and compos_u8 (= clip(255 compos) truncated) may be NULL.
// PA (rn_phong_shade_ambient): the item's ambient term is loaded from ambient_b[b] instead of passed; the arithmetic is the same.
template <bool TF, bool PA>
__global__ void __launch_bounds__(256) phong_shade_kernel(const float* __restrict__ normal, const float* __restrict__ albedo,
                                                          const float* __restrict__ light_dir, const float* __restrict__ light_col,
                                                          float ambient, float k_diffuse, int white, int with_mask,
                                                          float* __restrict__ shade_f32, float* __restrict__ compos_f32,
                                                          uint8_t* __restrict__ compos_u8, int HW, const float* __restrict__ ambient_b) {
  const int b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  if constexpr (PA) ambient = __ldg(ambient_b + b);
  const size_t o = (static_cast<size_t>(b) * HW + p) * 3;
  const float l0 = __ldg(light_dir + 3 * b), l1 = __ldg(light_dir + 3 * b + 1), l2 = __ldg(light_dir + 3 * b + 2);
  const float col[3] = {__ldg(light_col + 3 * b), __ldg(light_col + 3 * b + 1), __ldg(light_col + 3 * b + 2)};
  const float n0 = normal[o], n1 = normal[o + 1], n2 = normal[o + 2];
  float s[3];
  if constexpr (TF) {
    const float lnorm = sqrtf(l0 * l0 + l1 * l1 + l2 * l2);                // as phong_recon_loss_grad_kernel normalises it
    const float L[3] = {l0 / lnorm, l1 / lnorm, l2 / lnorm};
    tf_phong_pixel(n0, n1, n2, L, col, ambient, k_diffuse, !white, with_mask, s);
  } else {
    phong_pixel(n0, n1, n2, l0, l1, l2, col, ambient, k_diffuse, white, with_mask, s);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = albedo != nullptr ? albedo[o + c] * s[c] : s[c];
    if (shade_f32 != nullptr) shade_f32[o + c] = s[c];
    if (compos_f32 != nullptr) compos_f32[o + c] = v;
    if (compos_u8 != nullptr) compos_u8[o + c] = phong_u8(v);
  }
}

static inline int grid_for(long long n, int block, int cap = 132 * 32) {
  long long g = (n + block - 1) / block;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

static void same_pad(int n_in, int k, int s, int* n_out, int* pb) {
  *n_out = (n_in + s - 1) / s;
  int total = (*n_out - 1) * s + k - n_in;
  if (total < 0) total = 0;
  *pb = total / 2;
}

}  // namespace rn

using namespace rn;

extern "C" int rn_version(void) { return 100; }

extern "C" const char* rn_error_string(int code) {
  if (code == 0) return "ok";
  if (code < 0) return "rendernet_b200: invalid argument";
  if (code >= 1000) return "rendernet_b200: cuTensorMapEncodeTiled failed";
  return cudaGetErrorString(static_cast<cudaError_t>(code));
}

// the rows [y0, y0+ph) x columns [x0, x0+pw) of the new_size^2 rows per item
static int resample_launch(const float* vox, const float* minv, float* out, int B, int C, int size, int new_size, int transform,
                           int y0, int x0, int ph, int pw, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = static_cast<long long>(B) * ph * pw;
  const int block = 256;
  const int grid = static_cast<int>((rows * 32 + block - 1) / block);
  switch (C) {
    case 1: resample_kernel<1><<<grid, block, 0, st>>>(vox, minv, out, B, size, new_size, transform, y0, x0, ph, pw); break;
    case 2: resample_kernel<2><<<grid, block, 0, st>>>(vox, minv, out, B, size, new_size, transform, y0, x0, ph, pw); break;
    case 3: resample_kernel<3><<<grid, block, 0, st>>>(vox, minv, out, B, size, new_size, transform, y0, x0, ph, pw); break;
    case 4: resample_kernel<4><<<grid, block, 0, st>>>(vox, minv, out, B, size, new_size, transform, y0, x0, ph, pw); break;
    default: return -2;
  }
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

// A patch window of the axis-transformed grid: ph, pw multiples of 16 (8^3-output tiles of the stride-2 e_conv1) inside
// [0, new_size).  Shared by every *_window entry point.
static bool window_ok(int new_size, int y0, int x0, int ph, int pw) {
  return ph >= 16 && pw >= 16 && ph % 16 == 0 && pw % 16 == 0 && y0 >= 0 && x0 >= 0 && y0 <= new_size - ph &&
         x0 <= new_size - pw;
}

extern "C" int rn_resample_f32(const float* vox, const float* minv, float* out, int B, int C, int size, int new_size,
                               int transform, void* stream) {
  if (!vox || !minv || !out || B < 1 || size < 2 || new_size < 1) return -1;
  return resample_launch(vox, minv, out, B, C, size, new_size, transform, 0, 0, new_size, new_size, stream);
}

extern "C" int rn_resample_window_f32(const float* vox, const float* minv, float* out, int B, int C, int size, int new_size,
                                      int y0, int x0, int ph, int pw, void* stream) {
  if (!vox || !minv || !out || B < 1 || size < 2 || new_size < 16) return -1;
  if ((C != 1 && C != 4) || !window_ok(new_size, y0, x0, ph, pw)) return -2;
  return resample_launch(vox, minv, out, B, C, size, new_size, 1, y0, x0, ph, pw, stream);
}

// plane: element offset of the LO plane for fmt 2 (0 = right after this call's own output)
static int pack_conv_weights_impl(const float* w, void* packed, int ntaps_total, int Cin, int Cout, int cout_pad,
                                  int transposed, const int* tap_sel, int n_sel, int fmt, long long plane, void* stream) {
  if (!w || !packed || Cin < 1 || Cout < 1 || cout_pad < Cout || fmt < 0 || fmt > 2) return -1;
  TapSel sel;
  if (tap_sel == nullptr) {
    if (ntaps_total > 64) return -2;
    sel.n = ntaps_total;
    for (int i = 0; i < ntaps_total; ++i) sel.idx[i] = i;
  } else {
    if (n_sel > 64 || n_sel < 1) return -2;
    sel.n = n_sel;
    for (int i = 0; i < n_sel; ++i) {
      if (tap_sel[i] < 0 || tap_sel[i] >= ntaps_total) return -3;
      sel.idx[i] = tap_sel[i];
    }
  }
  const long long total = static_cast<long long>(sel.n) * cout_pad * Cin;
  pack_weights_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, static_cast<uint16_t*>(packed), Cin, Cout, cout_pad, transposed, sel, fmt, plane > 0 ? plane : total);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_interpolate_f32(const float* vox, const float* x, const float* y, const float* z, float* out, int B, int C,
                                  int size, long long n_per_item, void* stream) {
  if (!vox || !x || !y || !z || !out || B < 1 || C < 1 || size < 2 || n_per_item < 1) return -1;
  const long long n = static_cast<long long>(B) * n_per_item;
  const long long blocks = (n + 255) / 256;
  if (blocks > 0x7fffffffLL) return -2;
  interpolate_kernel<<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(vox, x, y, z, out, n, n_per_item, C,
                                                                                         size);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_pack_conv_weights(const float* w, void* packed, int ntaps_total, int Cin, int Cout, int cout_pad,
                                    int transposed, const int* tap_sel, int n_sel, int fmt, void* stream) {
  return pack_conv_weights_impl(w, packed, ntaps_total, Cin, Cout, cout_pad, transposed, tap_sel, n_sel, fmt, 0, stream);
}

extern "C" int rn_cast_f32_to_16(const float* src, void* dst, long long n, long long n_pad, int fmt, void* stream) {
  if (!src || !dst || n < 0 || n_pad < n) return -1;
  if (n_pad == 0) return 0;
  cast_f32_to_16_kernel<<<grid_for(n_pad, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, static_cast<uint16_t*>(dst), n, n_pad, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_cast_16_to_f32(const void* src, float* dst, long long n, int fmt, void* stream) {
  if (!src || !dst || n < 0) return -1;
  if (n == 0) return 0;
  cast_16_to_f32_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(src), dst, n, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}


extern "C" int rn_bias_act_16(const void* x, const float* bias, const float* alpha, int act, const void* residual,
                              void* out16, float* out32, long long n, int C, int fmt, void* stream) {
  if (!x || (!out16 && !out32) || n < 0 || C < 1 || (act == 1 && !alpha)) return -1;
  if (n == 0) return 0;
  bias_act_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(x), bias, alpha, act, static_cast<const uint16_t*>(residual),
      static_cast<uint16_t*>(out16), out32, n, C, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------- igemm wrappers
static void apply_tuning(rn_conv_desc& d, const rn_tuning* t) {
  if (t == nullptr) return;
  d.cluster = t->cluster; d.cta_group = t->cta_group; d.force_kps = t->kps; d.msub = t->msub;
  d.epi_groups = t->epilogue_groups; d.res_prefetch = t->res_prefetch; d.tma_store = t->tma_store;
}
static bool want_yhalo(const rn_tuning* t) { return (t != nullptr && t->yhalo != 0) ? t->yhalo > 0 : tuning().yhalo != 0; }

extern "C" int rn_conv2d_same_scaled(const void* x, const void* w_packed, const float* w_unscale, const float* bias,
                                     const float* alpha, int act, const void* residual, int residual_is_f32, void* out16,
                                     float* out32, int B, int H, int W, int Cin, int Cout, int cout_pad, int kh, int kw,
                                     int fmt, const rn_tuning* tune, void* stream) {
  if (kh * kw > kMaxTaps || kh < 1 || kw < 1) return -20;
  int8_t taps[kMaxTaps * 3];
  const int pby = (kh - 1) / 2, pbx = (kw - 1) / 2;  // SAME, stride 1: before = (k-1)//2
  for (int ky = 0; ky < kh; ++ky)
    for (int kx = 0; kx < kw; ++kx) {
      int8_t* t = taps + 3 * (ky * kw + kx);
      t[0] = static_cast<int8_t>(kx - pbx); t[1] = static_cast<int8_t>(ky - pby); t[2] = 0;
    }
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 2; d.B = B; d.H = H; d.W = W; d.D = 1; d.Cin = Cin; d.Cout = Cout; d.cout_pad = cout_pad;
  d.ntaps = kh * kw; d.taps = taps; d.x = x; d.w_packed = w_packed; d.bias = bias; d.alpha = alpha; d.act = act;
  d.residual = residual; d.residual_is_f32 = residual_is_f32; d.out16 = out16; d.out32 = out32;
  d.o_base = 0; d.o_x = Cout; d.o_y = static_cast<long long>(W) * Cout; d.o_b = static_cast<long long>(H) * W * Cout;
  d.o_z = 0; d.fmt = fmt;
  if (fmt == 2) {   // fp16 hi/lo pairs: [2][numel]
    d.x_plane = static_cast<long long>(B) * H * W * Cin;
    d.w_plane = static_cast<long long>(kh) * kw * cout_pad * Cin;
    d.o_plane = static_cast<long long>(B) * H * W * Cout;
  }
  d.w_unscale = w_unscale;
  apply_tuning(d, tune);
  if (kh == 3 && Cin % 64 == 0 && want_yhalo(tune)) d.ny = 3;   // taps are already ordered ky*kw + kx with dy = ky - 1
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_conv2d_same(const void* x, const void* w_packed, const float* bias, const float* alpha, int act,
                              const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H,
                              int W, int Cin, int Cout, int cout_pad, int kh, int kw, int fmt, const rn_tuning* tune,
                              void* stream) {
  return rn_conv2d_same_scaled(x, w_packed, nullptr, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, Cin,
                               Cout, cout_pad, kh, kw, fmt, tune, stream);
}

extern "C" int rn_conv3d_same_scaled(const void* x, const void* w_packed, const float* w_unscale, const float* bias,
                                     const float* alpha, int act, const void* residual, int residual_is_f32, void* out16,
                                     float* out32, int B, int H, int W, int D, int Cin, int Cout, int cout_pad, int k,
                                     int fmt, const rn_tuning* tune, void* stream) {
  if (k * k * k > kMaxTaps || k < 1) return -20;
  int8_t taps[kMaxTaps * 3];
  const int pb = (k - 1) / 2;
  for (int k0 = 0; k0 < k; ++k0)
    for (int k1 = 0; k1 < k; ++k1)
      for (int k2 = 0; k2 < k; ++k2) {
        int8_t* t = taps + 3 * ((k0 * k + k1) * k + k2);  // TF filter [k0,k1,k2,..] over axes (H, W, D)
        t[0] = static_cast<int8_t>(k1 - pb); t[1] = static_cast<int8_t>(k0 - pb); t[2] = static_cast<int8_t>(k2 - pb);
      }
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 3; d.B = B; d.H = H; d.W = W; d.D = D; d.Cin = Cin; d.Cout = Cout; d.cout_pad = cout_pad;
  d.ntaps = k * k * k; d.taps = taps; d.x = x; d.w_packed = w_packed; d.bias = bias; d.alpha = alpha; d.act = act;
  d.residual = residual; d.residual_is_f32 = residual_is_f32; d.out16 = out16; d.out32 = out32;
  d.o_base = 0; d.o_z = Cout; d.o_x = static_cast<long long>(D) * Cout; d.o_y = static_cast<long long>(W) * D * Cout;
  d.o_b = static_cast<long long>(H) * W * D * Cout; d.fmt = fmt;
  if (fmt == 2) {
    d.x_plane = static_cast<long long>(B) * H * W * D * Cin;
    d.w_plane = static_cast<long long>(k) * k * k * cout_pad * Cin;
    d.o_plane = static_cast<long long>(B) * H * W * D * Cout;
  }
  d.w_unscale = w_unscale;
  apply_tuning(d, tune);
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_conv3d_same(const void* x, const void* w_packed, const float* bias, const float* alpha, int act,
                              const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H,
                              int W, int D, int Cin, int Cout, int cout_pad, int k, int fmt, const rn_tuning* tune,
                              void* stream) {
  return rn_conv3d_same_scaled(x, w_packed, nullptr, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, D,
                               Cin, Cout, cout_pad, k, fmt, tune, stream);
}

// Transposed SAME conv: o = i*s + kk - pb, pb = max(k-s,0)/2.  Output phase a (o = j*s + a) receives the
// filter taps kk == (a+pb) mod s, read at input offset d = (a + pb - kk)/s.
namespace {
struct PhaseTaps { int n; int src[kMaxTaps]; int8_t d[kMaxTaps * 3]; };
void phase_taps(int kh, int kw, int s, int ay, int ax, PhaseTaps* pt) {
  const int pby = (kh - s > 0 ? kh - s : 0) / 2, pbx = (kw - s > 0 ? kw - s : 0) / 2;
  pt->n = 0;
  for (int ky = 0; ky < kh; ++ky) {
    const int ny = ay + pby - ky;
    if (((ny % s) + s) % s != 0) continue;
    for (int kx = 0; kx < kw; ++kx) {
      const int nx = ax + pbx - kx;
      if (((nx % s) + s) % s != 0) continue;
      const int dy = (ny >= 0) ? ny / s : -((-ny) / s), dx = (nx >= 0) ? nx / s : -((-nx) / s);
      pt->src[pt->n] = ky * kw + kx;
      pt->d[3 * pt->n + 0] = static_cast<int8_t>(dx);
      pt->d[3 * pt->n + 1] = static_cast<int8_t>(dy);
      pt->d[3 * pt->n + 2] = 0;
      ++pt->n;
    }
  }
}
}  // namespace

extern "C" int rn_pack_conv2d_transpose_weights(const float* w, void* packed, int kh, int kw, int Cin, int Cout,
                                                int cout_pad, int stride, int fmt, void* stream) {
  if (kh * kw > kMaxTaps || stride < 1) return -20;
  size_t off = 0;
  for (int ay = 0; ay < stride; ++ay)
    for (int ax = 0; ax < stride; ++ax) {
      PhaseTaps pt;
      phase_taps(kh, kw, stride, ay, ax, &pt);
      if (pt.n == 0) continue;
      // fmt 2: [all phases, hi][all phases, lo] -- the LO plane starts after the kh*kw taps of the HI plane
      int r = pack_conv_weights_impl(w, static_cast<uint16_t*>(packed) + off, kh * kw, Cin, Cout, cout_pad, 1, pt.src, pt.n,
                                     fmt, static_cast<long long>(kh) * kw * cout_pad * Cin, stream);
      if (r != 0) return r;
      off += static_cast<size_t>(pt.n) * cout_pad * Cin;
    }
  return 0;
}

extern "C" int rn_conv2d_transpose_same_scaled(const void* x, const void* w_packed, const float* w_unscale,
                                               const float* bias, const float* alpha, int act, void* out16, float* out32,
                                               int B, int H, int W, int Cin, int Cout, int cout_pad, int kh, int kw,
                                               int stride, int fmt, const rn_tuning* tune, void* stream) {
  if (kh * kw > kMaxTaps || stride < 1) return -20;
  const int Ho = H * stride, Wo = W * stride;
  size_t off = 0;
  for (int ay = 0; ay < stride; ++ay)
    for (int ax = 0; ax < stride; ++ax) {
      PhaseTaps pt;
      phase_taps(kh, kw, stride, ay, ax, &pt);
      if (pt.n == 0) return -21;  // k < stride: holes in the output are not supported
      rn_conv_desc d;
      memset(&d, 0, sizeof(d));
      d.ndim = 2; d.B = B; d.H = H; d.W = W; d.D = 1; d.Cin = Cin; d.Cout = Cout; d.cout_pad = cout_pad;
      d.ntaps = pt.n; d.taps = pt.d; d.x = x;
      d.w_packed = static_cast<const uint16_t*>(w_packed) + off;
      d.bias = bias; d.alpha = alpha; d.act = act; d.out16 = out16; d.out32 = out32;
      d.o_base = (static_cast<long long>(ay) * Wo + ax) * Cout;
      d.o_x = static_cast<long long>(stride) * Cout;
      d.o_y = static_cast<long long>(stride) * Wo * Cout;
      d.o_b = static_cast<long long>(Ho) * Wo * Cout;
      d.fmt = fmt;
      if (fmt == 2) {
        d.x_plane = static_cast<long long>(B) * H * W * Cin;
        d.w_plane = static_cast<long long>(kh) * kw * cout_pad * Cin;   // LO plane follows ALL phases of the HI plane
        d.o_plane = static_cast<long long>(B) * Ho * Wo * Cout;
      }
      d.w_unscale = w_unscale;
      apply_tuning(d, tune);
      int r = rn_conv_igemm(&d, stream);
      if (r != 0) return r;
      off += static_cast<size_t>(pt.n) * cout_pad * Cin;
    }
  return 0;
}

extern "C" int rn_conv2d_transpose_same(const void* x, const void* w_packed, const float* bias, const float* alpha,
                                        int act, void* out16, float* out32, int B, int H, int W, int Cin, int Cout,
                                        int cout_pad, int kh, int kw, int stride, int fmt, const rn_tuning* tune,
                                        void* stream) {
  return rn_conv2d_transpose_same_scaled(x, w_packed, nullptr, bias, alpha, act, out16, out32, B, H, W, Cin, Cout, cout_pad,
                                         kh, kw, stride, fmt, tune, stream);
}


// ---------------------------------------------------------------------------------- depth-folded conv3d
static bool banded_ok(int Cin, int Cout, int sz) {
  return !(Cin < 8 || Cout < 8 || 64 % Cin != 0 || 128 % Cout != 0 || sz < 1 || sz > 2);
}

extern "C" long long rn_conv3d_banded_bytes(int Cin, int Cout, int sz) {
  if (!banded_ok(Cin, Cout, sz)) return -1;
  const BandLayout L = band_layout(Cin, Cout, sz);
  if (L.kblocks > 8) return -1;
  return 9LL * L.kblocks * 128 * 64 * 2;             // 16-bit
}

extern "C" int rn_pack_conv3d_banded(const float* w, void* packed, int Cin, int Cout, int sz, int fmt, void* stream) {
  if (!w || !packed || rn_conv3d_banded_bytes(Cin, Cout, sz) < 0 || fmt < 0 || fmt > 2) return -1;
  const BandLayout L = band_layout(Cin, Cout, sz);
  const long long total = 9LL * L.kblocks * 128 * 64;
  pack_banded_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, static_cast<uint16_t*>(packed), Cin, Cout, L, sz, fmt, total);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_pack_conv3d_sliced(const float* w, void* packed, int fmt, void* stream) {
  if (!w || !packed || fmt < 0 || fmt > 2) return -1;
  pack_sliced_kernel<<<grid_for(9 * 96 * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, static_cast<uint16_t*>(packed), fmt, 9 * 96 * 32);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_expand_channels(const float* v, float* v_full, int C, int D, void* stream) {
  if (!v || !v_full || C < 1 || D < 1) return -1;
  const int n = C * D;
  expand_channels_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(v, v_full, C, n);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_conv3d_banded_same_scaled(const void* x, const void* w_banded, const float* w_unscale,
                                            const float* bias_full, const float* alpha_full, int act, const void* residual,
                                            int residual_is_f32, void* out16, float* out32, int B, int H, int W, int D,
                                            int Cin, int Cout, int sz, int fmt, const rn_tuning* tune, void* stream) {
  if (rn_conv3d_banded_bytes(Cin, Cout, sz) < 0) return -30;
  int Do, pz;
  same_pad(D, 3, sz, &Do, &pz);                     // TF SAME along z: out = ceil(D/sz), pad-before pz
  const long long Fi = static_cast<long long>(D) * Cin, Fo = static_cast<long long>(Do) * Cout;
  if (Fo % 128 != 0 || Fi % 8 != 0) return -31;
  int8_t taps[27];
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      int8_t* t = taps + 3 * (ky * 3 + kx);
      t[0] = static_cast<int8_t>(kx - 1); t[1] = static_cast<int8_t>(ky - 1); t[2] = 0;
    }
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 2; d.B = B; d.H = H; d.W = W; d.D = 1;
  d.Cin = band_layout(Cin, Cout, sz).kblocks * 64;  // K elements per (ky,kx) tap
  d.band_cin = Cin; d.band_cout = Cout; d.band_sz = sz;
  d.Cout = static_cast<int>(Fo); d.cout_pad = static_cast<int>(Fo);
  d.ntaps = 9; d.taps = taps; d.x = x; d.w_packed = w_banded; d.bias = bias_full; d.alpha = alpha_full; d.act = act;
  d.residual = residual; d.residual_is_f32 = residual_is_f32; d.out16 = out16; d.out32 = out32;
  d.o_base = 0; d.o_x = Fo; d.o_y = static_cast<long long>(W) * Fo; d.o_b = static_cast<long long>(H) * W * Fo;
  d.fmt = fmt; d.force_bn = 128;
  d.x_channels = static_cast<int>(Fi);
  d.a_c_base = -pz * Cin;                           // first input depth of N tile 0 is z = -pz (zero filled)
  d.a_c_ntile = (128 / Cout) * sz * Cin;            // each N tile advances 128/Cout output = sz*128/Cout input depths
  d.w_banded = 1;
  if (fmt == 2) {
    d.x_plane = static_cast<long long>(B) * H * W * Fi;
    d.w_plane = rn_conv3d_banded_bytes(Cin, Cout, sz) / 2;
    d.o_plane = static_cast<long long>(B) * H * W * Fo;
  }
  d.w_unscale = w_unscale;
  apply_tuning(d, tune);
  if (want_yhalo(tune)) d.ny = 3;
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_conv3d_banded_same(const void* x, const void* w_banded, const float* bias_full,
                                     const float* alpha_full, int act, const void* residual, int residual_is_f32,
                                     void* out16, float* out32, int B, int H, int W, int D, int Cin, int Cout,
                                     int sz, int fmt, const rn_tuning* tune, void* stream) {
  return rn_conv3d_banded_same_scaled(x, w_banded, nullptr, bias_full, alpha_full, act, residual, residual_is_f32, out16,
                                      out32, B, H, W, D, Cin, Cout, sz, fmt, tune, stream);
}


// ---------------------------------------------------------------------------------- texture decoder ops
extern "C" int rn_fully_connected(const float* x, const float* w, const float* bias, const float* alpha, void* out16,
                                  float* out32, int B, int K, int N, int fmt, void* stream) {
  if (!x || !w || (!out16 && !out32) || B < 1 || K < 1 || N < 1) return -1;
  if (B > 32) return -2;
  const size_t smem = static_cast<size_t>(B) * K * sizeof(float);
  if (smem > 48 * 1024) return -3;
  const int grid = (N + 255) / 256;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint16_t* o16 = static_cast<uint16_t*>(out16);
  if (B <= 8) fc_kernel<8><<<grid, 256, smem, st>>>(x, w, bias, alpha, o16, out32, B, K, N, fmt);
  else fc_kernel<32><<<grid, 256, smem, st>>>(x, w, bias, alpha, o16, out32, B, K, N, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_conv3d_small(const void* x, int x_is_f32, const float* w, const float* bias, const float* alpha,
                               void* out16, float* out32, int B, int H, int W, int D, int Cin, int Cout, int k,
                               int stride, int transposed, int fmt, void* stream) {
  if (!x || !w || (!out16 && !out32) || k < 1 || stride < 1) return -1;
  int Ho, Wo, Do, pb;
  if (transposed) {
    Ho = H * stride; Wo = W * stride; Do = D * stride;
    pb = (k - stride > 0 ? k - stride : 0) / 2;
  } else {
    int p2, p3;
    same_pad(H, k, stride, &Ho, &pb);
    same_pad(W, k, stride, &Wo, &p2);
    same_pad(D, k, stride, &Do, &p3);
    if (p2 != pb || p3 != pb) return -2;  // cubic inputs only
  }
  const long long total = static_cast<long long>(B) * Ho * Wo * Do;
  const int grid = static_cast<int>((total + 255) / 256);
  const size_t smem = static_cast<size_t>(k) * k * k * Cin * Cout * sizeof(float);
  if (smem > 48 * 1024) return -3;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint16_t* o16 = static_cast<uint16_t*>(out16);
  if (Cin == 8 && Cout == 4 && k == 4 && stride == 1 && !transposed && x_is_f32 && out32 != nullptr && out16 == nullptr &&
      H % 8 == 0 && W % 8 == 0 && D % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && tuning().tiled_tex_conv) {
    // texture decoder's last layer: shared-memory tiled kernel (bit-identical to the generic one)
    const size_t sm = (static_cast<size_t>(8) * T4_PLANE + 64 * 32) * sizeof(float);
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return static_cast<int>(cudaErrorInvalidDevice);
    if (!attr_set[dev].load(std::memory_order_acquire)) {
      cudaError_t e = cudaFuncSetAttribute(conv3d_k4_8to4_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sm));
      if (e != cudaSuccess) return static_cast<int>(e);
      attr_set[dev].store(true, std::memory_order_release);
    }
    const long long blocks = static_cast<long long>(B) * (H / 8) * (W / 8) * (D / 8);
    conv3d_k4_8to4_tiled_kernel<<<static_cast<int>(blocks), 256, sm, st>>>(static_cast<const float*>(x), w, bias, alpha, out32, B, H, W, D);
    RN_COUNT_LAUNCH();
    return static_cast<int>(cudaGetLastError());
  }
#define RN_SMALL(CI, CO)                                                                                            \
  conv3d_small_kernel<CI, CO><<<grid, 256, smem, st>>>(x, x_is_f32, w, bias, alpha, o16, out32, B, H, W, D, Ho, Wo, \
                                                        Do, k, stride, pb, transposed, fmt)
  if (Cin == 4 && Cout == 4) RN_SMALL(4, 4);
  else if (Cin == 4 && Cout == 8) RN_SMALL(4, 8);
  else if (Cin == 8 && Cout == 4) RN_SMALL(8, 4);
  else if (Cin == 2 && Cout == 3) RN_SMALL(2, 3);
  else return -4;
#undef RN_SMALL
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_concat_channels_f32(const float* a, const float* b, float* out, long long n, int Ca, int Cb,
                                      void* stream) {
  if (!a || !b || !out || n < 0 || Ca < 1 || Cb < 1) return -1;
  if (n == 0) return 0;
  concat_channels_kernel<<<grid_for(n * (Ca + Cb), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, b, out, n, Ca,
                                                                                                     Cb);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}


// ---------------------------------------------------------------------------------- x-folded thin transposed conv
extern "C" int rn_xfold_factor(int Cin, int W) {
  if (Cin >= 64 || Cin < 8 || 64 % Cin != 0) return 1;
  const int F = 64 / Cin;
  return (W % F == 0) ? F : 1;
}

extern "C" int rn_pack_conv2d_transpose_xfold(const float* w, void* packed, int kh, int kw, int Cin, int Cout, int F,
                                              int cout_pad, int fmt, void* stream) {
  if (!w || !packed || F < 2 || kw > 2 * F || cout_pad < F * Cout || kh * 3 > kMaxTaps) return -1;
  const long long total = static_cast<long long>(kh) * 3 * cout_pad * F * Cin;
  pack_xfold_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, static_cast<uint16_t*>(packed), kh, kw, Cin, Cout, F, cout_pad, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

// x [B,H,W,Cin] 16-bit; w_xfold from rn_pack_conv2d_transpose_xfold ([kh*3][cout_pad][F*Cin]); bias_x / alpha_x are the
// per-Cout vectors tiled F times and zero padded to cout_pad (rn_expand_channels + padding by the caller).
extern "C" int rn_conv2d_transpose_s1_xfold_scaled(const void* x, const void* w_xfold, const float* w_unscale,
                                                   const float* bias_x, const float* alpha_x, int act, void* out16,
                                                   float* out32, int B, int H, int W, int Cin, int Cout, int kh, int kw, int F,
                                                   int cout_pad, int fmt, const rn_phong* phong, const rn_tuning* tune,
                                                   void* stream) {
  if (F < 2 || W % F != 0 || kh * 3 > kMaxTaps) return -20;
  int8_t taps[kMaxTaps * 3];
  const int pby = (kh - 1) / 2;                     // SAME stride-1 transposed: dy = pb - ky
  for (int kyr = 0; kyr < kh; ++kyr)                // ky-reversed order (see pack_xfold_kernel): dy = kyr - (kh-1-pby)
    for (int j = 0; j < 3; ++j) {
      int8_t* t = taps + 3 * (kyr * 3 + j);
      t[0] = static_cast<int8_t>(j - 1); t[1] = static_cast<int8_t>(pby - (kh - 1 - kyr)); t[2] = 0;
    }
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 2; d.B = B; d.H = H; d.W = W / F; d.D = 1; d.Cin = F * Cin; d.Cout = F * Cout; d.cout_pad = cout_pad;
  d.ntaps = kh * 3; d.taps = taps; d.x = x; d.w_packed = w_xfold; d.bias = bias_x; d.alpha = alpha_x; d.act = act;
  d.out16 = out16; d.out32 = out32;
  d.o_base = 0; d.o_x = static_cast<long long>(F) * Cout; d.o_y = static_cast<long long>(W) * Cout;
  d.o_b = static_cast<long long>(H) * W * Cout; d.fmt = fmt;
  if (fmt == 2) {
    d.x_plane = static_cast<long long>(B) * H * W * Cin;
    d.w_plane = static_cast<long long>(kh) * 3 * cout_pad * F * Cin;
    d.o_plane = static_cast<long long>(B) * H * W * Cout;
  }
  if (phong != nullptr && (Cout != 3 || act != RN_ACT_SIGMOID || cout_pad != 16)) return -22;
  d.phong = phong;
  d.w_unscale = w_unscale;
  apply_tuning(d, tune);
  if (want_yhalo(tune) && (F * Cin) % 64 == 0) d.ny = kh;    // tap = kyr*3 + j, dy consecutive in kyr: the kh taps share one halo load
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_conv2d_transpose_s1_xfold(const void* x, const void* w_xfold, const float* bias_x, const float* alpha_x,
                                            int act, void* out16, float* out32, int B, int H, int W, int Cin, int Cout,
                                            int kh, int kw, int F, int cout_pad, int fmt, const rn_phong* phong,
                                            const rn_tuning* tune, void* stream) {
  return rn_conv2d_transpose_s1_xfold_scaled(x, w_xfold, nullptr, bias_x, alpha_x, act, out16, out32, B, H, W, Cin, Cout, kh,
                                             kw, F, cout_pad, fmt, phong, tune, stream);
}


// ---------------------------------------------------------------------------------- merged-phase transposed conv
extern "C" int rn_pack_conv2d_transpose_s2_merged(const float* w, void* packed, int Cin, int Cout, int fmt,
                                                  void* stream) {
  if (!w || !packed || Cin < 16 || Cout < 16 || Cout % 16 != 0) return -1;
  pack_tconv_s2_merged_kernel<<<grid_for(9LL * 4 * Cout * Cin, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, static_cast<uint16_t*>(packed), Cin, Cout, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_conv2d_transpose_s2_merged_scaled(const void* x, const void* w_merged, const float* w_unscale,
                                                    const float* bias4, const float* alpha4, int act, void* out16,
                                                    float* out32, int B, int H, int W, int Cin, int Cout, int fmt,
                                                    const rn_tuning* tune, void* stream) {
  if (Cout % 16 != 0) return -20;
  int8_t taps[27];
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      int8_t* t = taps + 3 * (ky * 3 + kx);
      t[0] = static_cast<int8_t>(kx - 1); t[1] = static_cast<int8_t>(ky - 1); t[2] = 0;
    }
  const long long Wo = 2LL * W, Ho = 2LL * H;
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 2; d.B = B; d.H = H; d.W = W; d.D = 1; d.Cin = Cin; d.Cout = 4 * Cout; d.cout_pad = 4 * Cout;
  d.ntaps = 9; d.taps = taps; d.x = x; d.w_packed = w_merged; d.bias = bias4; d.alpha = alpha4; d.act = act;
  d.out16 = out16; d.out32 = out32;
  d.o_base = 0; d.o_x = 2LL * Cout; d.o_y = 2LL * Wo * Cout; d.o_b = Ho * Wo * Cout;
  d.o_nsplit = 2 * Cout; d.o_nhi = Wo * Cout;      // n = (ay, ax, co): row 2y+ay, columns (2x+ax)*Cout + co
  d.fmt = fmt;
  if (fmt == 2) {
    d.x_plane = static_cast<long long>(B) * H * W * Cin;
    d.w_plane = 9LL * 4 * Cout * Cin;
    d.o_plane = static_cast<long long>(B) * Ho * Wo * Cout;
  }
  d.w_unscale = w_unscale;
  apply_tuning(d, tune);
  if (Cin % 64 == 0 && want_yhalo(tune)) d.ny = 3;
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_conv2d_transpose_s2_merged(const void* x, const void* w_merged, const float* bias4,
                                             const float* alpha4, int act, void* out16, float* out32, int B, int H,
                                             int W, int Cin, int Cout, int fmt, const rn_tuning* tune, void* stream) {
  return rn_conv2d_transpose_s2_merged_scaled(x, w_merged, nullptr, bias4, alpha4, act, out16, out32, B, H, W, Cin, Cout, fmt,
                                              tune, stream);
}

// ---------------------------------------------------------------------------------- thin conv3d
extern "C" int rn_conv3d_direct(const void* x, int x_is_f32, const float* w, const float* bias, const float* alpha,
                                void* out16, int B, int H, int W, int D, int Cin, int Cout, int k, int sy, int sx,
                                int sz, int fmt, void* stream) {
  if (!x || !w || !bias || !out16) return -1;
  int Ho, Wo, Do, py, px, pz;
  same_pad(H, k, sy, &Ho, &py);
  same_pad(W, k, sx, &Wo, &px);
  same_pad(D, k, sz, &Do, &pz);
  const long long total = static_cast<long long>(B) * Ho * Wo * Do;
  const int block = 256;
  const int grid = static_cast<int>((total + block - 1) / block);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint16_t* o = static_cast<uint16_t*>(out16);
#define RN_LAUNCH_DIRECT(CI, CO, KK, XF)                                                                          \
  conv3d_direct_kernel<CI, CO, KK, XF><<<grid, block, 0, st>>>(x, w, bias, alpha, o, B, H, W, D, Ho, Wo, Do, sy, \
                                                                  sx, sz, py, px, pz, fmt)
  if (Cin == 1 && Cout == 8 && k == 5 && x_is_f32) RN_LAUNCH_DIRECT(1, 8, 5, true);
  else if (Cin == 5 && Cout == 8 && k == 5 && x_is_f32) RN_LAUNCH_DIRECT(5, 8, 5, true);
  else if (Cin == 8 && Cout == 16 && k == 3 && !x_is_f32) RN_LAUNCH_DIRECT(8, 16, 3, false);
  else if (Cin == 8 && Cout == 8 && k == 3 && !x_is_f32) RN_LAUNCH_DIRECT(8, 8, 3, false);
  else if (Cin == 2 && Cout == 8 && k == 3 && x_is_f32) RN_LAUNCH_DIRECT(2, 8, 3, true);
  else return -2;
#undef RN_LAUNCH_DIRECT
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_resample_conv1_fused_window(const float* vox, const float* minv, const float* w, const float* bias,
                                              const float* alpha, void* out16, int B, int size, int new_size, int y0, int x0,
                                              int ph, int pw, int fmt, void* stream) {
  if (!vox || !minv || !w || !bias || !out16 || B < 1 || size < 2) return -1;
  if (new_size < 16 || new_size % 16 != 0 || !window_ok(new_size, y0, x0, ph, pw)) return -2;   // 8^3-output tiles
  const long long blocks = static_cast<long long>(B) * (ph / 16) * (pw / 16) * (new_size / 16);
  if (blocks > 0x7fffffffLL) return -3;
  resample_conv1_kernel<<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      vox, minv, w, bias, alpha, static_cast<uint16_t*>(out16), B, size, new_size, fmt, y0, x0, ph, pw);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_resample_conv1_fused(const float* vox, const float* minv, const float* w, const float* bias,
                                       const float* alpha, void* out16, int B, int size, int new_size, int fmt,
                                       void* stream) {
  return rn_resample_conv1_fused_window(vox, minv, w, bias, alpha, out16, B, size, new_size, 0, 0, new_size, new_size, fmt,
                                        stream);
}

extern "C" int rn_resample5_conv1_fused_window(const float* vox, const float* tex, const float* minv, const float* w,
                                               const float* bias, const float* alpha, void* out16, int B, int size,
                                               int new_size, int y0, int x0, int ph, int pw, int fmt, void* stream) {
  if (!vox || !tex || !minv || !w || !bias || !out16 || B < 1 || size < 2 || fmt < 0 || fmt > 2) return -1;
  if (new_size < 16 || new_size % 16 != 0 || !window_ok(new_size, y0, x0, ph, pw)) return -2;
  if ((reinterpret_cast<uintptr_t>(tex) & 15) != 0) return -4;      // float4 gathers of the 4-channel texture volume
  const long long blocks = static_cast<long long>(B) * (ph / 16) * (pw / 16) * (new_size / 16);
  if (blocks > 0x7fffffffLL) return -3;
  const size_t smem = (static_cast<size_t>(RC5_C) * RC5_TILE + 125 * RC5_C * 8) * sizeof(float);
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return static_cast<int>(cudaErrorInvalidDevice);
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(resample5_conv1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set[dev].store(true, std::memory_order_release);
  }
  resample5_conv1_kernel<<<static_cast<int>(blocks), 256, smem, static_cast<cudaStream_t>(stream)>>>(
      vox, tex, minv, w, bias, alpha, static_cast<uint16_t*>(out16), B, size, new_size, fmt, y0, x0, ph, pw);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_resample5_conv1_fused(const float* vox, const float* tex, const float* minv, const float* w,
                                        const float* bias, const float* alpha, void* out16, int B, int size, int new_size,
                                        int fmt, void* stream) {
  return rn_resample5_conv1_fused_window(vox, tex, minv, w, bias, alpha, out16, B, size, new_size, 0, 0, new_size, new_size,
                                         fmt, stream);
}

extern "C" int rn_binvox_decode(const uint8_t* pairs, const int* run_start, const int* item_first_run, float* out,
                                int n_items, int d0, int d1, int d2, int fix_coords, void* stream) {
  if (!pairs || !run_start || !item_first_run || !out || n_items < 1 || d0 < 1 || d1 < 1 || d2 < 1) return -1;
  const long long total = static_cast<long long>(d0) * d1 * d2 * n_items;
  if (static_cast<long long>(d0) * d1 * d2 > 0x7fffffffLL) return -2;
  binvox_decode_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      pairs, run_start, item_first_run, out, n_items, d0, d1, d2, fix_coords);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_phong_composite(const float* img, const float* light_dir, const float* light_col, float ambient,
                                  float k_diffuse, int background_white, int with_mask, float* out_f32,
                                  uint8_t* out_u8, int B, int H, int W, void* stream) {
  if (!img || !light_dir || !light_col || (!out_f32 && !out_u8)) return -1;
  return rn_phong_shade(img, nullptr, light_dir, light_col, ambient, k_diffuse, RN_PHONG_NUMPY, background_white, with_mask,
                        nullptr, out_f32, out_u8, B, H, W, stream);
}

namespace {
int phong_shade_launch(const float* normal, const float* albedo, const float* light_dir, const float* light_col, float ambient,
                       const float* ambient_b, float k_diffuse, int composite, int background_white, int with_mask,
                       float* shade_f32, float* compos_f32, uint8_t* compos_u8, int B, int H, int W, void* stream) {
  if (!normal || !light_dir || !light_col || (!shade_f32 && !compos_f32 && !compos_u8) || B < 1 || H < 1 || W < 1) return -1;
  if (composite != RN_PHONG_NUMPY && composite != RN_PHONG_TF) return -1;
  if (B > 65535 || static_cast<long long>(H) * W > 0x7fffffffLL - 255) return -2;
  const int HW = H * W;
  const dim3 grid((HW + 255) / 256, B);
  const int white = background_white != 0, mask = with_mask != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (composite == RN_PHONG_TF && ambient_b)
    phong_shade_kernel<true, true><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, 0.f, k_diffuse, white, mask,
                                                         shade_f32, compos_f32, compos_u8, HW, ambient_b);
  else if (composite == RN_PHONG_TF)
    phong_shade_kernel<true, false><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, ambient, k_diffuse, white, mask,
                                                          shade_f32, compos_f32, compos_u8, HW, nullptr);
  else if (ambient_b)
    phong_shade_kernel<false, true><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, 0.f, k_diffuse, white, mask,
                                                          shade_f32, compos_f32, compos_u8, HW, ambient_b);
  else
    phong_shade_kernel<false, false><<<grid, 256, 0, st>>>(normal, albedo, light_dir, light_col, ambient, k_diffuse, white, mask,
                                                           shade_f32, compos_f32, compos_u8, HW, nullptr);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}
}  // namespace

extern "C" int rn_phong_shade(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                              float ambient, float k_diffuse, int composite, int background_white, int with_mask, float* shade_f32,
                              float* compos_f32, uint8_t* compos_u8, int B, int H, int W, void* stream) {
  return phong_shade_launch(normal, albedo, light_dir, light_col, ambient, nullptr, k_diffuse, composite, background_white,
                            with_mask, shade_f32, compos_f32, compos_u8, B, H, W, stream);
}

extern "C" int rn_phong_shade_ambient(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                                      const float* ambient, float k_diffuse, int composite, int background_white, int with_mask,
                                      float* shade_f32, float* compos_f32, uint8_t* compos_u8, int B, int H, int W, void* stream) {
  if (!ambient) return -1;
  return phong_shade_launch(normal, albedo, light_dir, light_col, 0.f, ambient, k_diffuse, composite, background_white,
                            with_mask, shade_f32, compos_f32, compos_u8, B, H, W, stream);
}
