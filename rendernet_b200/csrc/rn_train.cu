// rn_train.cu -- what the TRAINING step of the Shader network needs beyond the input-gradient pass (SURVEY §8 f-4, stage 2;
// RenderNet_Shader.py:154-167: dropout after ten layers, MSE / BCE reconstruction loss, tf.train.AdamOptimizer(beta1 = 0.5) over
// every filter, bias and PReLU slope):
//   * rn_conv_weight_grad_direct : weight gradient of ANY convolution or transposed convolution of the network (2-D or 3-D, any
//     stride, TF SAME) as a strided correlation  dW[tap][a][b] = sum_p P[p][a] * Q[p*s + tap - pad][b]  on the CUDA cores, fp32
//     accumulation.  The thin layers (e_conv1 / e_conv2, the transposed convs) go through it; the wide stride-1 2-D layers and
//     the depth-folded 3^3 layers use the wgmma kernel of rn_wgrad.cu (97 % of the parameters, 90 % of the MACs).
//   * rn_prelu_alpha_grad        : dL/dalpha[c] = sum_{z<0} g * z  (tools/layer_util.py:27-45, alpha is initialised to 0, so the
//     pre-activation z cannot be recovered from the stored output and is recomputed by the caller).
//   * rn_dropout_16              : tf.nn.dropout (x / keep where a counter-based hash of (seed, layer, element) < keep, else 0);
//     the same call applied to the gradient is its backward (the mask is recomputed, never stored).
//   * rn_image_loss_grad         : reconstruction loss and its gradient w.r.t. the image (MSE :163, BCE :160-161).
//   * rn_adam_step               : one Adam update of a flat fp32 parameter (TF formulation: lr_t folded by the caller).
//   * rn_voxel_fit_grad          : the shape fit's gradient w.r.t. the shared occupancy grid (views summed, smoothness and
//     binary regularisers, carve mask) and the two regularisers, with a fixed-order reduction.
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <initializer_list>

#include "../../include/rendernet_b200.h"
#include "rn_dropout_hash.h"

namespace rn {
extern std::atomic<long long> g_launch_count;
}
#define RN_COUNT_LAUNCH() rn::g_launch_count.fetch_add(1, std::memory_order_relaxed)

namespace {

// element i of a tensor in format fmt: 0 fp16, 1 bf16, 2 fp16 hi/lo planes (value = hi + lo), 3 fp32
__device__ __forceinline__ float ld_any(const void* __restrict__ base, long long i, int fmt, long long plane) {
  if (fmt == 3) return static_cast<const float*>(base)[i];
  const uint16_t* p = static_cast<const uint16_t*>(base);
  const uint16_t u = p[i];
  if (fmt == 1) return __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&u));
  float v = __half2float(*reinterpret_cast<const __half*>(&u));
  if (fmt == 2) {
    const uint16_t l = p[i + plane];
    v += __half2float(*reinterpret_cast<const __half*>(&l));
  }
  return v;
}
__device__ __forceinline__ void st_16(void* __restrict__ base, long long i, float v, int fmt, long long plane) {
  uint16_t* p = static_cast<uint16_t*>(base);
  if (fmt == 1) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    p[i] = *reinterpret_cast<const uint16_t*>(&h);
    return;
  }
  const __half h = __float2half_rn(v);
  p[i] = *reinterpret_cast<const uint16_t*>(&h);
  if (fmt == 2) {
    const __half l = __float2half_rn(v - __half2float(h));
    p[i + plane] = *reinterpret_cast<const uint16_t*>(&l);
  }
}

struct WgradDirectParams {
  const void* P;      // coarse-grid operand  [B, Dp, Hp, Wp, Cap]  (channel pitch Cap, Ca channels used)
  const void* Q;      // fine-grid operand    [B, Dq, Hq, Wq, Cbp]
  float* dW;          // [taps][Ca][Cb] fp32, accumulated with atomics (zeroed by the wrapper)
  int B, Dp, Hp, Wp, Ca, Cap, Dq, Hq, Wq, Cb, Cbp;
  int kd, kh, kw, sd, sh, sw, pd, ph, pw;
  int fmtP, fmtQ;
  long long planeP, planeQ, npos;   // npos = B * Dp * Hp * Wp
  int a_tiles, b_tiles;
  float scale;
};

constexpr int kTile = 32;     // dW tile: 32 (a) x 32 (b) per CTA, 2 x 2 per thread
constexpr int kChunk = 32;    // positions per shared-memory stage

// One CTA: one filter tap, one 32 x 32 tile of (a, b), a strided set of 32-position chunks of the coarse grid.
__global__ void __launch_bounds__(256) wgrad_direct_kernel(const WgradDirectParams p) {
  __shared__ float Ps[kChunk][kTile + 1];
  __shared__ float Qs[kChunk][kTile + 1];
  const int tap = blockIdx.z;
  const int kx = tap % p.kw, ky = (tap / p.kw) % p.kh, kz = tap / (p.kw * p.kh);
  const int a0 = (static_cast<int>(blockIdx.y) / p.b_tiles) * kTile, b0 = (static_cast<int>(blockIdx.y) % p.b_tiles) * kTile;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lp = threadIdx.x >> 3, lc = (threadIdx.x & 7) * 4;      // loader: position lp of the chunk, channels lc..lc+3
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  const long long nchunks = (p.npos + kChunk - 1) / kChunk;
  for (long long ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const long long pos = ch * kChunk + lp;
    float pv[4] = {0.f, 0.f, 0.f, 0.f}, qv[4] = {0.f, 0.f, 0.f, 0.f};
    if (pos < p.npos) {
      long long r = pos;
      const int x = static_cast<int>(r % p.Wp); r /= p.Wp;
      const int y = static_cast<int>(r % p.Hp); r /= p.Hp;
      const int z = static_cast<int>(r % p.Dp);
      const int n = static_cast<int>(r / p.Dp);
      const int qx = x * p.sw + kx - p.pw, qy = y * p.sh + ky - p.ph, qz = z * p.sd + kz - p.pd;
      if (qx >= 0 && qx < p.Wq && qy >= 0 && qy < p.Hq && qz >= 0 && qz < p.Dq) {      // outside the fine grid: zero padding
        const long long pb = pos * p.Cap;
        const long long qb = (((static_cast<long long>(n) * p.Dq + qz) * p.Hq + qy) * p.Wq + qx) * p.Cbp;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (a0 + lc + j < p.Ca) pv[j] = ld_any(p.P, pb + a0 + lc + j, p.fmtP, p.planeP);
          if (b0 + lc + j < p.Cb) qv[j] = ld_any(p.Q, qb + b0 + lc + j, p.fmtQ, p.planeQ);
        }
      }
    }
    __syncthreads();                // the previous chunk has been consumed
#pragma unroll
    for (int j = 0; j < 4; ++j) { Ps[lp][lc + j] = pv[j]; Qs[lp][lc + j] = qv[j]; }
    __syncthreads();
#pragma unroll 8
    for (int i = 0; i < kChunk; ++i) {
      const float pa0 = Ps[i][ty], pa1 = Ps[i][ty + 16], qb0 = Qs[i][tx], qb1 = Qs[i][tx + 16];
      acc[0][0] = fmaf(pa0, qb0, acc[0][0]); acc[0][1] = fmaf(pa0, qb1, acc[0][1]);
      acc[1][0] = fmaf(pa1, qb0, acc[1][0]); acc[1][1] = fmaf(pa1, qb1, acc[1][1]);
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int a = a0 + ty + 16 * i, b = b0 + tx + 16 * j;
      if (a < p.Ca && b < p.Cb && acc[i][j] != 0.f)
        atomicAdd(&p.dW[(static_cast<long long>(tap) * p.Ca + a) * p.Cb + b], acc[i][j] * p.scale);
    }
}

// Thin layers (e_conv1: 8 x 1 channels, 125 taps; e_conv11: 16 x 3): a 32 x 32 tile would be >95 % padding.  Here a thread owns a
// whole CA x CB block of partial sums over its own positions (consecutive threads = consecutive positions: coalesced), and the
// CTA (one tap) reduces them by warp shuffles + shared memory before CA x CB atomics.
template <int CA, int CB>
__global__ void __launch_bounds__(256) wgrad_thin_kernel(const WgradDirectParams p) {
  __shared__ float red[8][CA * CB];
  const int tap = blockIdx.y;
  const int kx = tap % p.kw, ky = (tap / p.kw) % p.kh, kz = tap / (p.kw * p.kh);
  float acc[CA][CB];
#pragma unroll
  for (int a = 0; a < CA; ++a)
#pragma unroll
    for (int b = 0; b < CB; ++b) acc[a][b] = 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long pos = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; pos < p.npos; pos += stride) {
    long long r = pos;
    const int x = static_cast<int>(r % p.Wp); r /= p.Wp;
    const int y = static_cast<int>(r % p.Hp); r /= p.Hp;
    const int z = static_cast<int>(r % p.Dp);
    const int n = static_cast<int>(r / p.Dp);
    const int qx = x * p.sw + kx - p.pw, qy = y * p.sh + ky - p.ph, qz = z * p.sd + kz - p.pd;
    if (qx < 0 || qx >= p.Wq || qy < 0 || qy >= p.Hq || qz < 0 || qz >= p.Dq) continue;
    const long long pb = pos * p.Cap;
    const long long qb = (((static_cast<long long>(n) * p.Dq + qz) * p.Hq + qy) * p.Wq + qx) * p.Cbp;
    float qv[CB];
#pragma unroll
    for (int b = 0; b < CB; ++b) qv[b] = ld_any(p.Q, qb + b, p.fmtQ, p.planeQ);
#pragma unroll
    for (int a = 0; a < CA; ++a) {
      const float pv = ld_any(p.P, pb + a, p.fmtP, p.planeP);
#pragma unroll
      for (int b = 0; b < CB; ++b) acc[a][b] = fmaf(pv, qv[b], acc[a][b]);
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < CA; ++a)
#pragma unroll
    for (int b = 0; b < CB; ++b) {
      float v = acc[a][b];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[warp][a * CB + b] = v;
    }
  __syncthreads();
  if (threadIdx.x < CA * CB) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += red[w][threadIdx.x];
    if (v != 0.f) atomicAdd(&p.dW[static_cast<long long>(tap) * CA * CB + threadIdx.x], v * p.scale);
  }
}

// dalpha[c] += scale * sum over elements of channel c with z < 0 of g * z
__global__ void __launch_bounds__(256) prelu_alpha_grad_kernel(const void* __restrict__ g, const void* __restrict__ z,
                                                               float* __restrict__ dalpha, long long n, int C, int fmt, float scale) {
  extern __shared__ float acc[];        // [C]
  for (int c = threadIdx.x; c < C; c += blockDim.x) acc[c] = 0.f;
  __syncthreads();
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float zv = ld_any(z, i, fmt, n);
    if (zv < 0.f) atomicAdd(&acc[static_cast<int>(i % C)], ld_any(g, i, fmt, n) * zv);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    if (acc[c] != 0.f) atomicAdd(&dalpha[c], acc[c] * scale);
}

// Parameter gradient of the texture decoder's FC + PReLU (e_tex_fc1, RenderNet_Texture_Face_Normal.py:37-38) in one pass over
// gy and z.  A thread owns four adjacent columns: gz = gy * (z > 0 ? 1 : alpha) of all BT (>= B, zero padded) rows stays in
// registers, and dW[k][n..n+3] = sum_b x[b][k] gz[b][n..n+3] is one float4 store per k, x read as a broadcast from shared
// memory.  blockIdx.x splits K (the CTAs of one column block run side by side and share gy / z in L2); only the K part 0
// writes gz, db and dalpha.  Every sum runs over b in a fixed order: the result is reproducible bit for bit.  z == NULL: an FC
// without activation (the shape decoder's g_gc1), gz = gy, no slope and no dalpha.
template <int BT>
__global__ void __launch_bounds__(128) fc_param_grad_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                            const float* __restrict__ z, const float* __restrict__ alpha,
                                                            float* __restrict__ gz, float* __restrict__ dw, float* __restrict__ db,
                                                            float* __restrict__ dalpha, int B, int K, int N, int kchunk) {
  extern __shared__ float sx[];                     // [BT][kchunk], rows b >= B zero
  const int k0 = blockIdx.x * kchunk;
  const int kn = min(kchunk, K - k0);
  for (int i = threadIdx.x; i < BT * kchunk; i += blockDim.x) {
    const int b = i / kchunk, k = i % kchunk;
    sx[i] = (b < B && k < kn) ? x[static_cast<long long>(b) * K + k0 + k] : 0.f;
  }
  __syncthreads();
  const long long n = (static_cast<long long>(blockIdx.y) * blockDim.x + threadIdx.x) * 4;
  if (n >= N) return;
  const bool ident = z == nullptr;
  const float4 a = ident ? make_float4(1.f, 1.f, 1.f, 1.f) : *reinterpret_cast<const float4*>(alpha + n);
  const bool first = blockIdx.x == 0;
  float4 g[BT];
  float4 sb = make_float4(0.f, 0.f, 0.f, 0.f), sa = sb;
#pragma unroll
  for (int b = 0; b < BT; ++b) {
    g[b] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (b < B) {
      const long long o = static_cast<long long>(b) * N + n;
      const float4 gv = *reinterpret_cast<const float4*>(gy + o);
      const float4 zv = ident ? make_float4(1.f, 1.f, 1.f, 1.f) : *reinterpret_cast<const float4*>(z + o);
      g[b] = make_float4(zv.x > 0.f ? gv.x : gv.x * a.x, zv.y > 0.f ? gv.y : gv.y * a.y, zv.z > 0.f ? gv.z : gv.z * a.z,
                         zv.w > 0.f ? gv.w : gv.w * a.w);
      if (first) {
        sb.x += g[b].x; sb.y += g[b].y; sb.z += g[b].z; sb.w += g[b].w;
        if (zv.x < 0.f) sa.x = fmaf(gv.x, zv.x, sa.x);
        if (zv.y < 0.f) sa.y = fmaf(gv.y, zv.y, sa.y);
        if (zv.z < 0.f) sa.z = fmaf(gv.z, zv.z, sa.z);
        if (zv.w < 0.f) sa.w = fmaf(gv.w, zv.w, sa.w);
        if (gz) *reinterpret_cast<float4*>(gz + o) = g[b];
      }
    }
  }
  if (first) {
    *reinterpret_cast<float4*>(db + n) = sb;
    if (dalpha) *reinterpret_cast<float4*>(dalpha + n) = sa;
  }
  for (int k = 0; k < kn; ++k) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      const float xv = sx[b * kchunk + k];
      acc.x = fmaf(xv, g[b].x, acc.x); acc.y = fmaf(xv, g[b].y, acc.y);
      acc.z = fmaf(xv, g[b].z, acc.z); acc.w = fmaf(xv, g[b].w, acc.w);
    }
    __stcs(reinterpret_cast<float4*>(dw + static_cast<long long>(k0 + k) * N + n), acc);     // streamed: dW is not re-read here
  }
}

// fp32 PReLU derivative with the bias and slope gradients of a thin decoder conv (C = 4 or 8 channels, 16-byte aligned):
// gz = gy * (z > 0 ? 1 : alpha[c]), db[c] += sum gz, dalpha[c] += sum_{z<0} gy * z.  A thread walks whole voxels and keeps the
// 2C partial sums in registers; warp shuffles and shared memory reduce them, then one atomic per CTA and channel.
template <int C>
__global__ void __launch_bounds__(256) prelu_grad_f32_kernel(const float* __restrict__ gy, const float* __restrict__ z,
                                                             const float* __restrict__ alpha, float* __restrict__ gz,
                                                             float* __restrict__ db, float* __restrict__ dalpha, long long nvox) {
  constexpr int Q = C / 4;
  __shared__ float red[8][2 * C];
  float a[C], sb[C], sa[C];
#pragma unroll
  for (int c = 0; c < C; ++c) { a[c] = alpha[c]; sb[c] = 0.f; sa[c] = 0.f; }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvox; v += stride) {
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const long long o = v * C + 4 * q;
      const float4 gv = *reinterpret_cast<const float4*>(gy + o), zv = *reinterpret_cast<const float4*>(z + o);
      const float gs[4] = {gv.x, gv.y, gv.z, gv.w}, zs[4] = {zv.x, zv.y, zv.z, zv.w};
      float os[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = 4 * q + j;
        os[j] = zs[j] > 0.f ? gs[j] : gs[j] * a[c];
        sb[c] += os[j];
        if (zs[j] < 0.f) sa[c] = fmaf(gs[j], zs[j], sa[c]);
      }
      *reinterpret_cast<float4*>(gz + o) = make_float4(os[0], os[1], os[2], os[3]);
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    float u = sb[c], w = sa[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      u += __shfl_xor_sync(0xffffffffu, u, o);
      w += __shfl_xor_sync(0xffffffffu, w, o);
    }
    if (lane == 0) { red[warp][c] = u; red[warp][C + c] = w; }
  }
  __syncthreads();
  if (threadIdx.x < 2 * C) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    atomicAdd(threadIdx.x < C ? &db[threadIdx.x] : &dalpha[threadIdx.x - C], s);
  }
}

__global__ void __launch_bounds__(256) dropout_kernel(const void* x, void* out, long long n, float keep,
                                                      unsigned long long threshold, uint32_t seed, uint32_t salt, int fmt) {
  const float inv = 1.0f / keep;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool kept = rn_dropout_hash(seed, salt, static_cast<unsigned long long>(i)) < threshold;
    st_16(out, i, kept ? ld_any(x, i, fmt, n) * inv : 0.f, fmt, n);
  }
}

// kind 0: MSE  (tf.losses.mean_squared_error: mean over every element)          dL/dp = 2 (p - t) / n
// kind 1: BCE  (-mean_b sum_hwc [t log(1e-6 + p) + (1 - t) log(1e-6 + 1 - p)])  dL/dp = -(t / (1e-6 + p) - (1 - t) / (1e-6 + 1 - p)) / B
__global__ void __launch_bounds__(256) image_loss_grad_kernel(const float* __restrict__ img, const float* __restrict__ target,
                                                              float* __restrict__ dimg, double* __restrict__ loss, long long n,
                                                              int batch, int kind) {
  __shared__ double red[256];
  double s = 0.0;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const float inv_n = 1.0f / static_cast<float>(n), inv_b = 1.0f / static_cast<float>(batch);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float p = img[i], t = target[i];
    if (kind == 0) {
      const float d = p - t;
      s += static_cast<double>(d) * d;
      if (dimg) dimg[i] = 2.0f * d * inv_n;
    } else {
      const float a = 1e-6f + p, b = 1e-6f + 1.0f - p;
      s -= static_cast<double>(t * logf(a) + (1.0f - t) * logf(b));
      if (dimg) dimg[i] = -(t / a - (1.0f - t) / b) * inv_b;
    }
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(loss, red[0] * (kind == 0 ? 1.0 / static_cast<double>(n) : 1.0 / static_cast<double>(batch)));
}

// Per item (rn_image_loss_grad_items): blockIdx.y = item b of m elements.  kind 0: loss[b] = mean (p - t)^2, dL/dp = 2 (p - t) / m;
// kind 1: loss[b] = -sum [t log(1e-6 + p) + (1 - t) log(1e-6 + 1 - p)], dL/dp = -(t / (1e-6 + p) - (1 - t) / (1e-6 + 1 - p)).
// dimg is the gradient of sum_b loss[b].  One double atomic per block.
__global__ void __launch_bounds__(256) image_loss_grad_items_kernel(const float* __restrict__ img, const float* __restrict__ target,
                                                                    float* __restrict__ dimg, double* __restrict__ loss, long long m,
                                                                    int kind) {
  __shared__ double red[256];
  const long long base = static_cast<long long>(blockIdx.y) * m;
  double s = 0.0;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const float inv_m = 1.0f / static_cast<float>(m);
  for (long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; j < m; j += stride) {
    const long long i = base + j;
    const float p = img[i], t = target[i];
    if (kind == 0) {
      const float d = p - t;
      s += static_cast<double>(d) * d;
      if (dimg) dimg[i] = 2.0f * d * inv_m;
    } else {
      const float a = 1e-6f + p, b = 1e-6f + 1.0f - p;
      s -= static_cast<double>(t * logf(a) + (1.0f - t) * logf(b));
      if (dimg) dimg[i] = -(t / a - (1.0f - t) / b);
    }
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(loss + blockIdx.y, kind == 0 ? red[0] / static_cast<double>(m) : red[0]);
}

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, long long n, float lr_t, float beta1, float beta2, float eps) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = g[i];
    const float mi = m[i] + (gi - m[i]) * (1.0f - beta1);           // tf.train.AdamOptimizer: m += (g - m) (1 - beta1)
    const float vi = v[i] + (gi * gi - v[i]) * (1.0f - beta2);      //                         v += (g^2 - v) (1 - beta2)
    m[i] = mi;
    v[i] = vi;
    p[i] -= lr_t * mi / (sqrtf(vi) + eps);                          //                         var -= lr_t m / (sqrt(v) + eps)
  }
}

// Shape fit (rn_voxel_fit_grad): one thread per voxel i = (a*S + b)*S + c of the shared grid.  R_s takes the pairs (i, i+1) along
// each axis once, from their lower voxel; dR_s/docc_i = (2/N) sum over i's in-grid axis neighbours j of (occ_i - occ_j).  The sum
// over views runs v = 0..V-1 in double.  Each block writes its (R_s, R_b) partial sums; voxel_fit_reg_kernel adds them in order.
__global__ void __launch_bounds__(256) voxel_fit_grad_kernel(const float* __restrict__ dvox, const float* __restrict__ occ,
                                                             const unsigned char* __restrict__ keep, float* __restrict__ g,
                                                             double* __restrict__ part, int V, int S, double ls, double lb) {
  __shared__ double red[2][256];
  const long long n = static_cast<long long>(S) * S * S, ss = static_cast<long long>(S) * S;
  const double inv_n = 1.0 / static_cast<double>(n);
  double rs = 0.0, rb = 0.0;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned iu = static_cast<unsigned>(i), su = static_cast<unsigned>(S);        // n <= 2^30
    const int c = static_cast<int>(iu % su), b = static_cast<int>((iu / su) % su), a = static_cast<int>(iu / (su * su));
    const double o = occ[i];
    double ds = 0.0;
    auto axis = [&](int p, long long step) {
      if (p + 1 < S) {
        const double d = o - static_cast<double>(occ[i + step]);
        rs += d * d;
        ds += d;
      }
      if (p > 0) ds += o - static_cast<double>(occ[i - step]);
    };
    axis(c, 1);
    axis(b, S);
    axis(a, ss);
    rb += o * (1.0 - o);
    if (keep && !keep[i]) {
      g[i] = 0.0f;
      continue;
    }
    double s = 0.0;
    for (int v = 0; v < V; ++v) s += static_cast<double>(dvox[static_cast<long long>(v) * n + i]);
    g[i] = static_cast<float>(s + (ls * 2.0 * ds + lb * (1.0 - 2.0 * o)) * inv_n);
  }
  red[0][threadIdx.x] = rs;
  red[1][threadIdx.x] = rb;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      red[0][threadIdx.x] += red[0][threadIdx.x + w];
      red[1][threadIdx.x] += red[1][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = red[0][0];
    part[2 * blockIdx.x + 1] = red[1][0];
  }
}

__global__ void __launch_bounds__(256) voxel_fit_reg_kernel(const double* __restrict__ part, int nblocks, double* __restrict__ reg,
                                                            double inv_n) {
  __shared__ double red[2][256];
  double rs = 0.0, rb = 0.0;
  for (int k = threadIdx.x; k < nblocks; k += blockDim.x) {
    rs += part[2 * k];
    rb += part[2 * k + 1];
  }
  red[0][threadIdx.x] = rs;
  red[1][threadIdx.x] = rb;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      red[0][threadIdx.x] += red[0][threadIdx.x + w];
      red[1][threadIdx.x] += red[1][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    reg[0] = red[0][0] * inv_n;
    reg[1] = red[1][0] * inv_n;
  }
}

// blocks of voxel_fit_grad_kernel: a function of S alone, so the partial sums (and the result) do not depend on the device
inline int voxel_fit_blocks(int S) {
  const long long n = static_cast<long long>(S) * S * S;
  const long long b = (n + 1023) / 1024;
  return static_cast<int>(b < 1 ? 1 : (b > 1024 ? 1024 : b));
}

inline int grid_for(long long n, int block, int cap = 132 * 16) {
  long long g = (n + block - 1) / block;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}
}  // namespace

extern "C" int rn_conv_weight_grad_direct(const void* P, const void* Q, float* dW, int B, int Dp, int Hp, int Wp, int Ca, int Cap,
                                          int Dq, int Hq, int Wq, int Cb, int Cbp, int kd, int kh, int kw, int sd, int sh, int sw,
                                          int pd, int ph, int pw, int fmtP, int fmtQ, float scale, void* stream) {
  if (!P || !Q || !dW || B < 1 || Dp < 1 || Hp < 1 || Wp < 1 || Dq < 1 || Hq < 1 || Wq < 1) return -1;
  if (Ca < 1 || Cb < 1 || Cap < Ca || Cbp < Cb || kd < 1 || kh < 1 || kw < 1 || sd < 1 || sh < 1 || sw < 1) return -1;
  if (fmtP < 0 || fmtP > 3 || fmtQ < 0 || fmtQ > 3) return -1;
  const long long taps = static_cast<long long>(kd) * kh * kw;
  if (taps > 65535) return -2;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(dW, 0, static_cast<size_t>(taps) * Ca * Cb * sizeof(float), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  WgradDirectParams p;
  p.P = P; p.Q = Q; p.dW = dW;
  p.B = B; p.Dp = Dp; p.Hp = Hp; p.Wp = Wp; p.Ca = Ca; p.Cap = Cap; p.Dq = Dq; p.Hq = Hq; p.Wq = Wq; p.Cb = Cb; p.Cbp = Cbp;
  p.kd = kd; p.kh = kh; p.kw = kw; p.sd = sd; p.sh = sh; p.sw = sw; p.pd = pd; p.ph = ph; p.pw = pw;
  p.fmtP = fmtP; p.fmtQ = fmtQ;
  p.npos = static_cast<long long>(B) * Dp * Hp * Wp;
  p.planeP = p.npos * Cap;
  p.planeQ = static_cast<long long>(B) * Dq * Hq * Wq * Cbp;
  p.a_tiles = (Ca + kTile - 1) / kTile;
  p.b_tiles = (Cb + kTile - 1) / kTile;
  p.scale = scale;
  // thin layers: per-thread channel blocks, positions across threads.  Shader: e_conv1 (8,1), e_conv11 (16,3); Texture+Normal:
  // e_tex_conv0 (4,4), e_tex_conv1 / e_tex_conv2 (4,8), e_conv1 (8,5)
  const bool thin = (Ca == 8 && Cb == 1) || (Ca == 16 && Cb == 3) || (Ca == 4 && Cb == 4) || (Ca == 4 && Cb == 8) ||
                    (Ca == 8 && Cb == 5);
  if (thin) {
    long long nsplit = (132LL * 8 + taps - 1) / taps;
    const long long maxsplit = (p.npos + 255) / 256;
    if (nsplit > maxsplit) nsplit = maxsplit;
    if (nsplit < 1) nsplit = 1;
    dim3 grid(static_cast<unsigned>(nsplit), static_cast<unsigned>(taps));
    if (Ca == 8 && Cb == 1) wgrad_thin_kernel<8, 1><<<grid, 256, 0, st>>>(p);
    else if (Ca == 16) wgrad_thin_kernel<16, 3><<<grid, 256, 0, st>>>(p);
    else if (Ca == 4 && Cb == 4) wgrad_thin_kernel<4, 4><<<grid, 256, 0, st>>>(p);
    else if (Ca == 4) wgrad_thin_kernel<4, 8><<<grid, 256, 0, st>>>(p);
    else wgrad_thin_kernel<8, 5><<<grid, 256, 0, st>>>(p);
    RN_COUNT_LAUNCH();
    return static_cast<int>(cudaGetLastError());
  }
  const long long tiles = taps * p.a_tiles * p.b_tiles;
  const long long nchunks = (p.npos + kChunk - 1) / kChunk;
  long long nsplit = (132LL * 8 + tiles - 1) / tiles;               // ~8 CTAs per SM in flight
  if (nsplit < 1) nsplit = 1;
  if (nsplit > nchunks) nsplit = nchunks;
  if (p.a_tiles * p.b_tiles > 65535) return -2;
  dim3 grid(static_cast<unsigned>(nsplit), static_cast<unsigned>(p.a_tiles * p.b_tiles), static_cast<unsigned>(taps));
  wgrad_direct_kernel<<<grid, 256, 0, st>>>(p);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_prelu_alpha_grad(const void* g, const void* z, float* dalpha, long long n, int C, int fmt, float scale,
                                   void* stream) {
  if (!g || !z || !dalpha || n < 1 || C < 1 || C > 8192 || n % C != 0 || fmt < 0 || fmt > 2) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(dalpha, 0, static_cast<size_t>(C) * sizeof(float), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  prelu_alpha_grad_kernel<<<grid_for(n, 256 * 16), 256, static_cast<size_t>(C) * sizeof(float), st>>>(g, z, dalpha, n, C, fmt, scale);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_fully_connected_param_grad(const float* x, const float* gy, const float* z, const float* alpha, float* gz,
                                             float* dw, float* db, float* dalpha, int B, int K, int N, void* stream) {
  const bool ident = !z && !alpha && !dalpha;                                   // FC without activation: gz = gy
  if (!x || !gy || !dw || !db || B < 1 || K < 1 || N < 1) return -1;
  if (!ident && (!z || !alpha || !dalpha)) return -1;
  if (B > 32) return -2;
  if (N % 4 != 0) return -3;
  for (const void* q : {static_cast<const void*>(gy), static_cast<const void*>(z), static_cast<const void*>(alpha),
                        static_cast<const void*>(gz), static_cast<const void*>(dw), static_cast<const void*>(db),
                        static_cast<const void*>(dalpha)})
    if ((reinterpret_cast<uintptr_t>(q) & 15) != 0) return -3;                   // float4 rows
  const int kparts = (K + 63) / 64;
  const int kchunk = (K + kparts - 1) / kparts;
  const int BT = B <= 4 ? 4 : B <= 8 ? 8 : B <= 16 ? 16 : B <= 24 ? 24 : 32;
  const size_t smem = static_cast<size_t>(BT) * kchunk * sizeof(float);           // <= 8 KB
  const dim3 grid(static_cast<unsigned>(kparts), static_cast<unsigned>((N / 4 + 127) / 128));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define RN_FCPG(T) fc_param_grad_kernel<T><<<grid, 128, smem, st>>>(x, gy, z, alpha, gz, dw, db, dalpha, B, K, N, kchunk)
  switch (BT) {
    case 4: RN_FCPG(4); break;
    case 8: RN_FCPG(8); break;
    case 16: RN_FCPG(16); break;
    case 24: RN_FCPG(24); break;
    default: RN_FCPG(32); break;
  }
#undef RN_FCPG
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_prelu_grad_f32(const float* gy, const float* z, const float* alpha, float* gz, float* db, float* dalpha,
                                 long long n, int C, void* stream) {
  if (!gy || !z || !alpha || !gz || !db || !dalpha || n < 1 || n % C != 0) return -1;
  if (C != 4 && C != 8) return -2;
  for (const float* q : {gy, z, static_cast<const float*>(gz)})
    if ((reinterpret_cast<uintptr_t>(q) & 15) != 0) return -3;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(db, 0, static_cast<size_t>(C) * sizeof(float), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(dalpha, 0, static_cast<size_t>(C) * sizeof(float), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long nvox = n / C;
  const int grid = grid_for(nvox, 256 * 8, 132 * 8);
  if (C == 4) prelu_grad_f32_kernel<4><<<grid, 256, 0, st>>>(gy, z, alpha, gz, db, dalpha, nvox);
  else prelu_grad_f32_kernel<8><<<grid, 256, 0, st>>>(gy, z, alpha, gz, db, dalpha, nvox);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_dropout_16(const void* x, void* out, long long n, float keep, unsigned seed, unsigned salt, int fmt,
                             void* stream) {
  if (!x || !out || n < 0 || !(keep > 0.f) || keep > 1.f || fmt < 0 || fmt > 2) return -1;
  if (n == 0) return 0;
  dropout_kernel<<<grid_for(n, 256 * 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, n, keep, rn_dropout_threshold(keep),
                                                                                     seed, salt, fmt);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_image_loss_grad(const float* img, const float* target, float* dimg, double* loss, long long n, int batch,
                                  int kind, void* stream) {
  if (!img || !target || !loss || n < 1 || batch < 1 || (kind != 0 && kind != 1)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(double), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  image_loss_grad_kernel<<<grid_for(n, 256 * 8, 132 * 4), 256, 0, st>>>(img, target, dimg, loss, n, batch, kind);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_image_loss_grad_items(const float* img, const float* target, float* dimg, double* loss, long long npix, int C,
                                        int batch, int kind, void* stream) {
  if (!img || !target || !loss || npix < 1 || (C != 1 && C != 3) || batch < 1 || batch > 65535 || (kind != 0 && kind != 1))
    return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(loss, 0, static_cast<size_t>(batch) * sizeof(double), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long m = npix * C;
  const int per_item = (132 * 4 + batch - 1) / batch;
  const dim3 grid(static_cast<unsigned>(grid_for(m, 256 * 8, per_item)), static_cast<unsigned>(batch));
  image_loss_grad_items_kernel<<<grid, 256, 0, st>>>(img, target, dimg, loss, m, kind);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_adam_step(float* param, const float* grad, float* m, float* v, long long n, float lr_t, float beta1, float beta2,
                            float eps, void* stream) {
  if (!param || !grad || !m || !v || n < 0) return -1;
  if (n == 0) return 0;
  adam_kernel<<<grid_for(n, 256 * 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(param, grad, m, v, n, lr_t, beta1, beta2, eps);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

extern "C" long long rn_voxel_fit_grad_workspace(int S) {
  if (S < 1 || S > 1024) return -1;
  return 2LL * voxel_fit_blocks(S);
}

extern "C" int rn_voxel_fit_grad(const float* dvox, const float* occ, const unsigned char* keep, float* g, double* reg, double* work,
                                 int V, int S, float lambda_smooth, float lambda_bin, void* stream) {
  if (!dvox || !occ || !g || !reg || !work || V < 1 || S < 1 || S > 1024) return -1;
  if (!(lambda_smooth >= 0.f) || !(lambda_bin >= 0.f) || isinf(lambda_smooth) || isinf(lambda_bin)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nb = voxel_fit_blocks(S);
  voxel_fit_grad_kernel<<<nb, 256, 0, st>>>(dvox, occ, keep, g, work, V, S, lambda_smooth, lambda_bin);
  RN_COUNT_LAUNCH();
  voxel_fit_reg_kernel<<<1, 256, 0, st>>>(work, nb, reg, 1.0 / (static_cast<double>(S) * S * S));
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

// host-side restatement of the dropout mask (tests and data pipelines that must reproduce a step's masks): 1 = kept
extern "C" int rn_dropout_mask_host(unsigned char* mask, long long n, float keep, unsigned seed, unsigned salt) {
  if (!mask || n < 0 || !(keep > 0.f) || keep > 1.f) return -1;
  const unsigned long long thr = rn_dropout_threshold(keep);
  for (long long i = 0; i < n; ++i) mask[i] = rn_dropout_hash(seed, salt, static_cast<unsigned long long>(i)) < thr ? 1 : 0;
  return 0;
}
