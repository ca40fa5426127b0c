// rn_decoder3d.cu -- fp32 3-D convolutions with 16..256 channels and a cubic 4^3 kernel: the face-reconstruction shape decoder
// (Reconstruct_RenderNet_Face.py:31-75, decoder_3d_pretrained: four conv3d_transpose k4 s2 + ELU, one conv3d_transpose k4 s1 +
// sigmoid) and its data gradients, which TF defines as conv3d on the same filter arrays.  fp32 on the CUDA cores in both precision
// modes, like the texture decoder: the reference computes in fp32 and the decoder is ~2.3 GMAC per item.
//
// Implicit GEMM: M = output voxels, N = Cout, K = taps x Cin.  Operand tiles are staged in shared memory (A gathered from the
// channel-last input, B read from the TF-layout filter), the next tile is prefetched into registers while the current one is
// multiplied, and each thread accumulates a TM x TN register micro-tile.  A stride-2 transposed conv is split into its 8 output
// phases (gridDim.z): each phase is a dense 2^3-tap convolution over the input grid, so no structural zero is multiplied.
// Small-M layers split K over CTAs and sum the slices in a fixed order in a second kernel: no float atomics, the result is
// reproducible bit for bit.
//
// Weight gradients (fine-tuning the decoder, decoder_3d_pretrained(trainable=True)): the same phase decomposition turned around.
// Per phase, dW is a GEMM with M = taps x Cin, N = Cout and K = the phase's voxel rows (A gathered from the layer input at the
// tap's offset, B = dL/d(pre-activation) at the phase's output voxels); each of the 64 filter taps belongs to exactly one phase,
// so the phases write disjoint slices of dW.  K is split over CTAs to fill the SMs, the slices are summed in a fixed order by a
// second kernel, which also sums the bias gradient the first kernel took from its staged B tiles.  The 1-channel output layer
// (g_conv5) has a direct kernel of its own, like its forward.
#include <cstdint>
#include <cuda_runtime.h>

#include <atomic>

#include "../../include/rendernet_b200.h"

namespace rn {
extern std::atomic<long long> g_launch_count;
#define RN_COUNT_LAUNCH() rn::g_launch_count.fetch_add(1, std::memory_order_relaxed)

namespace {
// Geometry of one call.  mode: 0 = conv3d_transpose s2 (8 phases, 2^3 taps), 1 = conv3d_transpose s1, 2 = conv3d s2,
// 3 = conv3d s1 (64 taps).  M rows of a phase enumerate (b, my, mx, mz) over (Mh, Mw, Md); output voxel = (my*os + py, ...).
struct Geo {
  int mode, B, H, W, D, Cin, Cout;      // input grid and channels
  int Ho, Wo, Do;                       // output grid
  int Mh, Mw, Md;                       // per-phase row grid
  int T, ntaps, os, is, pb;             // taps per axis, total taps, output-phase stride, input stride, SAME pad-before
  long long M;                          // rows per phase
  int K;                                // ntaps * Cin
};

// input offset and filter index of tap t along one axis for output phase ph
__device__ __forceinline__ void tap_axis(const Geo& g, int t, int ph, int* off, int* k) {
  if (g.mode == 0) { *k = 2 * t + 1 - ph; *off = ph - t; }        // o = 2i + k - 1, o = 2m + ph
  else if (g.mode == 1) { *k = t; *off = g.pb - t; }               // o = i + k - pb
  else { *k = t; *off = t - g.pb; }                                // i = o*s + k - pb
}

__device__ __forceinline__ float act_fwd(float v, int act) {
  if (act == RN_ACT_ELU) return v < 0.f ? expf(v) - 1.f : v;                    // TF-1 Elu: exp(x) - 1, not expm1
  if (act == RN_ACT_SIGMOID) return 1.f / (1.f + expf(-v));
  return v;
}

// A row = (b, my, mx, mz) packed into one int (7 bits per coordinate, b above them); -1 = past the last row
__device__ __forceinline__ int pack_row(const Geo& g, long long m) {
  if (m >= g.M) return -1;
  const int mz = static_cast<int>(m % g.Md); m /= g.Md;
  const int mx = static_cast<int>(m % g.Mw); m /= g.Mw;
  const int my = static_cast<int>(m % g.Mh);
  const int b = static_cast<int>(m / g.Mh);
  return (b << 21) | (my << 14) | (mx << 7) | mz;
}

// B element (column kk, output channel co) from the TF-layout filter: transposed [4,4,4,Cout,Cin], forward [4,4,4,Cin,Cout]
__device__ __forceinline__ float load_b(const float* __restrict__ w, const Geo& g, int py, int px, int pz, int kk, int co) {
  const int tap = kk / g.Cin, ci = kk - tap * g.Cin;
  const int tz = tap % g.T, tx = (tap / g.T) % g.T, ty = tap / (g.T * g.T);
  int d, ky, kx, kz;
  tap_axis(g, ty, py, &d, &ky);
  tap_axis(g, tx, px, &d, &kx);
  tap_axis(g, tz, pz, &d, &kz);
  const int kidx = (ky * 4 + kx) * 4 + kz;
  if (g.mode <= 1) return __ldg(w + ((static_cast<long long>(kidx) * g.Cout + co) * g.Cin + ci));
  return __ldg(w + ((static_cast<long long>(kidx) * g.Cin + ci) * g.Cout + co));
}

// blockIdx.x = M tile, blockIdx.y = N tile, blockIdx.z = phase * splits + split.  splits == 1: bias + activation, write out.
// splits > 1: write the raw partial sum of K slice `split` to part[split][phase-row][co] (fixed-order reduction follows).
template <int BM, int BN, int TM, int TN, int BK>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) conv3d_f32_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                            const float* __restrict__ bias, float* __restrict__ out,
                                                                            float* __restrict__ part, Geo g, int splits,
                                                                            int kslice, int act) {
  constexpr int NT = (BM / TM) * (BN / TN);
  static_assert(NT % BK == 0 && (BM * BK) % NT == 0, "each thread loads one A column of the tile");
  constexpr int LA = BM * BK / NT;
  constexpr int RS = NT / BK;                      // row step between a thread's A loads
  constexpr int LB = (BN * BK + NT - 1) / NT;
  constexpr int AP = BM + 4;                       // padded row of the k-major A tile (float4 reads stay aligned)
  __shared__ __align__(16) float As[BK][AP];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x;
  const int phase = blockIdx.z / splits, split = blockIdx.z - phase * splits;
  const int py = phase >> 2, px = (phase >> 1) & 1, pz = phase & 1;
  const long long m0 = static_cast<long long>(blockIdx.x) * BM;
  const int n0 = blockIdx.y * BN;
  const int k_begin = split * kslice;
  const int k_end = min(g.K, k_begin + kslice);

  // A: this thread loads column kq of the tile for rows tid / BK + i * RS (fixed for the whole K loop)
  const int kq = tid % BK, r0 = tid / BK;
  int rows[LA];
#pragma unroll
  for (int i = 0; i < LA; ++i) rows[i] = pack_row(g, m0 + r0 + i * RS);
  const long long plane_b = static_cast<long long>(g.H) * g.W * g.D;
  // B tile mapping: filter-contiguous index fastest (ci for the transposed layout, co for the forward one)
  const bool b_k_fast = g.mode <= 1;
  float ra[LA], rbv[LB];
  auto fetch = [&](int k0) {
    const int kk = k0 + kq;
    const bool kin = kk < k_end;
    int oy = 0, ox = 0, oz = 0, ci = 0;
    if (kin) {                                     // the tap and channel of column kk: shared by all of this thread's rows
      const int tap = kk / g.Cin;
      ci = kk - tap * g.Cin;
      int kd;
      tap_axis(g, tap / (g.T * g.T), py, &oy, &kd);
      tap_axis(g, (tap / g.T) % g.T, px, &ox, &kd);
      tap_axis(g, tap % g.T, pz, &oz, &kd);
    }
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int r = rows[i];
      float v = 0.f;
      if (kin && r >= 0) {
        const int iy = ((r >> 14) & 127) * g.is + oy, ix = ((r >> 7) & 127) * g.is + ox, iz = (r & 127) * g.is + oz;
        if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W && iz >= 0 && iz < g.D)
          v = __ldg(x + (((r >> 21) * plane_b + (static_cast<long long>(iy) * g.W + ix) * g.D + iz) * g.Cin + ci));
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int e = tid + i * NT;
      int kl, nl;
      if (b_k_fast) { nl = e / BK; kl = e - nl * BK; } else { kl = e / BN; nl = e - kl * BN; }
      const int kk = k0 + kl, co = n0 + nl;
      rbv[i] = (e < BN * BK && kk < k_end && co < g.Cout) ? load_b(w, g, py, px, pz, kk, co) : 0.f;
    }
  };
  auto stash = [&]() {
#pragma unroll
    for (int i = 0; i < LA; ++i) As[kq][r0 + i * RS] = ra[i];
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int e = tid + i * NT;
      if (e >= BN * BK) continue;
      int kl, nl;
      if (b_k_fast) { nl = e / BK; kl = e - nl * BK; } else { kl = e / BN; nl = e - kl * BN; }
      Bs[kl][nl] = rbv[i];
    }
  };

  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  fetch(k_begin);
  for (int k0 = k_begin; k0 < k_end; k0 += BK) {
    __syncthreads();
    stash();
    __syncthreads();
    if (k0 + BK < k_end) fetch(k0 + BK);           // global loads of the next tile overlap the FMAs below
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long m = m0 + ty * TM + i;
    if (m >= g.M) continue;
    long long orow;
    if (splits > 1) {
      orow = (static_cast<long long>(split) * 8 + phase) * g.M + m;     // partial-sum row
    } else {
      long long q = m;
      const int mz = static_cast<int>(q % g.Md); q /= g.Md;
      const int mx = static_cast<int>(q % g.Mw); q /= g.Mw;
      const int my = static_cast<int>(q % g.Mh);
      const int b = static_cast<int>(q / g.Mh);
      const int oy = my * g.os + py, ox = mx * g.os + px, oz = mz * g.os + pz;
      orow = ((static_cast<long long>(b) * g.Ho + oy) * g.Wo + ox) * g.Do + oz;
    }
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int co = n0 + tx * TN + j;
      if (co >= g.Cout) continue;
      if (splits > 1) part[orow * g.Cout + co] = acc[i][j];
      else out[orow * g.Cout + co] = act_fwd(acc[i][j] + (bias != nullptr ? __ldg(bias + co) : 0.f), act);
    }
  }
}

// out = act(sum_{s = 0..splits-1} part[s] + bias), summed in split order
__global__ void conv3d_f32_reduce_kernel(const float* __restrict__ part, const float* __restrict__ bias, float* __restrict__ out,
                                         Geo g, int nphase, int splits, int act) {
  const long long per = g.M * g.Cout;
  const long long total = per * nphase;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int phase = static_cast<int>(e / per);
    const long long r = e - phase * per;
    const long long m = r / g.Cout;
    const int co = static_cast<int>(r - m * g.Cout);
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[(static_cast<long long>(s) * 8 + phase) * per + r];
    const int py = phase >> 2, px = (phase >> 1) & 1, pz = phase & 1;
    long long q = m;
    const int mz = static_cast<int>(q % g.Md); q /= g.Md;
    const int mx = static_cast<int>(q % g.Mw); q /= g.Mw;
    const int my = static_cast<int>(q % g.Mh);
    const int b = static_cast<int>(q / g.Mh);
    const long long o = ((static_cast<long long>(b) * g.Ho + my * g.os + py) * g.Wo + mx * g.os + px) * g.Do + mz * g.os + pz;
    out[o * g.Cout + co] = act_fwd(v + (bias != nullptr ? __ldg(bias + co) : 0.f), act);
  }
}

// g_conv5 (conv3d_transpose k4 s1, Cin -> 1 channel, :71-74): with N = 1 the implicit GEMM has no operand reuse, so this layer
// runs as a direct convolution instead.  One CTA = an 8 x 8 x 16 output tile; the 11 x 11 x 19 input tile is staged in shared
// memory 4 channels at a time (z rows contiguous), the filter once; each thread computes 4 consecutive z outputs from a 7-wide
// register window.  o = i + k - 1, so output o reads inputs o + 1 - k, k = 0..3.  Fixed (channel, ky, kx, kz) order.
constexpr int T5_Y = 8, T5_X = 8, T5_Z = 16, T5_ZP = T5_Z + 4;
__global__ void __launch_bounds__(256) tconv_s1_to1_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ bias, float* __restrict__ out, int B, int H,
                                                           int W, int D, int Cin, int act) {
  __shared__ __align__(16) float xs[4][T5_Y + 3][T5_X + 3][T5_ZP];
  __shared__ float ws[64 * 16];
  const int tid = threadIdx.x;
  const int ntz = D / T5_Z, ntx = W / T5_X, nty = H / T5_Y;
  int t = blockIdx.x;
  const int tz = t % ntz; t /= ntz;
  const int tx = t % ntx; t /= ntx;
  const int ty = t % nty;
  const int b = t / nty;
  const int y0 = ty * T5_Y - 2, x0 = tx * T5_X - 2, z0 = tz * T5_Z - 2;      // input origin of the tile
  for (int i = tid; i < 64 * Cin; i += 256) ws[i] = w[i];                    // [4,4,4,1,Cin]
  const int ly = tid >> 5, lx = (tid >> 2) & 7, lz = (tid & 3) * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  constexpr int NV = (T5_Y + 3) * (T5_X + 3) * (T5_Z + 3);
  for (int c0 = 0; c0 < Cin; c0 += 4) {
    __syncthreads();
    for (int e = tid; e < NV; e += 256) {
      const int zz = e % (T5_Z + 3), xx = (e / (T5_Z + 3)) % (T5_X + 3), yy = e / ((T5_Z + 3) * (T5_X + 3));
      const int iy = y0 + yy, ix = x0 + xx, iz = z0 + zz;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < H && ix >= 0 && ix < W && iz >= 0 && iz < D)
        v = __ldg(reinterpret_cast<const float4*>(x + ((((static_cast<long long>(b) * H + iy) * W + ix) * D + iz) * Cin + c0)));
      xs[0][yy][xx][zz] = v.x; xs[1][yy][xx][zz] = v.y; xs[2][yy][xx][zz] = v.z; xs[3][yy][xx][zz] = v.w;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 4; ++c) {
#pragma unroll
      for (int ky = 0; ky < 4; ++ky) {
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) {
          const float* row = &xs[c][ly + 3 - ky][lx + 3 - kx][lz];
          float r[7];
#pragma unroll
          for (int j = 0; j < 7; ++j) r[j] = row[j];
#pragma unroll
          for (int kz = 0; kz < 4; ++kz) {
            const float wv = ws[((ky * 4 + kx) * 4 + kz) * Cin + c0 + c];
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[j] = fmaf(r[j + 3 - kz], wv, acc[j]);
          }
        }
      }
    }
  }
  const float bv = bias != nullptr ? __ldg(bias) : 0.f;
  const long long o = (((static_cast<long long>(b) * H + ty * T5_Y + ly) * W + tx * T5_X + lx) * D + tz * T5_Z + lz);
#pragma unroll
  for (int j = 0; j < 4; ++j) out[o + j] = act_fwd(acc[j] + bv, act);
}

__global__ void act_backward_f32_kernel(const float* __restrict__ g, const float* __restrict__ y, float* __restrict__ out,
                                        long long n, int act) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gv = g[i], yv = y[i];
    // TF-1 EluGrad(g, y): y < 0 ? g * (y + 1) : g;  SigmoidGrad(y, g): g * y * (1 - y)
    out[i] = act == RN_ACT_ELU ? (yv < 0.f ? gv * (yv + 1.f) : gv) : gv * yv * (1.f - yv);
  }
}

// ---------------------------------------------------------------------------------------------------------- weight gradients
// Filter index of tap `tap` (0 .. ntaps-1) of phase (py, px, pz).
__device__ __forceinline__ int tap_kidx(const Geo& g, int tap, int py, int px, int pz) {
  int d, ky, kx, kz;
  tap_axis(g, tap / (g.T * g.T), py, &d, &ky);
  tap_axis(g, (tap / g.T) % g.T, px, &d, &kx);
  tap_axis(g, tap % g.T, pz, &d, &kz);
  return (ky * 4 + kx) * 4 + kz;
}

// blockIdx.x = M tile (M = (tap, ci) of the phase), blockIdx.y = N tile (co), blockIdx.z = phase * splits + split.
//   part[split][phase][m][co] = sum over rows r of the slice  x[input voxel of r at tap][ci] * gz[output voxel of r][co]
// Rows are decoded once per K tile into rowv (double-buffered: the next tile's rows are decoded while this one is multiplied).
// The CTAs of M tile 0 also sum their staged gz tiles: dbpart[split][phase][co].
template <int BM, int BN, int TM, int TN, int BK>
__global__ void __launch_bounds__((BM / TM) * (BN / TN), 2) conv3d_f32_wgrad_kernel(const float* __restrict__ x,
                                                                                    const float* __restrict__ gz,
                                                                                    float* __restrict__ part,
                                                                                    float* __restrict__ dbpart, Geo g,
                                                                                    int splits, long long kslice) {
  constexpr int NT = (BM / TM) * (BN / TN);
  static_assert(NT % BM == 0 && NT % BN == 0 && (BM * BK) % NT == 0 && BK <= NT, "fixed (m, co) per loading thread");
  constexpr int LA = BM * BK / NT, RA = NT / BM;             // A: this thread's column m, rows tid / BM + i * RA
  constexpr int RB = NT / BN, LB = (BK + RB - 1) / RB;       // B: this thread's column co, rows tid / BN + i * RB
  constexpr int AP = BM + 4;
  __shared__ __align__(16) float As[BK][AP];
  __shared__ __align__(16) float Bs[BK][BN];
  __shared__ int rowv[2][BK];
  const int tid = threadIdx.x;
  const int nphase = g.mode == 0 ? 8 : 1;
  const int phase = blockIdx.z / splits, split = blockIdx.z - phase * splits;
  const int py = phase >> 2, px = (phase >> 1) & 1, pz = phase & 1;
  const int Mt = g.ntaps * g.Cin;
  const long long k_begin = static_cast<long long>(split) * kslice;
  const long long k_end = min(g.M, k_begin + kslice);
  const int nk = k_end > k_begin ? static_cast<int>((k_end - k_begin + BK - 1) / BK) : 0;

  const int ml = tid % BM, m = blockIdx.x * BM + ml;
  const bool m_in = m < Mt;
  int oy = 0, ox = 0, oz = 0, ci = 0;
  if (m_in) {
    const int tap = m / g.Cin;
    ci = m - tap * g.Cin;
    int kd;
    tap_axis(g, tap / (g.T * g.T), py, &oy, &kd);
    tap_axis(g, (tap / g.T) % g.T, px, &ox, &kd);
    tap_axis(g, tap % g.T, pz, &oz, &kd);
  }
  const int nl = tid % BN, co = blockIdx.y * BN + nl;
  const bool n_in = co < g.Cout;
  const long long plane_b = static_cast<long long>(g.H) * g.W * g.D;
  auto decode = [&](long long r) { return r < k_end ? pack_row(g, r) : -1; };

  float ra[LA], rb[LB];
  auto fetch = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int r = rowv[buf][tid / BM + i * RA];
      float v = 0.f;
      if (m_in && r >= 0) {
        const int iy = ((r >> 14) & 127) * g.is + oy, ix = ((r >> 7) & 127) * g.is + ox, iz = (r & 127) * g.is + oz;
        if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W && iz >= 0 && iz < g.D)
          v = __ldg(x + (((r >> 21) * plane_b + (static_cast<long long>(iy) * g.W + ix) * g.D + iz) * g.Cin + ci));
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int kl = tid / BN + i * RB;
      float v = 0.f;
      if (kl < BK && n_in) {
        const int r = rowv[buf][kl];
        if (r >= 0) {
          const long long o = ((static_cast<long long>(r >> 21) * g.Ho + ((r >> 14) & 127) * g.os + py) * g.Wo +
                               ((r >> 7) & 127) * g.os + px) * g.Do + (r & 127) * g.os + pz;
          v = __ldg(gz + o * g.Cout + co);
        }
      }
      rb[i] = v;
    }
  };

  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  const bool db_cta = blockIdx.x == 0 && tid < BN;
  float dbacc = 0.f;

  if (tid < BK) rowv[0][tid] = decode(k_begin + tid);
  __syncthreads();
  fetch(0);
  for (int t = 0; t < nk; ++t) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < LA; ++i) As[tid / BM + i * RA][ml] = ra[i];
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int kl = tid / BN + i * RB;
      if (kl < BK) Bs[kl][nl] = rb[i];
    }
    if (tid < BK) rowv[(t + 1) & 1][tid] = decode(k_begin + static_cast<long long>(t + 1) * BK + tid);
    __syncthreads();
    if (t + 1 < nk) fetch((t + 1) & 1);            // global loads of the next tile overlap the FMAs below
    if (db_cta) {
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) dbacc += Bs[kk][tid];
    }
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
      if constexpr (TM % 4 == 0) {
#pragma unroll
        for (int i = 0; i < TM; i += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
          a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
      }
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }

  const long long slab = static_cast<long long>(split) * nphase + phase;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int mm = blockIdx.x * BM + ty * TM + i;
    if (mm >= Mt) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int c = blockIdx.y * BN + tx * TN + j;
      if (c < g.Cout) part[(slab * Mt + mm) * g.Cout + c] = acc[i][j];
    }
  }
  if (db_cta && n_in) dbpart[slab * g.Cout + co] = dbacc;
}

// dw[kidx] = sum_{s = 0..splits-1} part[s][phase][m] in split order, scattered to the TF filter layout ([4,4,4,Cout,Cin]
// transposed, [4,4,4,Cin,Cout] forward); block 0 also sums db[co] over (phase, split) in that order.
__global__ void conv3d_f32_wgrad_reduce_kernel(const float* __restrict__ part, const float* __restrict__ dbpart, float* __restrict__ dw,
                                               float* __restrict__ db, Geo g, int nphase, int splits) {
  const int Mt = g.ntaps * g.Cin;
  const long long per = static_cast<long long>(Mt) * g.Cout;
  const long long slab = per * nphase;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < slab;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int phase = static_cast<int>(e / per);
    const long long r = e - phase * per;
    const int m = static_cast<int>(r / g.Cout);
    const int co = static_cast<int>(r - static_cast<long long>(m) * g.Cout);
    float v = 0.f;
#pragma unroll 8
    for (int s = 0; s < splits; ++s) v += part[s * slab + e];
    const int tap = m / g.Cin, ci = m - tap * g.Cin;
    const int kidx = tap_kidx(g, tap, phase >> 2, (phase >> 1) & 1, phase & 1);
    if (g.mode <= 1) dw[(static_cast<long long>(kidx) * g.Cout + co) * g.Cin + ci] = v;
    else dw[(static_cast<long long>(kidx) * g.Cin + ci) * g.Cout + co] = v;
  }
  if (blockIdx.x == 0) {
    for (int co = threadIdx.x; co < g.Cout; co += blockDim.x) {
      float v = 0.f;
      for (int p = 0; p < nphase; ++p)
#pragma unroll 8
        for (int s = 0; s < splits; ++s) v += dbpart[(static_cast<long long>(s) * nphase + p) * g.Cout + co];
      db[co] = v;
    }
  }
}

// g_conv5's weight gradient (conv3d_transpose k4 s1, 16 -> 1 channel): with N = 1 the GEMM above reads every input element once
// per tap, so this layer has a direct kernel.  A persistent CTA walks 4 x 4 x 16 output tiles (tile t = blockIdx.x, +gridDim.x,
// ...): the tile's gz and the 7 x 7 x 19 x 16 input halo are staged in shared memory, and thread (ky, kx, ci) accumulates the
// four kz taps  dw[ky][kx][kz][0][ci] += sum_{y,x,z} gz[y,x,z] x[y+1-ky][x+1-kx][z+1-kz][ci]  from a 20-wide register window of
// the input row.  Writes part[blockIdx.x][tap * 16 + ci] and dbpart[blockIdx.x] (the CTA's sum of gz), summed over CTAs in
// order by conv3d_f32_wgrad_reduce_kernel.  The grid size depends on the shape alone: reproducible bit for bit.
constexpr int W5_Y = 4, W5_X = 4, W5_Z = 16, W5_CIN = 16;
constexpr int W5_HY = W5_Y + 3, W5_HX = W5_X + 3, W5_HZ = W5_Z + 3, W5_ZP = W5_Z + 4;
constexpr int W5_CH = W5_HY * W5_HX * W5_ZP;                  // channel stride: 980 floats = 20 mod 32, conflict-free float4 rows
constexpr int W5_SMEM = (W5_CIN * W5_CH + W5_Y * W5_X * W5_Z + 64 * 4) * 4;
constexpr int W5_MAX_CTAS = 3 * 132;
__global__ void __launch_bounds__(256) tconv_s1_to1_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ gz,
                                                                 float* __restrict__ part, float* __restrict__ dbpart, int B, int H,
                                                                 int W, int D) {
  extern __shared__ __align__(16) float smem5[];
  float* xs = smem5;                                          // [16][7][7][20]
  float* gs = smem5 + W5_CIN * W5_CH;                         // [4][4][16]
  float* red = gs + W5_Y * W5_X * W5_Z;                       // [64][4]
  const int tid = threadIdx.x;
  const int ci = tid & 15, kx = (tid >> 4) & 3, ky = tid >> 6;
  const int ntz = D / W5_Z, ntx = W / W5_X, nty = H / W5_Y;
  const int ntiles = B * nty * ntx * ntz;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float4 dbv = make_float4(0.f, 0.f, 0.f, 0.f);               // thread tid < 64: running sum of its float4 of the gz tile
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    int q = t;
    const int tz = q % ntz; q /= ntz;
    const int tx = q % ntx; q /= ntx;
    const int ty = q % nty;
    const int b = q / nty;
    const int y0 = ty * W5_Y - 2, x0 = tx * W5_X - 2, z0 = tz * W5_Z - 2;
    __syncthreads();
    constexpr int NV = W5_HY * W5_HX * W5_HZ * 4;             // float4 quads of the halo
    for (int e = tid; e < NV; e += 256) {
      const int qd = e & 3, v = e >> 2;
      const int zz = v % W5_HZ, xx = (v / W5_HZ) % W5_HX, yy = v / (W5_HZ * W5_HX);
      const int iy = y0 + yy, ix = x0 + xx, iz = z0 + zz;
      float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < H && ix >= 0 && ix < W && iz >= 0 && iz < D)
        val = __ldg(reinterpret_cast<const float4*>(
            x + ((((static_cast<long long>(b) * H + iy) * W + ix) * D + iz) * W5_CIN + qd * 4)));
      float* dst = xs + (qd * 4) * W5_CH + (yy * W5_HX + xx) * W5_ZP + zz;
      dst[0] = val.x; dst[W5_CH] = val.y; dst[2 * W5_CH] = val.z; dst[3 * W5_CH] = val.w;
    }
    if (tid < 64) {                                           // gz tile: 16 rows of 16 z values
      const int row = tid >> 2, zq = (tid & 3) * 4;
      const int oy = ty * W5_Y + (row >> 2), ox = tx * W5_X + (row & 3);
      const float4 v = __ldg(reinterpret_cast<const float4*>(
          gz + (((static_cast<long long>(b) * H + oy) * W + ox) * D + tz * W5_Z + zq)));
      *reinterpret_cast<float4*>(gs + row * W5_Z + zq) = v;
      dbv.x += v.x; dbv.y += v.y; dbv.z += v.z; dbv.w += v.w;
    }
    __syncthreads();
#pragma unroll
    for (int yy = 0; yy < W5_Y; ++yy) {
#pragma unroll
      for (int xx = 0; xx < W5_X; ++xx) {
        const float* xr = xs + ci * W5_CH + ((yy + 3 - ky) * W5_HX + xx + 3 - kx) * W5_ZP;
        const float* gr = gs + (yy * W5_X + xx) * W5_Z;
        float r[W5_ZP], gv[W5_Z];
#pragma unroll
        for (int j = 0; j < W5_ZP; j += 4) {
          const float4 v = *reinterpret_cast<const float4*>(xr + j);
          r[j] = v.x; r[j + 1] = v.y; r[j + 2] = v.z; r[j + 3] = v.w;
        }
#pragma unroll
        for (int j = 0; j < W5_Z; j += 4) {
          const float4 v = *reinterpret_cast<const float4*>(gr + j);
          gv[j] = v.x; gv[j + 1] = v.y; gv[j + 2] = v.z; gv[j + 3] = v.w;
        }
#pragma unroll
        for (int z = 0; z < W5_Z; ++z)
#pragma unroll
          for (int kz = 0; kz < 4; ++kz) acc[kz] = fmaf(gv[z], r[z + 3 - kz], acc[kz]);
      }
    }
  }
#pragma unroll
  for (int kz = 0; kz < 4; ++kz) part[static_cast<long long>(blockIdx.x) * 1024 + ((ky * 4 + kx) * 4 + kz) * W5_CIN + ci] = acc[kz];
  if (tid < 64) *reinterpret_cast<float4*>(red + tid * 4) = dbv;
  __syncthreads();
  if (tid == 0) {
    float v = 0.f;
    for (int i = 0; i < 256; ++i) v += red[i];
    dbpart[blockIdx.x] = v;
  }
}

// Tile shape per output width (N = Cout): 64 x 64 for wide layers, 128 x 32, 256 x 16, and 1024 x 1 for the 1-channel output.
enum { CFG_64x64, CFG_128x32, CFG_256x16, CFG_1024x1 };
struct Plan {
  Geo g;
  int cfg, BM, BN, BK, nphase, splits, kslice;
  long long work;          // floats of split-K workspace (0 without split)
};

int make_plan(int B, int H, int W, int D, int Cin, int Cout, int stride, int transposed, Plan* p) {
  if (B < 1 || B > 32 || H < 1 || W < 1 || D < 1 || Cin < 1 || Cout < 1 || Cin > 512 || Cout > 512) return -1;
  if (stride != 1 && stride != 2) return -2;
  Geo& g = p->g;
  g.B = B; g.H = H; g.W = W; g.D = D; g.Cin = Cin; g.Cout = Cout;
  g.mode = transposed ? (stride == 2 ? 0 : 1) : (stride == 2 ? 2 : 3);
  if (transposed) {
    g.Ho = H * stride; g.Wo = W * stride; g.Do = D * stride;
    g.pb = (4 - stride) / 2;
  } else {
    g.Ho = (H + stride - 1) / stride; g.Wo = (W + stride - 1) / stride; g.Do = (D + stride - 1) / stride;
    const int ty = (g.Ho - 1) * stride + 4 - H, tx = (g.Wo - 1) * stride + 4 - W, tz = (g.Do - 1) * stride + 4 - D;
    if (ty != tx || ty != tz) return -2;           // one SAME pad for all three axes (cubic inputs)
    g.pb = (ty > 0 ? ty : 0) / 2;
  }
  g.T = g.mode == 0 ? 2 : 4;
  g.ntaps = g.T * g.T * g.T;
  g.os = g.mode == 0 ? 2 : 1;
  g.is = g.mode == 2 ? 2 : 1;
  if (g.mode == 0) { g.Mh = H; g.Mw = W; g.Md = D; } else { g.Mh = g.Ho; g.Mw = g.Wo; g.Md = g.Do; }
  if (g.Mh > 127 || g.Mw > 127 || g.Md > 127) return -2;        // 7-bit row coordinates (pack_row)
  g.M = static_cast<long long>(B) * g.Mh * g.Mw * g.Md;
  g.K = g.ntaps * Cin;
  p->nphase = g.mode == 0 ? 8 : 1;
  if (Cout >= 64) { p->cfg = CFG_64x64; p->BM = 64; p->BN = 64; p->BK = 16; }
  else if (Cout >= 24) { p->cfg = CFG_128x32; p->BM = 128; p->BN = 32; p->BK = 16; }
  else if (Cout >= 2) { p->cfg = CFG_256x16; p->BM = 256; p->BN = 16; p->BK = 16; }
  else { p->cfg = CFG_1024x1; p->BM = 1024; p->BN = 1; p->BK = 8; }
  const long long tiles = ((g.M + p->BM - 1) / p->BM) * ((Cout + p->BN - 1) / p->BN) * p->nphase;
  // split K until about two waves of CTAs fill the 132 SMs, keeping >= 256 K per slice
  int splits = 1;
  while (tiles * splits * 2 <= 264 && g.K / (splits * 2) >= 256) splits *= 2;
  p->splits = splits;
  p->kslice = ((g.K + splits - 1) / splits + p->BK - 1) / p->BK * p->BK;
  p->work = splits > 1 ? static_cast<long long>(splits) * 8 * g.M * Cout : 0;
  if ((g.M + p->BM - 1) / p->BM > 0x7fffffffLL) return -3;
  return 0;
}
}  // namespace
}  // namespace rn

using namespace rn;

extern "C" long long rn_conv3d_f32_workspace(int B, int H, int W, int D, int Cin, int Cout, int stride, int transposed) {
  Plan p;
  const int rc = make_plan(B, H, W, D, Cin, Cout, stride, transposed, &p);
  return rc != 0 ? rc : p.work;
}

extern "C" int rn_conv3d_f32(const float* x, const float* w, const float* bias, float* out, float* work, int B, int H, int W, int D,
                             int Cin, int Cout, int k, int stride, int transposed, int act, void* stream) {
  if (!x || !w || !out || k != 4) return -1;
  if (act != RN_ACT_NONE && act != RN_ACT_ELU && act != RN_ACT_SIGMOID) return -1;
  Plan p;
  const int rc = make_plan(B, H, W, D, Cin, Cout, stride, transposed, &p);
  if (rc != 0) return rc;
  if (p.work > 0 && !work) return -4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (transposed && stride == 1 && Cout == 1 && Cin % 4 == 0 && Cin <= 16 && H % T5_Y == 0 && W % T5_X == 0 && D % T5_Z == 0 &&
      (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const long long blocks = static_cast<long long>(B) * (H / T5_Y) * (W / T5_X) * (D / T5_Z);
    tconv_s1_to1_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(x, w, bias, out, B, H, W, D, Cin, act);
    RN_COUNT_LAUNCH();
    return static_cast<int>(cudaGetLastError());
  }
  const dim3 grid(static_cast<unsigned>((p.g.M + p.BM - 1) / p.BM), static_cast<unsigned>((Cout + p.BN - 1) / p.BN),
                  static_cast<unsigned>(p.nphase * p.splits));
  float* part = p.splits > 1 ? work : nullptr;
#define RN_F32(BM, BN, TM, TN, BK) \
  conv3d_f32_kernel<BM, BN, TM, TN, BK><<<grid, (BM / TM) * (BN / TN), 0, st>>>(x, w, bias, out, part, p.g, p.splits, p.kslice, act)
  switch (p.cfg) {
    case CFG_64x64: RN_F32(64, 64, 4, 4, 16); break;
    case CFG_128x32: RN_F32(128, 32, 4, 4, 16); break;
    case CFG_256x16: RN_F32(256, 16, 4, 4, 16); break;
    default: RN_F32(1024, 1, 4, 1, 8); break;
  }
#undef RN_F32
  RN_COUNT_LAUNCH();
  if (p.splits > 1) {
    const long long n = p.g.M * Cout * p.nphase;
    const long long blocks = (n + 255) / 256;
    conv3d_f32_reduce_kernel<<<static_cast<int>(blocks < 132 * 32 ? blocks : 132 * 32), 256, 0, st>>>(work, bias, out, p.g, p.nphase,
                                                                                                     p.splits, act);
    RN_COUNT_LAUNCH();
  }
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_act_backward_f32(const float* g, const float* y, float* out, long long n, int act, void* stream) {
  if (!g || !y || !out || n < 0 || (act != RN_ACT_ELU && act != RN_ACT_SIGMOID)) return -1;
  if (n == 0) return 0;
  const long long blocks = (n + 255) / 256;
  act_backward_f32_kernel<<<static_cast<int>(blocks < 132 * 32 ? blocks : 132 * 32), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      g, y, out, n, act);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}

namespace rn {
namespace {
// Weight-gradient plan: the forward's geometry (make_plan), a tile shape per Cout, and a K split that gives the SMs about four
// CTAs each while every slice keeps >= 1024 rows.  g_conv5's shape (transposed s1, 16 -> 1, tiles of 4 x 4 x 16) runs the
// direct kernel.
struct WPlan {
  Plan p;
  bool direct;
  int cfg, BM, BN, splits, grid5;
  long long kslice, work;   // floats of workspace: partial dW slices + partial bias sums
};

int make_wgrad_plan(int B, int H, int W, int D, int Cin, int Cout, int stride, int transposed, WPlan* q) {
  const int rc = make_plan(B, H, W, D, Cin, Cout, stride, transposed, &q->p);
  if (rc != 0) return rc;
  const Geo& g = q->p.g;
  const long long Mt = static_cast<long long>(g.ntaps) * Cin;
  q->direct = g.mode == 1 && Cout == 1 && Cin == W5_CIN && H % W5_Y == 0 && W % W5_X == 0 && D % W5_Z == 0;
  if (q->direct) {
    const long long ntiles = static_cast<long long>(B) * (H / W5_Y) * (W / W5_X) * (D / W5_Z);
    q->grid5 = static_cast<int>(ntiles < W5_MAX_CTAS ? ntiles : W5_MAX_CTAS);
    q->splits = q->grid5;
    q->kslice = 0;
    q->work = static_cast<long long>(q->grid5) * (Mt + 1);
    return 0;
  }
  if (Cout >= 64) { q->cfg = CFG_64x64; q->BM = 64; q->BN = 64; }
  else if (Cout >= 24) { q->cfg = CFG_128x32; q->BM = 128; q->BN = 32; }
  else if (Cout >= 2) { q->cfg = CFG_256x16; q->BM = 256; q->BN = 16; }
  else { q->cfg = CFG_1024x1; q->BM = 256; q->BN = 1; }
  const long long tiles = ((Mt + q->BM - 1) / q->BM) * ((Cout + q->BN - 1) / q->BN) * q->p.nphase;
  int splits = 1;
  while (tiles * splits < 4 * 132 && g.M / (splits * 2) >= 1024) splits *= 2;
  q->splits = splits;
  q->kslice = ((g.M + splits - 1) / splits + 15) / 16 * 16;
  q->work = static_cast<long long>(splits) * q->p.nphase * (Mt * Cout + Cout);
  return 0;
}
}  // namespace
}  // namespace rn

extern "C" long long rn_conv3d_f32_weight_grad_workspace(int B, int H, int W, int D, int Cin, int Cout, int stride, int transposed) {
  WPlan q;
  const int rc = make_wgrad_plan(B, H, W, D, Cin, Cout, stride, transposed, &q);
  return rc != 0 ? rc : q.work;
}

extern "C" int rn_conv3d_f32_weight_grad(const float* x, const float* gz, float* dw, float* db, float* work, int B, int H, int W,
                                         int D, int Cin, int Ho, int Wo, int Do, int Cout, int k, int stride, int transposed,
                                         void* stream) {
  if (!x || !gz || !dw || !db || k != 4) return -1;
  WPlan q;
  const int rc = make_wgrad_plan(B, H, W, D, Cin, Cout, stride, transposed, &q);
  if (rc != 0) return rc;
  const Geo& g = q.p.g;
  if (Ho != g.Ho || Wo != g.Wo || Do != g.Do) return -2;      // gz is not this layer's output grid
  if (!work) return -4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nphase = q.p.nphase;
  const long long Mt = static_cast<long long>(g.ntaps) * Cin;
  float* part = work;
  float* dbpart = work + static_cast<long long>(q.splits) * nphase * Mt * Cout;
  if (q.direct) {
    if ((reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(gz) & 15) != 0) return -3;
    // > 48 KB of dynamic shared memory: opt in (per device, so on every call)
    const cudaError_t e = cudaFuncSetAttribute(tconv_s1_to1_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W5_SMEM);
    if (e != cudaSuccess) return static_cast<int>(e);
    tconv_s1_to1_wgrad_kernel<<<q.grid5, 256, W5_SMEM, st>>>(x, gz, part, dbpart, B, H, W, D);
    RN_COUNT_LAUNCH();
  } else {
    const dim3 grid(static_cast<unsigned>((Mt + q.BM - 1) / q.BM), static_cast<unsigned>((Cout + q.BN - 1) / q.BN),
                    static_cast<unsigned>(nphase * q.splits));
#define RN_WG(BM, BN, TM, TN) \
    conv3d_f32_wgrad_kernel<BM, BN, TM, TN, 16><<<grid, (BM / TM) * (BN / TN), 0, st>>>(x, gz, part, dbpart, g, q.splits, q.kslice)
    switch (q.cfg) {
      case CFG_64x64: RN_WG(64, 64, 4, 4); break;
      case CFG_128x32: RN_WG(128, 32, 4, 4); break;
      case CFG_256x16: RN_WG(256, 16, 4, 4); break;
      default: RN_WG(256, 1, 1, 1); break;
    }
#undef RN_WG
    RN_COUNT_LAUNCH();
  }
  const long long n = Mt * Cout * nphase;
  const long long blocks = (n + 255) / 256;
  conv3d_f32_wgrad_reduce_kernel<<<static_cast<int>(blocks < 132 * 8 ? blocks : 132 * 8), 256, 0, st>>>(part, dbpart, dw, db, g,
                                                                                                       nphase, q.splits);
  RN_COUNT_LAUNCH();
  return static_cast<int>(cudaGetLastError());
}
