// rn_winograd.cu -- the exact-mode (fp16 hi/lo) 3x3 C -> C trunk convolutions as Winograd F(2x2, 3x3) (Lavin & Gray 2016).
//
// Per 2x2 output block, with d the 4x4 input patch at (2ty-1, 2tx-1) and g the 3x3 filter of one (Cin, Cout) pair:
//   y = A^T [ (G g G^T) (.) (B^T d B) ] A,   B^T = [1 0 -1 0; 0 1 1 0; 0 -1 1 0; 0 1 0 -1],  A^T = [1 1 1 0; 0 1 -1 -1],
//   G = [1 0 0; 1/2 1/2 1/2; 1/2 -1/2 1/2; 0 0 1]
// Summed over Cin, the elementwise product becomes 16 independent GEMMs (one per position of the 4x4 tile), M = B*H/2*W/2,
// N = Cout, K = Cin: 16 products per block where the direct conv issues 36, and each output sums 16 K = C chains instead of
// one K = 9C chain.  Three launches:
//   * winograd_in_kernel: V = B^T d B in fp32 from hi + lo (exact: <= 22 significant bits), split once into hi/lo planes
//     [16][B,H/2,W/2,C];
//   * the 16 GEMMs as ONE igemm launch of a 1x1 conv over V viewed as [16*B, H/2, W/2, C] whose image b reads filter "tap"
//     b / B (IgemmParams::b_tap_div) of U = G g G^T, packed [16][Cout][Cin] (ops.winograd_filter); exact-mode pseudo-tap
//     order, raw fp32 output M (the igemm variant without bias that stores straight from its accumulators);
//   * winograd_out_kernel: A^T M A in fp32, then the igemm epilogue itself (epilogue_chunk: bias, PReLU, residual, hi/lo and
//     fp32 stores, one rounding).
// The transforms only use 0, +-1 and +-1/2, so they add a few fp32 roundings and no cancellation-prone coefficients.
#include <cstring>

#include "../../include/rendernet_b200.h"
#include "rn_igemm_kernel.cuh"

namespace rn {

constexpr int kWinoMinC = 1024;   // smallest C routed to Winograd (res2 trunk; scripts/winograd_time.py times 512 as well)
constexpr int kWinoGemmN = 256;   // N tile of the per-position GEMM: its raw-output igemm variant is built for this one only

__device__ __forceinline__ void load8(const uint16_t* __restrict__ hi, long long plane, long long off, float* v) {
  const uint4 h = __ldg(reinterpret_cast<const uint4*>(hi + off));
  const uint4 l = __ldg(reinterpret_cast<const uint4*>(hi + plane + off));
  const uint32_t wh[4] = {h.x, h.y, h.z, h.w}, wl[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&wh[j]));
    const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&wl[j]));
    v[2 * j] = fh.x + fl.x;
    v[2 * j + 1] = fh.y + fl.y;
  }
}

// One thread: 8 channels of one 2x2 output block.  Reads the 4x4 patch (zero outside the image), writes 16 positions.
__global__ void __launch_bounds__(128) winograd_in_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ v, int B,
                                                          int H, int W, int C) {
  const int H2 = H / 2, W2 = W / 2, CG = C / 8;
  const long long n = static_cast<long long>(B) * H2 * W2 * CG;
  const long long x_plane = static_cast<long long>(B) * H * W * C;
  const long long pos = static_cast<long long>(B) * H2 * W2 * C;   // one position of V
  const long long v_plane = 16 * pos;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % CG);
    long long r = i / CG;
    const int tx = static_cast<int>(r % W2);
    r /= W2;
    const int ty = static_cast<int>(r % H2);
    const int b = static_cast<int>(r / H2);
    float t[4][4][8];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int yy = 2 * ty - 1 + a;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int xx = 2 * tx - 1 + c;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
          load8(x, x_plane, ((static_cast<long long>(b) * H + yy) * W + xx) * C + cg * 8, t[a][c]);
        } else {
#pragma unroll
          for (int k = 0; k < 8; ++k) t[a][c][k] = 0.f;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c)            // rows: B^T d
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d0 = t[0][c][k], d1 = t[1][c][k], d2 = t[2][c][k], d3 = t[3][c][k];
        t[0][c][k] = d0 - d2; t[1][c][k] = d1 + d2; t[2][c][k] = d2 - d1; t[3][c][k] = d1 - d3;
      }
#pragma unroll
    for (int a = 0; a < 4; ++a)            // columns: (B^T d) B
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d0 = t[a][0][k], d1 = t[a][1][k], d2 = t[a][2][k], d3 = t[a][3][k];
        t[a][0][k] = d0 - d2; t[a][1][k] = d1 + d2; t[a][2][k] = d2 - d1; t[a][3][k] = d1 - d3;
      }
    const long long o = ((static_cast<long long>(b) * H2 + ty) * W2 + tx) * C + cg * 8;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t wh[4], wl[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // hi = fp16(v), lo = fp16(v - hi), as the igemm epilogue splits
          const __half2 h = __floats2half2_rn(t[a][c][2 * j], t[a][c][2 * j + 1]);
          const float2 hf = __half22float2(h);
          const __half2 l = __floats2half2_rn(t[a][c][2 * j] - hf.x, t[a][c][2 * j + 1] - hf.y);
          wh[j] = *reinterpret_cast<const uint32_t*>(&h);
          wl[j] = *reinterpret_cast<const uint32_t*>(&l);
        }
        uint4* dst = reinterpret_cast<uint4*>(v + (4 * a + c) * pos + o);
        dst[0] = make_uint4(wh[0], wh[1], wh[2], wh[3]);
        dst[v_plane >> 3] = make_uint4(wl[0], wl[1], wl[2], wl[3]);
      }
  }
}

// One thread: 8 channels of one 2x2 output block.  p carries the epilogue fields of IgemmParams (o_* unused: offsets are
// computed here).
__global__ void __launch_bounds__(128) winograd_out_kernel(const __grid_constant__ IgemmParams p, const float* __restrict__ m,
                                                           int B, int H, int W, int C) {
  const int H2 = H / 2, W2 = W / 2, CG = C / 8;
  const long long n = static_cast<long long>(B) * H2 * W2 * CG;
  const long long pos = static_cast<long long>(B) * H2 * W2 * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % CG);
    long long r = i / CG;
    const int tx = static_cast<int>(r % W2);
    r /= W2;
    const int ty = static_cast<int>(r % H2);
    const int b = static_cast<int>(r / H2);
    const long long o = ((static_cast<long long>(b) * H2 + ty) * W2 + tx) * C + cg * 8;
    float s[2][4][8];                      // A^T M, accumulated over the 4 rows of M as they are read
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float4* src = reinterpret_cast<const float4*>(m + (4 * a + c) * pos + o);
        const float4 q0 = __ldg(src), q1 = __ldg(src + 1);
        const float q[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          if (a == 0) { s[0][c][k] = q[k]; s[1][c][k] = 0.f; }
          else if (a == 1) { s[0][c][k] += q[k]; s[1][c][k] = q[k]; }
          else if (a == 2) { s[0][c][k] += q[k]; s[1][c][k] -= q[k]; }
          else s[1][c][k] -= q[k];
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int y = 2 * ty + a;
#pragma unroll
      for (int e = 0; e < 2; ++e) {        // (A^T M) A
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
          acc[k] = e == 0 ? s[a][0][k] + s[a][1][k] + s[a][2][k] : s[a][1][k] - s[a][2][k] - s[a][3][k];
        const long long off = ((static_cast<long long>(b) * H + y) * W + 2 * tx + e) * C;
        epilogue_chunk<8, true>(p, acc, cg * 8, off, true, b);
      }
    }
  }
}

static int wino_grid(long long n) {
  const long long g = (n + 127) / 128;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

static bool wino_shape_ok(int B, int H, int W, int C) {
  return B >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && C % 64 == 0;
}

}  // namespace rn

using namespace rn;

extern "C" long long rn_winograd_workspace_bytes(int B, int H, int W, int C) {
  if (!wino_shape_ok(B, H, W, C)) return -1;
  const long long pos = static_cast<long long>(B) * (H / 2) * (W / 2) * C;
  return 16 * pos * 2 * 2 + 16 * pos * 4;   // V: two fp16 planes, M: fp32
}

extern "C" int rn_conv2d_winograd_eligible(int fmt, int kh, int kw, int H, int W, int Cin, int Cout, int cout_pad,
                                           const rn_tuning* tune) {
  // tune->winograd = 1 also takes C below the threshold (A/B timing of the 512-channel res3 layers)
  const bool forced = tune != nullptr && tune->winograd > 0;
  const bool on = forced || (tune != nullptr && tune->winograd < 0 ? false : tuning().winograd != 0);
  return on && fmt == 2 && kh == 3 && kw == 3 && Cin == Cout && Cout == cout_pad && (forced || Cin >= kWinoMinC) &&
         Cin % kWinoGemmN == 0 && wino_shape_ok(1, H, W, Cin);
}

extern "C" int rn_winograd_in(const void* x, void* v, int B, int H, int W, int C, void* stream) {
  if (x == nullptr || v == nullptr || !wino_shape_ok(B, H, W, C)) return -1;
  const long long n = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 8);
  winograd_in_kernel<<<wino_grid(n), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(x), static_cast<uint16_t*>(v), B, H, W, C);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_winograd_gemm(const void* v, const void* u, float* m, int B, int H, int W, int C, const rn_tuning* tune,
                                void* stream) {
  if (v == nullptr || u == nullptr || m == nullptr || !wino_shape_ok(B, H, W, C) || C % kWinoGemmN != 0) return -1;
  const int8_t tap[3] = {0, 0, 0};
  const int H2 = H / 2, W2 = W / 2;
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 2; d.B = 16 * B; d.H = H2; d.W = W2; d.D = 1; d.Cin = C; d.Cout = C; d.cout_pad = C;
  d.ntaps = 1; d.taps = tap; d.x = v; d.w_packed = u; d.bias = nullptr; d.alpha = nullptr; d.act = ACT_NONE;
  d.out32 = m;
  d.o_x = C; d.o_y = static_cast<long long>(W2) * C; d.o_b = static_cast<long long>(H2) * W2 * C;
  d.fmt = 2;
  d.x_plane = 16LL * B * H2 * W2 * C;
  d.w_plane = 16LL * C * C;
  d.b_tap_div = B;
  d.force_bn = kWinoGemmN;
  if (tune != nullptr) { d.force_kps = tune->kps; d.msub = tune->msub; }
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_winograd_out(const float* m, const float* bias, const float* alpha, int act, const void* residual,
                               int residual_is_f32, void* out16, float* out32, int B, int H, int W, int C, void* stream) {
  if (m == nullptr || bias == nullptr || (out16 == nullptr && out32 == nullptr) || !wino_shape_ok(B, H, W, C)) return -1;
  if (act != ACT_NONE && act != ACT_PRELU && act != ACT_SIGMOID) return -1;
  if (act == ACT_PRELU && alpha == nullptr) return -5;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.out16 = out16; p.out32 = out32; p.res = residual; p.res_is_f32 = residual_is_f32;
  p.bias = bias; p.alpha = alpha; p.act = act; p.n_valid = C; p.vec_ok = 1; p.ab_fmt = 0; p.split = 1;
  p.o_plane = static_cast<long long>(B) * H * W * C;
  const long long n = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 8);
  winograd_out_kernel<<<wino_grid(n), 128, 0, static_cast<cudaStream_t>(stream)>>>(p, m, B, H, W, C);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_conv2d_winograd(const void* x, const void* u, const float* bias, const float* alpha, int act,
                                  const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                                  int C, void* workspace, long long workspace_bytes, const rn_tuning* tune, void* stream) {
  const long long need = rn_winograd_workspace_bytes(B, H, W, C);
  if (need < 0 || workspace == nullptr || workspace_bytes < need) return -1;
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x) || !al16(u) || !al16(workspace) || !al16(residual) || !al16(out16) || !al16(out32)) return -1;
  uint16_t* v = static_cast<uint16_t*>(workspace);
  float* m = reinterpret_cast<float*>(v + 2 * 16LL * B * (H / 2) * (W / 2) * C);
  int rc = rn_winograd_in(x, v, B, H, W, C, stream);
  if (rc == 0) rc = rn_winograd_gemm(v, u, m, B, H, W, C, tune, stream);
  if (rc == 0) rc = rn_winograd_out(m, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, C, stream);
  return rc;
}
