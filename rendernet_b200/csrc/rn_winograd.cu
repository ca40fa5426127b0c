// rn_winograd.cu -- the exact-mode (fp16 hi/lo) 3x3 C -> C trunk convolutions as Winograd F(2x2, 3x3) and F(4x4, 3x3)
// (Lavin & Gray 2016).
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
//
// F(4x4, 3x3) runs the same three steps on 6x6 input patches at (4ty-1, 4tx-1) and 4x4 output blocks: 36 products per 4x4
// block (2.25 per output pixel instead of 4), V and M 2.25x the activation instead of 4x.  Interpolation points 0, 1, -1,
// 1/2, -1/2 and infinity (not the textbook +-2: those grow V to 42 |x| and U's lo halves into fp16 subnormals, DESIGN §4):
//   B^T = [1/4  0   -5/4  0   1  0]    G = [ 4     0     0  ]    A^T = [1  1  1  1    1    0]
//         [0  -1/4  -1/4  1   1  0]        [ 2/3   2/3   2/3]          [0  1 -1  1/2 -1/2  0]
//         [0   1/4  -1/4 -1   1  0]        [ 2/3  -2/3   2/3]          [0  1  1  1/4  1/4  0]
//         [0  -1/2  -1   1/2  1  0]        [-8/3  -4/3  -2/3]          [0  1 -1  1/8 -1/8  1]
//         [0   1/2  -1  -1/2  1  0]        [-8/3   4/3  -2/3]
//         [0   1/4   0  -5/4  0  1]        [ 0     0     1  ]
// scaled by powers of two, which add no rounding: V = 1/2 B^T d B (|V| <= 4.5 |x|), U = 2^s G g G^T with s chosen per layer
// so that max |U| lies in (2^11, 2^12] (ops.winograd_filter: U's lo halves stay out of the fp16 subnormals), and
// y = 2^(1-s) A^T M A before the unchanged epilogue.
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
        epilogue_chunk<8, true>(p, acc, cg * 8, off, true, b, w_unscale_of(p));
      }
    }
  }
}

// B^T applied to one column (or row) of a 6-point patch, in place.
__device__ __forceinline__ void bt6(float& d0, float& d1, float& d2, float& d3, float& d4, float& d5) {
  const float p = fmaf(-0.25f, d2, d4), q = fmaf(-0.25f, d1, d3);   // d4 - d2/4, d3 - d1/4
  const float r = d4 - d2, s = 0.5f * (d3 - d1);
  const float t0 = fmaf(-1.25f, d2, fmaf(0.25f, d0, d4)), t5 = fmaf(-1.25f, d3, fmaf(0.25f, d1, d5));
  d0 = t0; d1 = p + q; d2 = p - q; d3 = r + s; d4 = r - s; d5 = t5;
}

// F(4x4, 3x3) input transform, streamed: every input row is read from HBM once per CTA.  One CTA: one image, kWi4Cs
// channels, kWi4Tw block columns (4 kWi4Tw + 2 input columns with the halo) and a band of block rows, swept top to bottom.
// Block row ty reads input rows 4ty-1 .. 4ty+4; the last two are the next block row's first two, so each step loads only
// 4 new rows.  The rows land by cp.async (zero-filled outside the image: the SAME padding) in a ring of kWi4Ring
// shared-memory rows, the next block row's 4 while this one is transformed.  One warp: one block column, 2 channels per
// lane, so each V store of a warp is 128 contiguous bytes.  Each element of V takes the same fp32 operations in the same
// order (hi + lo, bt6 down the columns, bt6 along the rows, x 1/2, split) whatever the tiling, band split or batch.
constexpr int kWi4Tw = 8;                     // block columns per CTA = warps
constexpr int kWi4Cs = 64;                    // channels per CTA
constexpr int kWi4Cols = 4 * kWi4Tw + 2;      // input columns per CTA
constexpr int kWi4Ring = 10;                  // input rows in shared memory: 6 being read + 4 being loaded
constexpr int kWi4Smem = kWi4Ring * 2 * kWi4Cols * kWi4Cs * 2;   // [row][hi, lo][column][channel] fp16

__global__ void __launch_bounds__(32 * kWi4Tw, 2) winograd4_in_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ v,
                                                                   int B, int H, int W, int C, int band) {
  constexpr int ROW = kWi4Cols * kWi4Cs;      // fp16 elements of one plane of one input row
  constexpr int CH = kWi4Cs / 8;              // 16-byte chunks per pixel and plane
  extern __shared__ __align__(16) uint16_t ring[];
  const int H4 = H / 4, W4 = W / 4;
  const int nslice = C / kWi4Cs, ntw = (W4 + kWi4Tw - 1) / kWi4Tw, nband = (H4 + band - 1) / band;
  int r = blockIdx.x;
  const int c0 = (r % nslice) * kWi4Cs;
  r /= nslice;
  const int tx0 = (r % ntw) * kWi4Tw;
  r /= ntw;
  const int ty0 = (r % nband) * band, ty1 = min(H4, ty0 + band);
  const int b = r / nband;
  const long long x_plane = static_cast<long long>(B) * H * W * C;
  const uint16_t* xb = x + static_cast<long long>(b) * H * W * C + c0;
  auto load_rows = [&](int y0, int nrows) {   // input rows y0 .. y0 + nrows - 1 -> ring row (y + 1) % kWi4Ring
    for (int i = threadIdx.x; i < nrows * 2 * kWi4Cols * CH; i += blockDim.x) {
      int q = i;
      const int ch = q % CH;
      q /= CH;
      const int col = q % kWi4Cols;
      q /= kWi4Cols;
      const int pl = q & 1, y = y0 + (q >> 1), xx = 4 * tx0 - 1 + col;
      const bool in = y >= 0 && y < H && xx >= 0 && xx < W;
      const uint16_t* src = in ? xb + pl * x_plane + (static_cast<long long>(y) * W + xx) * C + ch * 8 : x;
      cp_async16(ring + ((y + 1) % kWi4Ring * 2 + pl) * ROW + col * kWi4Cs + ch * 8, src, in ? 16 : 0);
    }
    cp_async_commit();
  };
  load_rows(4 * ty0 - 1, 6);
  const int warp = threadIdx.x / 32, cl = 2 * (threadIdx.x % 32);
  const int tx = tx0 + warp;
  const long long pos = static_cast<long long>(B) * H4 * W4 * C;   // one position of V
  const long long v_plane = 36 * pos;
  for (int ty = ty0; ty < ty1; ++ty) {
    cp_async_wait_all();
    __syncthreads();                          // rows of ty landed; every warp is done reading ty - 1's
    if (ty + 1 < ty1) load_rows(4 * ty + 5, 4);
    if (tx >= W4) continue;
    float t[6][6][2];
    const int s0 = 4 * ty % kWi4Ring;         // ring row of input row 4ty - 1
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      const uint16_t* row = ring + (s0 + a < kWi4Ring ? s0 + a : s0 + a - kWi4Ring) * 2 * ROW + 4 * warp * kWi4Cs + cl;
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(row + c * kWi4Cs));
        const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(row + ROW + c * kWi4Cs));
        t[a][c][0] = fh.x + fl.x;
        t[a][c][1] = fh.y + fl.y;
      }
    }
#pragma unroll
    for (int c = 0; c < 6; ++c)              // columns: B^T d
#pragma unroll
      for (int k = 0; k < 2; ++k) bt6(t[0][c][k], t[1][c][k], t[2][c][k], t[3][c][k], t[4][c][k], t[5][c][k]);
    const long long o = ((static_cast<long long>(b) * H4 + ty) * W4 + tx) * C + c0 + cl;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int k = 0; k < 2; ++k) bt6(t[a][0][k], t[a][1][k], t[a][2][k], t[a][3][k], t[a][4][k], t[a][5][k]);   // rows
#pragma unroll
      for (int e = 0; e < 6; ++e) {          // v = t / 2 (exact), hi = fp16(v), lo = fp16(v - hi)
        const float v0 = 0.5f * t[a][e][0], v1 = 0.5f * t[a][e][1];
        const __half2 h = __floats2half2_rn(v0, v1);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
        uint32_t* dst = reinterpret_cast<uint32_t*>(v + (6 * a + e) * pos + o);
        dst[0] = *reinterpret_cast<const uint32_t*>(&h);
        dst[v_plane >> 1] = *reinterpret_cast<const uint32_t*>(&l);
      }
    }
  }
}

// F(4x4, 3x3).  One thread: 8 channels of one 4x4 output block.  M is read one row of the 6x6 tile at a time and folded into
// the 16 outputs as it arrives (row A^T first, then the row's share of the column A^T), so only 16 x 8 sums stay live.
// y_scale = 2^(1-s) undoes the powers of two on U and V (exact).
__global__ void __launch_bounds__(128) winograd4_out_kernel(const __grid_constant__ IgemmParams p, const float* __restrict__ m,
                                                            float y_scale, int B, int H, int W, int C) {
  const int H4 = H / 4, W4 = W / 4, CG = C / 8;
  const long long n = static_cast<long long>(B) * H4 * W4 * CG;
  const long long pos = static_cast<long long>(B) * H4 * W4 * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % CG);
    long long r = i / CG;
    const int tx = static_cast<int>(r % W4);
    r /= W4;
    const int ty = static_cast<int>(r % H4);
    const int b = static_cast<int>(r / H4);
    const long long o = ((static_cast<long long>(b) * H4 + ty) * W4 + tx) * C + cg * 8;
    float s[4][4][8];                      // A^T M A, accumulated over the 6 rows of M
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      float q[6][8];
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const float4* src = reinterpret_cast<const float4*>(m + (6 * a + c) * pos + o);
        const float4 q0 = __ldg(src), q1 = __ldg(src + 1);
        q[c][0] = q0.x; q[c][1] = q0.y; q[c][2] = q0.z; q[c][3] = q0.w;
        q[c][4] = q1.x; q[c][5] = q1.y; q[c][6] = q1.z; q[c][7] = q1.w;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float s12 = q[1][k] + q[2][k], d12 = q[1][k] - q[2][k];
        const float s34 = q[3][k] + q[4][k], d34 = q[3][k] - q[4][k];
        const float row[4] = {q[0][k] + s12 + s34, fmaf(0.5f, d34, d12), fmaf(0.25f, s34, s12),
                              fmaf(0.125f, d34, d12) + q[5][k]};   // (row a of M) A
#pragma unroll
        for (int e = 0; e < 4; ++e) {      // s[i] += A^T[i][a] * row
          const float v = row[e];
          if (a == 0) { s[0][e][k] = v; s[1][e][k] = 0.f; s[2][e][k] = 0.f; s[3][e][k] = 0.f; }
          else if (a == 1) { s[0][e][k] += v; s[1][e][k] += v; s[2][e][k] += v; s[3][e][k] += v; }
          else if (a == 2) { s[0][e][k] += v; s[1][e][k] -= v; s[2][e][k] += v; s[3][e][k] -= v; }
          else if (a == 3) {
            s[0][e][k] += v; s[1][e][k] = fmaf(0.5f, v, s[1][e][k]);
            s[2][e][k] = fmaf(0.25f, v, s[2][e][k]); s[3][e][k] = fmaf(0.125f, v, s[3][e][k]);
          } else if (a == 4) {
            s[0][e][k] += v; s[1][e][k] = fmaf(-0.5f, v, s[1][e][k]);
            s[2][e][k] = fmaf(0.25f, v, s[2][e][k]); s[3][e][k] = fmaf(-0.125f, v, s[3][e][k]);
          } else {
            s[3][e][k] += v;
          }
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int y = 4 * ty + a;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = s[a][e][k] * y_scale;
        const long long off = ((static_cast<long long>(b) * H + y) * W + 4 * tx + e) * C;
        epilogue_chunk<8, true>(p, acc, cg * 8, off, true, b);   // U carries its own exponent (u_exp), never w_unscale
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

static bool wino4_shape_ok(int B, int H, int W, int C) {
  return B >= 1 && H >= 4 && W >= 4 && H % 4 == 0 && W % 4 == 0 && C % 64 == 0;
}

// U = 2^s G g G^T: s in [-kWino4MaxExp, kWino4MaxExp] keeps 2^(1-s) a normal fp32 number
constexpr int kWino4MaxExp = 100;

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

extern "C" int rn_winograd_out_scaled(const float* m, const float* w_unscale, const float* bias, const float* alpha, int act,
                                      const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H,
                                      int W, int C, void* stream) {
  if (m == nullptr || bias == nullptr || (out16 == nullptr && out32 == nullptr) || !wino_shape_ok(B, H, W, C)) return -1;
  if (act != ACT_NONE && act != ACT_PRELU && act != ACT_SIGMOID) return -1;
  if (act == ACT_PRELU && alpha == nullptr) return -5;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.out16 = out16; p.out32 = out32; p.res = residual; p.res_is_f32 = residual_is_f32;
  p.bias = bias; p.alpha = alpha; p.act = act; p.n_valid = C; p.vec_ok = 1; p.ab_fmt = 0; p.split = 1;
  p.o_plane = static_cast<long long>(B) * H * W * C;
  p.w_unscale = w_unscale;
  const long long n = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 8);
  winograd_out_kernel<<<wino_grid(n), 128, 0, static_cast<cudaStream_t>(stream)>>>(p, m, B, H, W, C);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_winograd_out(const float* m, const float* bias, const float* alpha, int act, const void* residual,
                               int residual_is_f32, void* out16, float* out32, int B, int H, int W, int C, void* stream) {
  return rn_winograd_out_scaled(m, nullptr, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, C, stream);
}

extern "C" int rn_conv2d_winograd_scaled(const void* x, const void* u, const float* w_unscale, const float* bias,
                                         const float* alpha, int act, const void* residual, int residual_is_f32, void* out16,
                                         float* out32, int B, int H, int W, int C, void* workspace, long long workspace_bytes,
                                         const rn_tuning* tune, void* stream) {
  const long long need = rn_winograd_workspace_bytes(B, H, W, C);
  if (need < 0 || workspace == nullptr || workspace_bytes < need) return -1;
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x) || !al16(u) || !al16(workspace) || !al16(residual) || !al16(out16) || !al16(out32)) return -1;
  uint16_t* v = static_cast<uint16_t*>(workspace);
  float* m = reinterpret_cast<float*>(v + 2 * 16LL * B * (H / 2) * (W / 2) * C);
  int rc = rn_winograd_in(x, v, B, H, W, C, stream);
  if (rc == 0) rc = rn_winograd_gemm(v, u, m, B, H, W, C, tune, stream);
  if (rc == 0)
    rc = rn_winograd_out_scaled(m, w_unscale, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, C, stream);
  return rc;
}

extern "C" int rn_conv2d_winograd(const void* x, const void* u, const float* bias, const float* alpha, int act,
                                  const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                                  int C, void* workspace, long long workspace_bytes, const rn_tuning* tune, void* stream) {
  return rn_conv2d_winograd_scaled(x, u, nullptr, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, C,
                                   workspace, workspace_bytes, tune, stream);
}

extern "C" int rn_conv2d_winograd_tile(int fmt, int kh, int kw, int H, int W, int Cin, int Cout, int cout_pad,
                                       const rn_tuning* tune) {
  if (!rn_conv2d_winograd_eligible(fmt, kh, kw, H, W, Cin, Cout, cout_pad, tune)) return 0;
  const int want = tune != nullptr && tune->wino_tile > 0 ? tune->wino_tile : tuning().wino_tile;
  return want == 4 && wino4_shape_ok(1, H, W, Cin) ? 4 : 2;
}

extern "C" long long rn_winograd4_workspace_bytes(int B, int H, int W, int C) {
  if (!wino4_shape_ok(B, H, W, C)) return -1;
  const long long pos = static_cast<long long>(B) * (H / 4) * (W / 4) * C;
  return 36 * pos * 2 * 2 + 36 * pos * 4;   // V: two fp16 planes, M: fp32
}

extern "C" int rn_winograd4_in(const void* x, void* v, int B, int H, int W, int C, void* stream) {
  if (x == nullptr || v == nullptr || !wino4_shape_ok(B, H, W, C)) return -1;
  static std::atomic<bool> attr_set[kMaxDevices];   // cudaFuncSetAttribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    const cudaError_t e = cudaFuncSetAttribute(winograd4_in_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWi4Smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set[dev].store(true, std::memory_order_release);
  }
  // Split the height into bands only when (image, channel slice, width tile) alone leave SMs idle: each band re-reads a
  // 2-row halo.
  const int H4 = H / 4;
  const long long base = static_cast<long long>(B) * (C / kWi4Cs) * ((W / 4 + kWi4Tw - 1) / kWi4Tw);
  const long long want = (2LL * num_sms() + base - 1) / base;   // 2 CTAs fit on an SM
  const int nband = static_cast<int>(want < H4 ? want : H4), band = (H4 + nband - 1) / nband;
  const long long grid = base * ((H4 + band - 1) / band);
  if (grid > 0x7fffffffLL) return -1;
  winograd4_in_kernel<<<static_cast<unsigned>(grid), 32 * kWi4Tw, kWi4Smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(x), static_cast<uint16_t*>(v), B, H, W, C, band);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_winograd4_gemm(const void* v, const void* u, float* m, int B, int H, int W, int C, const rn_tuning* tune,
                                 void* stream) {
  if (v == nullptr || u == nullptr || m == nullptr || !wino4_shape_ok(B, H, W, C) || C % kWinoGemmN != 0) return -1;
  const int8_t tap[3] = {0, 0, 0};
  const int H4 = H / 4, W4 = W / 4;
  rn_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.ndim = 2; d.B = 36 * B; d.H = H4; d.W = W4; d.D = 1; d.Cin = C; d.Cout = C; d.cout_pad = C;
  d.ntaps = 1; d.taps = tap; d.x = v; d.w_packed = u; d.bias = nullptr; d.alpha = nullptr; d.act = ACT_NONE;
  d.out32 = m;
  d.o_x = C; d.o_y = static_cast<long long>(W4) * C; d.o_b = static_cast<long long>(H4) * W4 * C;
  d.fmt = 2;
  d.x_plane = 36LL * B * H4 * W4 * C;
  d.w_plane = 36LL * C * C;
  d.b_tap_div = B;
  d.force_bn = kWinoGemmN;
  if (tune != nullptr) { d.force_kps = tune->kps; d.msub = tune->msub; }
  return rn_conv_igemm(&d, stream);
}

extern "C" int rn_winograd4_out(const float* m, const float* bias, const float* alpha, int act, const void* residual,
                                int residual_is_f32, void* out16, float* out32, int B, int H, int W, int C, int u_exp,
                                void* stream) {
  if (m == nullptr || bias == nullptr || (out16 == nullptr && out32 == nullptr) || !wino4_shape_ok(B, H, W, C)) return -1;
  if (u_exp < -kWino4MaxExp || u_exp > kWino4MaxExp) return -1;
  if (act != ACT_NONE && act != ACT_PRELU && act != ACT_SIGMOID) return -1;
  if (act == ACT_PRELU && alpha == nullptr) return -5;
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.out16 = out16; p.out32 = out32; p.res = residual; p.res_is_f32 = residual_is_f32;
  p.bias = bias; p.alpha = alpha; p.act = act; p.n_valid = C; p.vec_ok = 1; p.ab_fmt = 0; p.split = 1;
  p.o_plane = static_cast<long long>(B) * H * W * C;
  const long long n = static_cast<long long>(B) * (H / 4) * (W / 4) * (C / 8);
  winograd4_out_kernel<<<wino_grid(n), 128, 0, static_cast<cudaStream_t>(stream)>>>(p, m, ldexpf(1.f, 1 - u_exp), B, H, W,
                                                                                     C);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int rn_conv2d_winograd4(const void* x, const void* u, int u_exp, const float* bias, const float* alpha, int act,
                                   const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                                   int C, void* workspace, long long workspace_bytes, const rn_tuning* tune, void* stream) {
  const long long need = rn_winograd4_workspace_bytes(B, H, W, C);
  if (need < 0 || workspace == nullptr || workspace_bytes < need) return -1;
  if (u_exp < -kWino4MaxExp || u_exp > kWino4MaxExp) return -1;
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x) || !al16(u) || !al16(workspace) || !al16(residual) || !al16(out16) || !al16(out32)) return -1;
  uint16_t* v = static_cast<uint16_t*>(workspace);
  float* m = reinterpret_cast<float*>(v + 2 * 36LL * B * (H / 4) * (W / 4) * C);
  int rc = rn_winograd4_in(x, v, B, H, W, C, stream);
  if (rc == 0) rc = rn_winograd4_gemm(v, u, m, B, H, W, C, tune, stream);
  if (rc == 0)
    rc = rn_winograd4_out(m, bias, alpha, act, residual, residual_is_f32, out16, out32, B, H, W, C, u_exp, stream);
  return rc;
}
