// rn_wgrad.cu -- weight gradient of a stride-1 SAME 2-D convolution on the Hopper tensor cores (backward pass, stage 2;
// the training step of RenderNet_Shader.py:159-167 differentiates every conv filter).
//
//   dW[tap][ci][co] = sum over pixels p of  x[p + off(tap)][ci] * g[p][co]              (x = layer input, g = dL/d(conv output))
//
// A GEMM per tap with M = ci, N = co and K = pixels.  Both operands are channel-last ([pixel][channel]), i.e. M/N-contiguous:
// wgmma reads them as MN-MAJOR (transposed) operands straight from what TMA delivers -- a box {64 channels, 64 pixels} lands as 64
// rows of 128 bytes in the 128-byte swizzle, which is the canonical MN-major layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte
// units: SBO = 1024 B between 8-pixel groups, LBO = 8192 B between the 64-channel boxes of a tile.  No transposed copy of the
// activations is ever made.  The tap offset is a shifted TMA coordinate for x (zero fill outside the image = SAME padding).
//
// One CTA tile = (tap, 128 input channels, BN output channels); the K loop runs over pixel blocks of a slice of the batch
// (split-K over CTAs when there are fewer tiles than SMs or a slice would exceed kWgMaxChainPixels; partial results are
// combined with fp32 atomics into a zero-initialised dW).  Warpgroup 0 = TMA producer; warpgroups 1 and 2 each own 64 of the 128 input channels: m64nBNk16
// wgmmas into fp32 register accumulators, then the stores of those rows.  Exact mode (fmt 2): three passes x_lo.g_hi,
// x_hi.g_lo, x_hi.g_hi into the same accumulator, corrections first (DESIGN.md §4).
#include <atomic>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "../../include/rendernet_b200.h"
#include "rn_igemm.cuh"
#include "rn_ptx.cuh"

namespace rn {
extern std::atomic<long long> g_launch_count;

struct alignas(64) WgradParams {
  CUtensorMap tmX, tmX2;        // activations {Cin, W, H, B}, box {64, PX, PY, 1}; tmX2 = LO plane (fmt 2)
  CUtensorMap tmG, tmG2;        // output gradient {Cout, W, H, B}, same box
  float* dw;                    // [ntaps][Cin][Cout] fp32, accumulated with atomics
  int Cin, Cout, W, H, B;
  int PX, PY;                   // pixel block = PX x PY = 64 pixels
  int ntaps;
  int8_t tap[16][2];            // (dx, dy) of each filter tap
  int m_tiles, n_tiles;         // Cin / 128, Cout / BN
  int ksplit;                   // CTAs sharing one output tile (each takes a slice of the batch)
  int stages;
  int split;                    // fmt 2
};

constexpr int kWgBM = 128;                 // input channels per tile (2 boxes of 64)
constexpr int kBoxBytes = 64 * 128;        // one TMA box: 64 pixels x 64 channels x 2 B
constexpr int kWgMaxChainPixels = 4096;    // pixels one CTA accumulates in a single wgmma chain (when the batch can be split)

__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);            // start address
  d |= static_cast<uint64_t>(kBoxBytes >> 4) << 16;                   // LBO: next 64-channel box
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                        // SBO: next group of 8 pixels
  d |= wgmma_layout_code(128) << 62;                                  // SWIZZLE_128B
  return d;
}

template <int BN>
__global__ void __launch_bounds__(384, 1) wgrad2d_kernel(const __grid_constant__ WgradParams p) {
  constexpr int NBOX_B = BN / 64;
  constexpr int kStageBytes = (2 + NBOX_B) * kBoxBytes;
  constexpr int NACC = BN / 2;                       // accumulator registers per consumer thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(p.stages) * kStageBytes);
  uint64_t* empty_bar = full_bar + p.stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmX);
    tma_prefetch_desc(&p.tmG);
    if (p.split) { tma_prefetch_desc(&p.tmX2); tma_prefetch_desc(&p.tmG2); }
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  const int bx = p.W / p.PX, by = p.H / p.PY;
  const int kb_per_img = bx * by;
  // batch slice ks is the slowest index: CTAs running at the same time work on different output tiles (no atomics on the same
  // addresses) of the same images (shared in L2)
  const int tiles = p.ntaps * p.m_tiles * p.n_tiles;
  const int total_work = tiles * p.ksplit;
  const int passes = p.split ? 3 : 1;

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int wk = blockIdx.x; wk < total_work; wk += gridDim.x) {
        const int ks = wk / tiles; int t = wk % tiles;
        const int ni = t % p.n_tiles; t /= p.n_tiles;
        const int mi = t % p.m_tiles; const int tap = t / p.m_tiles;
        const int b0 = (p.B * ks) / p.ksplit, b1 = (p.B * (ks + 1)) / p.ksplit;
        const int dx = p.tap[tap][0], dy = p.tap[tap][1];
        for (int pass = 0; pass < passes; ++pass) {
          // pass order in exact mode: x_lo.g_hi, x_hi.g_lo, x_hi.g_hi
          const CUtensorMap* mx = (p.split && pass == 0) ? &p.tmX2 : &p.tmX;
          const CUtensorMap* mg = (p.split && pass == 1) ? &p.tmG2 : &p.tmG;
          for (int b = b0; b < b1; ++b)
            for (int kb = 0; kb < kb_per_img; ++kb) {
              const int x0 = (kb % bx) * p.PX, y0 = (kb / bx) * p.PY;
              mbar_wait(&empty_bar[stage], phase ^ 1);
              mbar_expect_tx(&full_bar[stage], kStageBytes);
              uint8_t* dst = smem + static_cast<size_t>(stage) * kStageBytes;
              tma_load_4d(dst, mx, &full_bar[stage], mi * kWgBM, x0 + dx, y0 + dy, b);
              tma_load_4d(dst + kBoxBytes, mx, &full_bar[stage], mi * kWgBM + 64, x0 + dx, y0 + dy, b);
#pragma unroll
              for (int j = 0; j < NBOX_B; ++j)
                tma_load_4d(dst + (2 + j) * kBoxBytes, mg, &full_bar[stage], ni * BN + 64 * j, x0, y0, b);
              if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // consumer warpgroup wg: input channels [64 wg, 64 wg + 64) of the tile = x box wg; M = 64, N = BN, both MN-major
    const int wg = (warp - 4) >> 2;
    const int fr = 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);   // accumulator fragment rows fr, fr+8
    float acc[NACC];
    int stage = 0; uint32_t phase = 0;
    for (int wk = blockIdx.x; wk < total_work; wk += gridDim.x) {
      const int ks = wk / tiles; int t = wk % tiles;
      const int ni = t % p.n_tiles; t /= p.n_tiles;
      const int mi = t % p.m_tiles; const int tap = t / p.m_tiles;
      const int b0 = (p.B * ks) / p.ksplit, b1 = (p.B * (ks + 1)) / p.ksplit;
      const int nkb = (b1 - b0) * kb_per_img * passes;
      int prev = -1;                               // stage whose wgmma group may still be in flight
      uint32_t scale_d = 0;
      for (int it = 0; it < nkb; ++it) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        const uint32_t a0 = smem_u32(smem + static_cast<size_t>(stage) * kStageBytes);
        const uint64_t da = make_smem_desc_mn(a0 + wg * kBoxBytes), db = make_smem_desc_mn(a0 + 2 * kBoxBytes);
#pragma unroll
        for (int k = 0; k < 4; ++k) {             // 64 pixels = 4 x (K = 16); 16 pixel rows = 2048 B further on
          wgmma_ss<BN, 1>(acc, da + static_cast<uint64_t>(k * (2048 >> 4)), db + static_cast<uint64_t>(k * (2048 >> 4)),
                          scale_d, 0);
          scale_d = 1;
        }
        wgmma_commit();
        wgmma_wait<1>();
        __syncwarp();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      // rows = input channels, columns = output channels: d[4j..4j+1] at (fr, 8j+fc), d[4j+2..4j+3] at (fr+8, 8j+fc)
      float* orow = p.dw + (static_cast<size_t>(tap) * p.Cin + (mi * kWgBM + 64 * wg + fr)) * p.Cout + ni * BN + fc;
      const size_t down8 = static_cast<size_t>(8) * p.Cout;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (p.ksplit == 1) {
          *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(orow + down8 + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        } else {
          atomicAdd(orow + 8 * j, acc[4 * j]);
          atomicAdd(orow + 8 * j + 1, acc[4 * j + 1]);
          atomicAdd(orow + down8 + 8 * j, acc[4 * j + 2]);
          atomicAdd(orow + down8 + 8 * j + 1, acc[4 * j + 3]);
        }
      }
    }
  }
  __syncthreads();
}

template <int BN>
static cudaError_t launch_wgrad(const WgradParams& p, int grid, size_t smem, cudaStream_t st) {
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(wgrad2d_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e != cudaSuccess) return e;
    attr_set[dev].store(true, std::memory_order_release);
  }
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  wgrad2d_kernel<BN><<<grid, 384, smem, st>>>(p);
  return cudaGetLastError();
}

// sum over pixels of a 16-bit channel-last tensor: db[c] = sum_p g[p][c] (bias gradient), fp32 atomics into a zeroed vector
__global__ void bias_grad_kernel(const uint16_t* __restrict__ g, float* __restrict__ db, long long npix, int C, int fmt,
                                 long long plane) {
  // one thread per (pixel chunk, channel): blockDim.x = channels handled per block row, grid-stride over pixel chunks
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (long long px = blockIdx.x; px < npix; px += gridDim.x) {
    const long long i = px * C + c;
    float v = __half2float(*reinterpret_cast<const __half*>(g + i));
    if (fmt == 2) v += __half2float(*reinterpret_cast<const __half*>(g + i + plane));
    acc += v;
  }
  atomicAdd(db + c, acc);
}

}  // namespace rn

using namespace rn;

extern "C" int rn_conv2d_weight_grad(const void* x, const void* g, float* dw, int B, int H, int W, int Cin, int Cout, int kh,
                                     int kw, int fmt, void* stream) {
  if (!x || !g || !dw || B < 1 || H < 1 || W < 1 || kh < 1 || kw < 1 || kh * kw > 16) return -1;
  if (fmt != 0 && fmt != 2) return -2;                                   // fp16 or fp16 hi/lo pairs
  if (Cin % 128 != 0 || Cout % 128 != 0) return -3;
  int PX = 64, PY = 1;
  while (PX > W) { PX >>= 1; PY <<= 1; }
  if (W % PX != 0 || H % PY != 0 || PX * PY != 64) return -4;
  const int BN = (Cout % 256 == 0) ? 256 : 128;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return -8;
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.dw = dw; p.Cin = Cin; p.Cout = Cout; p.W = W; p.H = H; p.B = B; p.PX = PX; p.PY = PY; p.ntaps = kh * kw;
  const int pby = (kh - 1) / 2, pbx = (kw - 1) / 2;                      // TF SAME, stride 1: pad-before = (k-1)//2
  for (int ky = 0; ky < kh; ++ky)
    for (int kx = 0; kx < kw; ++kx) { p.tap[ky * kw + kx][0] = static_cast<int8_t>(kx - pbx); p.tap[ky * kw + kx][1] = static_cast<int8_t>(ky - pby); }
  p.m_tiles = Cin / kWgBM; p.n_tiles = Cout / BN; p.split = fmt == 2 ? 1 : 0;
  const int tiles = p.ntaps * p.m_tiles * p.n_tiles;
  const int sms = num_sms();
  int ksplit = 1;
  while (tiles * ksplit < sms && ksplit * 2 <= B) ksplit *= 2;          // fewer tiles than SMs: split the batch over CTAs
  // The tensor core truncates its fp32 accumulator once per k-step, so one long wgmma chain shrinks its sum by ~1.6e-8 per step
  // (trunk layer, B = 24 in one chain: 6144 steps, a bias of -9.9e-5).  Cap a CTA's chain at kWgMaxChainPixels (256 steps,
  // bias ~ -4e-6) by splitting the batch further; the slices are summed by round-to-nearest fp32 atomics.
  const long long chain_split = (static_cast<long long>(B) * H * W + kWgMaxChainPixels - 1) / kWgMaxChainPixels;
  if (ksplit < chain_split) ksplit = static_cast<int>(chain_split < B ? chain_split : B);
  p.ksplit = ksplit;
  const int stage_bytes = (2 + BN / 64) * kBoxBytes;
  p.stages = (kMaxSmem - 1024 - 256) / stage_bytes;
  if (p.stages > 8) p.stages = 8;
  if (p.stages < 2) return -10;
  const size_t smem = static_cast<size_t>(p.stages) * stage_bytes + 1024 + 256;
  const cuuint32_t ones[4] = {1, 1, 1, 1};
  const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(PX), static_cast<cuuint32_t>(PY), 1};
  auto encode = [&](CUtensorMap* m, const void* base, int C) -> CUresult {
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(B)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * 2, static_cast<cuuint64_t>(C) * 2 * W, static_cast<cuuint64_t>(C) * 2 * W * H};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  const long long xplane = static_cast<long long>(B) * H * W * Cin, gplane = static_cast<long long>(B) * H * W * Cout;
  CUresult r = encode(&p.tmX, x, Cin);
  if (r == CUDA_SUCCESS) r = encode(&p.tmG, g, Cout);
  if (r == CUDA_SUCCESS && p.split) r = encode(&p.tmX2, static_cast<const uint16_t*>(x) + xplane, Cin);
  if (r == CUDA_SUCCESS && p.split) r = encode(&p.tmG2, static_cast<const uint16_t*>(g) + gplane, Cout);
  if (r != CUDA_SUCCESS) return 1000 + static_cast<int>(r);
  if (ksplit > 1) {
    cudaError_t e = cudaMemsetAsync(dw, 0, static_cast<size_t>(p.ntaps) * Cin * Cout * sizeof(float), st);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  int grid = tiles * ksplit;
  if (grid > sms) grid = sms;
  const cudaError_t e = (BN == 256) ? launch_wgrad<256>(p, grid, smem, st) : launch_wgrad<128>(p, grid, smem, st);
  return e == cudaSuccess ? 0 : static_cast<int>(e);
}

extern "C" int rn_bias_grad_16(const void* g, float* db, long long npix, int C, int fmt, void* stream) {
  if (!g || !db || npix < 1 || C < 1 || (fmt != 0 && fmt != 2)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(db, 0, static_cast<size_t>(C) * sizeof(float), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  const int bx = C < 128 ? C : 128;
  dim3 grid(static_cast<unsigned>(npix < 1024 ? npix : 1024), static_cast<unsigned>((C + bx - 1) / bx));
  bias_grad_kernel<<<grid, bx, 0, st>>>(static_cast<const uint16_t*>(g), db, npix, C, fmt, npix * C);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}
