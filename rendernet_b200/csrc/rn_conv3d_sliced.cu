// rn_conv3d_sliced.cu -- the 3^3, 32 -> 32-channel SAME conv3d of the Shader's res1 blocks (tools/layer_util.py:60-88,
// :228-265; RenderNet_Shader.py:45-64) as a depth-sliced implicit GEMM on Hopper tensor cores (wgmma, sm_90a).
//
// Operands keep the depth-folded view of rn_conv3d_banded_same: x [B,H,W,D*32], out [B,H,W,D*32], so nothing is
// transposed.  What differs from the banded igemm path:
//   * Tile = 8 x 8 output pixels (M = 64, one consumer warpgroup) x 8 output depths x 32 channels (N = 256); the fp32
//     accumulator is 64 x 256 per warpgroup.
//   * K walk without band zeros: input depth jl (0..9 of the ten the tile reads) feeds output depths jl-2..jl only, so its
//     two k16 steps go into those three 32-column accumulator slices and nowhere else: issued MACs == algorithmic MACs.
//     Each output depth is one m64n32k16 (see sliced_depth_mmas for why not one N = 96 MMA); the slice of each MMA is a
//     compile-time offset into the accumulator array (the depth loop is unrolled).
//   * The whole filter is resident in shared memory: per (ky, kx) one K-major [96 x 32] tile holding the kz = 2, 1, 0 slices in
//     output-depth order (rn_pack_conv3d_sliced); the end depths use the same tile at a row offset of 64 / 32.  The
//     persistent CTA loads it once; afterwards only activations stream (one 10 KB TMA box = 2 input depths x 8 x 10 pixels,
//     the y halo shared by the three ky taps, per pipeline stage).
//   * Exact mode (fp16 hi/lo pairs): the passes of a tile run x_lo.w_hi, x_hi.w_lo, then x_hi.w_hi -- every correction term
//     before the full-size products, the order of the banded kernel (DESIGN.md §4).
//   * Ping-pong: the two consumer warpgroups own alternate tiles of the CTA.  An ordering barrier lets a warpgroup start its
//     MMAs only when the other has issued its last ones, so one warpgroup's epilogue (bias, PReLU, residual, stores through
//     epilogue_chunk) runs while the other keeps the tensor cores busy.
#include <atomic>
#include <cstring>
#include <type_traits>

#include "../../include/rendernet_b200.h"
#include "rn_igemm_kernel.cuh"

namespace rn {

constexpr int kSlCh = 32;                        // Cin = Cout
constexpr int kSlDepths = 8;                     // output depths per tile
constexpr int kSlBoxes = 5;                      // A boxes per (pass, kx): 2 input depths each, 10 depths in all
constexpr int kSlTapRows = 3 * kSlCh;            // rows of one (ky, kx) filter tile: kz = 2, 1, 0 x Cout
constexpr int kSlTapBytes = kSlTapRows * kSlCh * 2;          // 6 KB, K-major 64-byte rows (64-byte swizzle)
constexpr int kSlBoxBytes = 2 * kSlCh * 2 * 8 * 10;          // 10 KB: 64 channels x 8 pixels x 10 rows (128-byte swizzle)
constexpr int kSlMaxStages = 14;                 // 2 x 14 + 3 barriers fit the 256 bytes reserved for them

struct SlicedPlan {
  int planes, stages, grid, tiles;
  size_t smem;
};

static int plan_sliced(int B, int H, int W, int D, int fmt, SlicedPlan& pl) {
  if (B < 1 || H < 1 || W < 1 || D < kSlDepths || D % kSlDepths != 0) return -31;
  if (fmt < 0 || fmt > 2) return -17;
  pl.planes = fmt == 2 ? 2 : 1;
  const size_t fixed = 1024 + static_cast<size_t>(pl.planes) * 9 * kSlTapBytes + 256 + kStgBytes;
  pl.stages = static_cast<int>((kMaxSmem - fixed) / kSlBoxBytes);
  if (pl.stages > kSlMaxStages) pl.stages = kSlMaxStages;
  if (pl.stages < 3) return -10;
  pl.smem = fixed + static_cast<size_t>(pl.stages) * kSlBoxBytes;
  pl.tiles = B * ((H + 7) / 8) * ((W + 7) / 8) * (D / kSlDepths);
  pl.grid = num_sms() < pl.tiles ? num_sms() : pl.tiles;
  return 0;
}

// Two k16 steps (K = 32: one input depth) into the N-column accumulator slice `acc`; the second step reads the next 32
// bytes of the swizzle rows of both operands.
template <int N, int BF16>
__device__ __forceinline__ void sliced_mma_k32(float* acc, uint64_t a, uint64_t b) {
  wgmma_ss<N>(acc, a, b, 1u, BF16);
  wgmma_ss<N>(acc, a + 2, b + 2, 1u, BF16);
}

// The MMAs of input depth JL (0..9) of the tile: it feeds output depths [JL-2, JL] clipped to [0, 7], each through its own
// 32-row filter slice d - (JL-2) of the (ky, kx) tile (32 rows of 64 bytes = 128 descriptor units).  Every MMA is N = 32:
// ptxas keeps the wgmma pipeline only when all wgmmas on the accumulator use one width at width-aligned offsets (N = 96
// windows at 32-column steps, or N = 64 pairs mixed with N = 32 singles, make it serialise every wgmma of the kernel).
template <int JL, int BF16>
__device__ __forceinline__ void sliced_depth_mmas(float* acc, uint64_t a, uint64_t b) {
#pragma unroll
  for (int d = JL - 2; d <= JL; ++d)
    if (d >= 0 && d < kSlDepths) sliced_mma_k32<32, BF16>(acc + 16 * d, a, b + 128u * (d - (JL - 2)));
}

// One stage (A box BOX = input depths 2 BOX, 2 BOX + 1) of one (pass, kx): the three ky taps read the halo 8 pixel rows
// (1024 B = 64 units) apart, and filter tiles (ky, kx) are 3 x 6 KB (= 1152 units) apart along ky.
template <int BOX, int BF16>
__device__ __forceinline__ void sliced_box_mmas(float* acc, uint64_t da, uint64_t db) {
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const uint64_t a = da + 64u * ky, b = db + 1152u * ky;
    sliced_depth_mmas<2 * BOX, BF16>(acc, a, b);
    sliced_depth_mmas<2 * BOX + 1, BF16>(acc, a + 4, b);     // the box's second depth: +64 bytes in the 128-byte row
  }
}

// p: tmA / tmA2 = x hi / lo planes, rank 4 {D*32, W, H, B}, box {64, 8, 10, 1}; tmB = the packed filter {32, 96, planes*9},
// box {32, 96, 1}; tiles_x/y/z, num_tiles, stages; the epilogue fields as for igemm_kernel.  The operand type is a template
// parameter (BF16: bf16, else fp16) so that no run-time branch sits between the wgmmas.
template <bool SPLIT, int BF16>
__global__ void __launch_bounds__(kNumThreads, 1) conv3d_sliced_kernel(const __grid_constant__ IgemmParams p) {
  constexpr int kPlanes = SPLIT ? 2 : 1;
  constexpr int kPasses = SPLIT ? 3 : 1;
  constexpr int kSteps = kPasses * 3 * kSlBoxes;              // pipeline stages per tile
  constexpr int kFilterBytes = kPlanes * 9 * kSlTapBytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_smem = smem + kFilterBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(a_smem + static_cast<size_t>(p.stages) * kSlBoxBytes);
  uint64_t* empty_bar = full_bar + p.stages;
  uint64_t* w_bar = empty_bar + p.stages;                    // the resident filter has landed
  uint64_t* order_bar = w_bar + 1;                           // [2]: warpgroup w may start the MMAs of its next tile
  float* stg_all = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full_bar) + 256);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    if constexpr (SPLIT) tma_prefetch_desc(&p.tmA2);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);                           // the 4 warps of the warpgroup that owns the tile
    }
    mbar_init(w_bar, 1);
    mbar_init(&order_bar[0], 1);
    mbar_init(&order_bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  // programmatic dependent launch, as in igemm_kernel
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  const int G = static_cast<int>(gridDim.x);
  auto decode = [&](int tile, int& b, int& x0, int& y0, int& z0) {
    z0 = (tile % p.tiles_z) * kSlDepths;
    int r = tile / p.tiles_z;
    x0 = (r % p.tiles_x) * 8;
    r /= p.tiles_x;
    y0 = (r % p.tiles_y) * 8;
    b = r / p.tiles_y;
  };

  if (warp < 4) {
    setmaxnreg_dec<40>();
    // ------------------------------------------------------------ TMA producer (one thread): filter once, then A boxes
    if (warp == 0 && elect_one()) {
      const uint64_t mapB = reinterpret_cast<uint64_t>(&p.tmB);
      const uint64_t mapA_hi = reinterpret_cast<uint64_t>(&p.tmA), mapA_lo = reinterpret_cast<uint64_t>(&p.tmA2);
      const uint32_t wb = smem_u32(w_bar);
      mbar_expect_tx_a(wb, kFilterBytes);
      for (int t = 0; t < kPlanes * 9; ++t) tma_a_3d(smem_u32(smem) + t * kSlTapBytes, mapB, wb, 0, 0, t);
      const uint32_t a_base = smem_u32(a_smem), full0 = smem_u32(full_bar);
      const int stages = p.stages;
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += G) {
        int b, x0, y0, z0;
        decode(tile, b, x0, y0, z0);
        const int c0 = (z0 - 1) * kSlCh;                     // input depth z0 - 1 (zero filled below 0 and beyond D)
        for (int pass = 0; pass < kPasses; ++pass) {
          const uint64_t mapA = (SPLIT && pass == 0) ? mapA_lo : mapA_hi;
          for (int kx = 0; kx < 3; ++kx)
            for (int box = 0; box < kSlBoxes; ++box) {
              mbar_wait(&empty_bar[stage], phase ^ 1);
              const uint32_t bar = full0 + 8u * stage;
              mbar_expect_tx_a(bar, kSlBoxBytes);
              tma_a_4d(a_base + static_cast<uint32_t>(stage) * kSlBoxBytes, mapA, bar, c0 + 2 * kSlCh * box, x0 + kx - 1,
                       y0 - 1, b);
              if (++stage == stages) { stage = 0; phase ^= 1; }
            }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ------------------------------------------------------------ consumers: warpgroup wg owns local tiles wg, wg + 2, ...
    const int wg = (warp - 4) >> 2;
    const int wtid = threadIdx.x - 128 * (1 + wg);
    const int stages = p.stages;
    const uint64_t descA = make_smem_desc(0, 128), descB = make_smem_desc(0, 64);
    const uint32_t a16 = (smem_u32(a_smem) & 0x3FFFFu) >> 4, w16 = (smem_u32(smem) & 0x3FFFFu) >> 4;
    constexpr uint32_t kBox16 = kSlBoxBytes >> 4, kTap16 = kSlTapBytes >> 4, kPlane16 = 9 * kTap16;
    float* stg = stg_all + wg * 64 * kStgStride;
    const int fr = 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);
    const int er = wtid >> 1, ec = (wtid & 1) * 16;          // epilogue: row er (pixel (er % 8, er / 8)), 16 columns at ec
    const int bar_id = 1 + wg;
    float acc[128];
    mbar_wait(w_bar, 0);
    int cnt = wg * kSteps;                                    // pipeline step of this warpgroup's next tile
    uint32_t order_phase = 0;
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    };
    for (int local = wg, tile = blockIdx.x + wg * G; tile < p.num_tiles; local += 2, tile += 2 * G, cnt += 2 * kSteps) {
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      // The stage ring is filled in tile order, so a warpgroup may wait on its tile's stages only once the previous tile's
      // MMAs are all issued: then no stage it waits on is more than one fill ahead (mbarrier parity).
      if (local > 0) {
        mbar_wait(&order_bar[wg], order_phase);
        order_phase ^= 1;
      }
      int stage = cnt % stages;
      uint32_t phase = static_cast<uint32_t>(cnt / stages) & 1u;
      int prev = -1;
      for (int pass = 0; pass < kPasses; ++pass) {
        const uint32_t wplane = w16 + ((SPLIT && pass == 1) ? kPlane16 : 0u);
        for (int kx = 0; kx < 3; ++kx) {
          const uint64_t db = descB | (wplane + kx * kTap16);
          auto step = [&](auto box_c) {
            constexpr int BOX = decltype(box_c)::value;
            mbar_wait(&full_bar[stage], phase);
            wgmma_fence();
            sliced_box_mmas<BOX, BF16>(acc, descA | (a16 + static_cast<uint32_t>(stage) * kBox16), db);
            wgmma_commit();
            wgmma_wait<1>();                                  // the previous stage's MMAs have retired: free it
            if (prev >= 0) release(prev);
            prev = stage;
            if (++stage == stages) { stage = 0; phase ^= 1; }
          };
          step(std::integral_constant<int, 0>{});
          step(std::integral_constant<int, 1>{});
          step(std::integral_constant<int, 2>{});
          step(std::integral_constant<int, 3>{});
          step(std::integral_constant<int, 4>{});
        }
      }
      if (wtid == 0) mbar_arrive(&order_bar[wg ^ 1]);       // the other warpgroup's next tile may start
      wgmma_wait<0>();
      release(prev);
      // epilogue: accumulator fragments -> staging panel (32 columns at a time) -> one row per thread -> epilogue_chunk
      int b, x0, y0, z0;
      decode(tile, b, x0, y0, z0);
      const int x = x0 + (er & 7), y = y0 + (er >> 3);
      const bool row_valid = x < p.W && y < p.H;
      const long long off = p.o_base + b * p.o_b + y * p.o_y + x * p.o_x;
      const float wsc = SPLIT ? w_unscale_of(p) : 1.f;
#pragma unroll
      for (int c0 = 0; c0 < kSlDepths * kSlCh; c0 += kStgCols) {
        named_bar_sync(bar_id, 128);                          // the previous pass has read the staging panel
#pragma unroll
        for (int jj = 0; jj < kStgCols / 8; ++jj) {
          const float* d = acc + 4 * (c0 / 8 + jj);
          *reinterpret_cast<float2*>(stg + fr * kStgStride + 8 * jj + fc) = make_float2(d[0], d[1]);
          *reinterpret_cast<float2*>(stg + (fr + 8) * kStgStride + 8 * jj + fc) = make_float2(d[2], d[3]);
        }
        named_bar_sync(bar_id, 128);
        if (row_valid) {
          float a[16];
          const float4* sp = reinterpret_cast<const float4*>(stg + er * kStgStride + ec);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 q = sp[i];
            a[4 * i] = q.x; a[4 * i + 1] = q.y; a[4 * i + 2] = q.z; a[4 * i + 3] = q.w;
          }
          epilogue_chunk<16, SPLIT>(p, a, z0 * kSlCh + c0 + ec, off, true, b, wsc);
        }
      }
    }
  }
  __syncthreads();
}

template <bool SPLIT, int BF16>
static cudaError_t launch_sliced(const IgemmParams& p, int grid, size_t smem, cudaStream_t stream) {
  static std::atomic<bool> attr_set[kMaxDevices];            // the shared-memory opt-in is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(conv3d_sliced_kernel<SPLIT, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e != cudaSuccess) return e;
    attr_set[dev].store(true, std::memory_order_release);
  }
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (tuning().pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, conv3d_sliced_kernel<SPLIT, BF16>, p);
}

}  // namespace rn

extern "C" int rn_conv3d_sliced_plan(int B, int H, int W, int D, int fmt, int* out, int n_out) {
  rn::SlicedPlan pl;
  const int rc = rn::plan_sliced(B, H, W, D, fmt, pl);
  if (rc != 0) return rc;
  const int v[7] = {pl.stages, static_cast<int>(pl.smem), pl.grid, pl.tiles, pl.planes * 9 * rn::kSlTapBytes,
                    rn::kSlBoxBytes, rn::kMaxSmem};
  for (int i = 0; i < n_out && i < 7; ++i) out[i] = v[i];
  return 0;
}

extern "C" int rn_conv3d_sliced_same_scaled(const void* x, const void* w_sliced, const float* w_unscale,
                                            const float* bias_full, const float* alpha_full, int act, const void* residual,
                                            int residual_is_f32, void* out16, float* out32, int B, int H, int W, int D,
                                            int Cin, int Cout, int fmt, void* stream) {
  using namespace rn;
  if (x == nullptr || w_sliced == nullptr || bias_full == nullptr) return -1;
  if (w_unscale != nullptr && fmt != 2) return -26;
  if (Cin != kSlCh || Cout != kSlCh) return -4;
  if (act != ACT_NONE && act != ACT_PRELU) return -5;
  if (act == ACT_PRELU && alpha_full == nullptr) return -5;
  if (out16 == nullptr && out32 == nullptr) return -6;
  SlicedPlan pl;
  const int prc = plan_sliced(B, H, W, D, fmt, pl);
  if (prc != 0) return prc;
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return -8;

  IgemmParams p;
  memset(&p, 0, sizeof(p));
  const long long F = static_cast<long long>(D) * kSlCh;       // folded channels of x and of the output
  const long long plane = static_cast<long long>(B) * H * W * F;
  const CUtensorMapDataType dt = fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const cuuint32_t ones[4] = {1, 1, 1, 1};
  {
    const cuuint64_t dims[4] = {(cuuint64_t)F, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)F * 2, (cuuint64_t)F * 2 * W, (cuuint64_t)F * 2 * W * H};
    const cuuint32_t box[4] = {2 * kSlCh, 8, 10, 1};
    CUresult r = enc(&p.tmA, dt, 4, const_cast<void*>(x), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS && fmt == 2)
      r = enc(&p.tmA2, dt, 4, const_cast<uint16_t*>(static_cast<const uint16_t*>(x) + plane), dims, strides, box, ones,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return 1000 + static_cast<int>(r);
  }
  {
    const cuuint64_t dims[3] = {(cuuint64_t)kSlCh, (cuuint64_t)kSlTapRows, (cuuint64_t)(pl.planes * 9)};
    const cuuint64_t strides[2] = {(cuuint64_t)kSlCh * 2, (cuuint64_t)kSlTapBytes};
    const cuuint32_t box[3] = {(cuuint32_t)kSlCh, (cuuint32_t)kSlTapRows, 1};
    const CUresult r = enc(&p.tmB, dt, 3, const_cast<void*>(w_sliced), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return 2000 + static_cast<int>(r);
  }
  p.W = W; p.H = H; p.D = D; p.B = B;
  p.tiles_x = (W + 7) / 8; p.tiles_y = (H + 7) / 8; p.tiles_z = D / kSlDepths;
  p.num_tiles = pl.tiles;
  p.stages = pl.stages;
  p.ab_fmt = fmt == 1 ? 1 : 0;
  p.split = fmt == 2 ? 1 : 0;
  p.o_plane = fmt == 2 ? plane : 0;
  p.out16 = out16; p.out32 = out32; p.res = residual; p.res_is_f32 = residual_is_f32;
  p.bias = bias_full; p.alpha = alpha_full; p.act = act; p.n_valid = static_cast<int>(F);
  p.o_base = 0; p.o_x = F; p.o_y = static_cast<long long>(W) * F; p.o_b = static_cast<long long>(H) * W * F;
  p.w_unscale = w_unscale;
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec_ok = al16(out16) && al16(out32) && al16(residual) ? 1 : 0;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = fmt == 2   ? launch_sliced<true, 0>(p, pl.grid, pl.smem, st)
                        : fmt == 1 ? launch_sliced<false, 1>(p, pl.grid, pl.smem, st)
                                   : launch_sliced<false, 0>(p, pl.grid, pl.smem, st);
  return e == cudaSuccess ? 0 : static_cast<int>(e);
}

extern "C" int rn_conv3d_sliced_same(const void* x, const void* w_sliced, const float* bias_full, const float* alpha_full,
                                     int act, const void* residual, int residual_is_f32, void* out16, float* out32, int B,
                                     int H, int W, int D, int Cin, int Cout, int fmt, void* stream) {
  return rn_conv3d_sliced_same_scaled(x, w_sliced, nullptr, bias_full, alpha_full, act, residual, residual_is_f32, out16,
                                      out32, B, H, W, D, Cin, Cout, fmt, stream);
}
