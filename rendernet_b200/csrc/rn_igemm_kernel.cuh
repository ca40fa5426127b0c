// rn_igemm_kernel.cuh -- implicit-GEMM convolution on Hopper tensor cores (wgmma) for sm_90a.
//
// One kernel serves every dense contraction of the RenderNet forward path (reference call sites:
// tools/layer_util.py:21 projection 1x1, :101-104 3x3 res blocks, :253 conv3d, :212 conv2d_transpose;
// RenderNet_Shader.py:83-129): M = output pixels/voxels, N = Cout, K = taps x Cin.
//
//   * A (activations, channel-last fp16/bf16) is never im2col'ed in memory: for filter tap (dx,dy,dz) the
//     128-row A tile is ONE tiled-TMA box {KB channels, BD, BW, BH} fetched at a shifted coordinate; TMA's
//     out-of-bounds zero fill implements TF "SAME" padding (asymmetric pads are just different offsets).
//   * B (weights) is pre-packed [tap][Cout][Cin] so a {KB, BN} box is a K-major operand tile.
//   * Both land in shared memory in the 32/64/128-byte swizzled K-major layout that wgmma reads through
//     shared-memory descriptors.
//   * Warpgroup roles: warpgroup 0 = TMA producer (one thread issues, the rest give their registers away through
//     setmaxnreg), warpgroups 1 and 2 = consumers: each issues m64nBNk16 wgmmas for 64 of the tile's 128 rows into fp32
//     register accumulators and then runs the epilogue of those rows (bias/PReLU/residual/sigmoid -> 16-byte stores).
//   * Persistent: grid = #SMs, static round-robin tile schedule with N fastest so concurrently running
//     CTAs share the same activation rows in L2.  The producer runs ahead into the next tile while the consumers drain.
//
// This header holds the device code and the per-variant launcher template `launch_ms`.  It is included only by
// rn_igemm_inst.cu, which the Makefile compiles once per <BN, CL, MS, SPLIT, HALF> variant (one object each, so that
// `make -j` spreads them over the cores); rn_igemm.cu (host side: validation, tile/pipeline sizing, tensor maps) declares
// the template and dispatches to the instantiated variants.
#pragma once
#include <atomic>
#include <cstdio>
#include <cstring>
#include <cuda_bf16.h>

#include "rn_igemm.cuh"
#include "rn_phong.cuh"
#include "rn_ptx.cuh"

namespace rn {

extern std::atomic<long long> g_launch_count;   // kernels launched by this library (bench.py's gpu_launches)

constexpr int kNumThreads = 384;                // producer warpgroup + two consumer warpgroups
constexpr int kMaxDevices = 64;                 // device ordinals with cached per-device state
constexpr int kStgCols = 32;                    // accumulator columns staged through shared memory per epilogue pass
constexpr int kStgStride = kStgCols + 4;        // floats per staged row (padding spreads the rows over the banks)
static_assert(kStgBytes == 2 * 64 * kStgStride * 4, "one 64-row staging panel per consumer warpgroup (rn_igemm.cuh)");

struct TileCoord {
  int b, x0, y0, z0, n0;
};

__device__ __forceinline__ TileCoord decode_tile(const IgemmParams& p, int tile, int BN) {
  TileCoord t;
  const int n_tile = tile % p.n_tiles;
  int m_tile = tile / p.n_tiles;
  const int per_img = p.tiles_x * p.tiles_y * p.tiles_z;
  t.b = m_tile / per_img;
  m_tile -= t.b * per_img;
  const int tz = m_tile % p.tiles_z;
  m_tile /= p.tiles_z;
  const int tx = m_tile % p.tiles_x;
  const int ty = m_tile / p.tiles_x;
  t.x0 = tx * p.BW;
  t.y0 = ty * p.BH * p.ms;
  t.z0 = tz * p.BD;
  t.n0 = n_tile * BN;
  return t;
}

// Epilogue of CW consecutive accumulator columns n0.. of one output row (element offset `off`): bias, activation, residual,
// 16-bit and/or fp32 stores.
template <int CW, bool SPLIT = false>
__device__ __forceinline__ void epilogue_chunk(const IgemmParams& p, const float* __restrict__ a, int n0, long long off,
                                               bool row_valid, int bidx) {
  if (!row_valid) return;
  float v[CW];
#pragma unroll
  for (int i = 0; i < CW; i += 4) {
    const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + i));
    v[i + 0] = a[i + 0] + b4.x;
    v[i + 1] = a[i + 1] + b4.y;
    v[i + 2] = a[i + 2] + b4.z;
    v[i + 3] = a[i + 3] + b4.w;
  }
  if (p.act == ACT_PRELU) {
#pragma unroll
    for (int i = 0; i < CW; i += 4) {
      const float4 a4 = __ldg(reinterpret_cast<const float4*>(p.alpha + n0 + i));
      v[i + 0] = fmaxf(v[i + 0], 0.f) + a4.x * fminf(v[i + 0], 0.f);
      v[i + 1] = fmaxf(v[i + 1], 0.f) + a4.y * fminf(v[i + 1], 0.f);
      v[i + 2] = fmaxf(v[i + 2], 0.f) + a4.z * fminf(v[i + 2], 0.f);
      v[i + 3] = fmaxf(v[i + 3], 0.f) + a4.w * fminf(v[i + 3], 0.f);
    }
  } else if (p.act == ACT_SIGMOID) {
#pragma unroll
    for (int i = 0; i < CW; ++i) v[i] = 1.f / (1.f + __expf(-v[i]));
  }
  if constexpr (CW == 16) {
    // Last up-conv of the Shader net (x-folded, N = F pixels x 3 channels <= 16): Phong composite + uint8 quantisation of the
    // sigmoid output while it is still in registers (tools/Phong_shading.py:202-228, RenderNet_demo.py:58).
    if (p.phong_light_dir != nullptr && p.act == ACT_SIGMOID && n0 == 0) {
      const float* ld = p.phong_light_dir + 3 * bidx;
      const float lx = __ldg(ld), ly = __ldg(ld + 1), lz = __ldg(ld + 2);
      float col[3] = {__ldg(p.phong_light_col + 3 * bidx), __ldg(p.phong_light_col + 3 * bidx + 1), __ldg(p.phong_light_col + 3 * bidx + 2)};
#pragma unroll
      for (int px = 0; px < 5; ++px) {
        if (px < p.phong_F) {
          float sh[3];
          phong_pixel(v[3 * px], v[3 * px + 1], v[3 * px + 2], lx, ly, lz, col, p.phong_ambient, p.phong_kd, p.phong_white,
                      p.phong_mask, sh);
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            if (p.out32 != nullptr) p.out32[off + 3 * px + c] = sh[c];
            if (p.out_u8 != nullptr) p.out_u8[off + 3 * px + c] = phong_u8(sh[c]);
          }
        }
      }
      return;
    }
  }
  const bool full = p.vec_ok && (n0 + CW <= p.n_valid);
  if (full) {
    if (p.res != nullptr) {
      if (p.res_is_f32) {
        const float4* rp = reinterpret_cast<const float4*>(static_cast<const float*>(p.res) + off + n0);
#pragma unroll
        for (int i = 0; i < CW / 4; ++i) {
          const float4 q = __ldg(rp + i);
          v[4 * i + 0] += q.x; v[4 * i + 1] += q.y; v[4 * i + 2] += q.z; v[4 * i + 3] += q.w;
        }
      } else {
        const uint4* rp = reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.res) + off + n0);
#pragma unroll
        for (int i = 0; i < CW / 8; ++i) {
          const uint4 q = __ldg(rp + i);
          const uint32_t w[4] = {q.x, q.y, q.z, q.w};
          if constexpr (SPLIT) {      // residual = hi + lo (exact in fp32: <= 22 significant bits)
            const uint4 ql = __ldg(rp + i + (p.o_plane >> 3));
            const uint32_t wl[4] = {ql.x, ql.y, ql.z, ql.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
              const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&wl[j]));
              v[8 * i + 2 * j] += fh.x + fl.x;
              v[8 * i + 2 * j + 1] += fh.y + fl.y;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float2 f;
              if (p.ab_fmt == 0) f = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
              else f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
              v[8 * i + 2 * j] += f.x;
              v[8 * i + 2 * j + 1] += f.y;
            }
          }
        }
      }
    }
    if (p.out16 != nullptr) {
      uint4* op = reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out16) + off + n0);
#pragma unroll
      for (int i = 0; i < CW / 8; ++i) {
        uint32_t w[4];
        if constexpr (SPLIT) {        // hi = fp16(v), lo = fp16(v - hi): two planes
          uint32_t wl[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const __half2 h = __floats2half2_rn(v[8 * i + 2 * j], v[8 * i + 2 * j + 1]);
            const float2 hf = __half22float2(h);
            const __half2 l = __floats2half2_rn(v[8 * i + 2 * j] - hf.x, v[8 * i + 2 * j + 1] - hf.y);
            w[j] = *reinterpret_cast<const uint32_t*>(&h);
            wl[j] = *reinterpret_cast<const uint32_t*>(&l);
          }
          op[i] = make_uint4(w[0], w[1], w[2], w[3]);
          op[i + (p.o_plane >> 3)] = make_uint4(wl[0], wl[1], wl[2], wl[3]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (p.ab_fmt == 0) {
              __half2 h = __floats2half2_rn(v[8 * i + 2 * j], v[8 * i + 2 * j + 1]);
              w[j] = *reinterpret_cast<uint32_t*>(&h);
            } else {
              __nv_bfloat162 h = __floats2bfloat162_rn(v[8 * i + 2 * j], v[8 * i + 2 * j + 1]);
              w[j] = *reinterpret_cast<uint32_t*>(&h);
            }
          }
          op[i] = make_uint4(w[0], w[1], w[2], w[3]);
        }
      }
    }
    if (p.out32 != nullptr) {
      float4* op = reinterpret_cast<float4*>(p.out32 + off + n0);
#pragma unroll
      for (int i = 0; i < CW / 4; ++i) op[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
  } else {
    // ragged / unaligned columns (e.g. the 3-channel image head): scalar path
#pragma unroll
    for (int i = 0; i < CW; ++i) {
      const int n = n0 + i;
      if (n < p.n_valid) {
        float x = v[i];
        if (p.res != nullptr) {
          if (p.res_is_f32) x += static_cast<const float*>(p.res)[off + n];
          else if (SPLIT) x += __half2float(static_cast<const __half*>(p.res)[off + n]) +
                                 __half2float(static_cast<const __half*>(p.res)[off + n + p.o_plane]);
          else if (p.ab_fmt == 0) x += __half2float(static_cast<const __half*>(p.res)[off + n]);
          else x += __bfloat162float(static_cast<const __nv_bfloat16*>(p.res)[off + n]);
        }
        if (p.out16 != nullptr) {
          if (SPLIT) {
            const __half h = __float2half_rn(x);
            static_cast<__half*>(p.out16)[off + n] = h;
            static_cast<__half*>(p.out16)[off + n + p.o_plane] = __float2half_rn(x - __half2float(h));
          } else if (p.ab_fmt == 0) static_cast<__half*>(p.out16)[off + n] = __float2half_rn(x);
          else static_cast<__nv_bfloat16*>(p.out16)[off + n] = __float2bfloat16_rn(x);
        }
        if (p.out32 != nullptr) p.out32[off + n] = x;
      }
    }
  }
}

// CL = thread-block-cluster size (1, 2 or 4).  The CL CTAs of a cluster work on CL consecutive M tiles of the SAME
// N tile; each loads 1/CL of every weight (B) tile and TMA-multicasts it to all of them, so B is fetched from L2
// once per cluster instead of once per CTA.  A smem stage may only be refilled when every CTA of the cluster has
// released it: the empty barrier counts the 8 consumer warps of each of the CL CTAs, and every consumer warp arrives on
// the barrier of every CTA of the cluster.
//
// MS = M sub-tiles (accumulators) per CTA tile: with MS = 2 every weight stage feeds two 128-row accumulators, halving the
// weight traffic per MAC (BN <= 128: 2 x BN/2 fp32 registers per consumer thread).
// SPLIT = operand-split "exact" mode (fmt 2, see IgemmParams::split).
// HALF = banded filter with half-tile K blocks (IgemmParams::band_half): the accumulator is kept as two N = BN/2 halves in
// separate register arrays, and an edge K block issues only the MMAs of the half it feeds.  (Selecting the MMA width at run
// time on one array makes ptxas serialise every wgmma of the kernel, so the other kernels do not carry this path.)
template <int BN, int CL, int MS, bool SPLIT, bool HALF>
__global__ void __launch_bounds__(kNumThreads, 1) igemm_kernel(const __grid_constant__ IgemmParams p) {
  static_assert(MS == 1 || (MS == 2 && BN <= 128), "two accumulators per tile need 2 x BN/2 <= 128 registers per thread");
  constexpr int NP = HALF ? 2 : 1;                             // accumulator parts per M sub-tile
  constexpr int NACC = BN / 2 / NP;                            // accumulator registers per thread, M sub-tile and part
  constexpr int JP = BN / 8 / NP;                              // 8-column blocks per part
  constexpr int SC = BN < kStgCols ? BN : kStgCols;            // columns per epilogue pass
  constexpr int TPR = SC / 16;                                 // epilogue threads per row (16 columns each)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int ny = p.ny;                                        // B tiles (ky taps) per A (halo) load
  const int sub_bytes = p.a_sub_bytes + ny * p.b_sub_bytes;   // one "group": A halo + ny weight tiles
  const int stage_bytes = p.kps * sub_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(p.stages) * stage_bytes);
  uint64_t* empty_bar = full_bar + p.stages;
  float* stg_all = reinterpret_cast<float*>(smem + static_cast<size_t>(p.stages) * stage_bytes + 256);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    if constexpr (SPLIT) { tma_prefetch_desc(&p.tmA2); tma_prefetch_desc(&p.tmB2); }
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8 * CL);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if constexpr (CL > 1) cluster_sync();   // peers' barriers are initialised before any multicast / remote arrive
  // Programmatic dependent launch (no-ops for a normally launched grid): everything above touched only kernel parameters
  // and this CTA's own shared memory, so it may run while the previous kernel of the stream drains.  Let OUR dependents be
  // scheduled as our CTAs retire, then wait for the previous grid to complete (and its writes to be visible) before any
  // thread reads or writes global memory.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int cta_rank = (CL > 1) ? static_cast<int>(cluster_ctarank()) : 0;
  // tile walk: cluster c handles "cluster tiles" c, c+nclusters, ...; cluster tile ct -> tiles (mg*CL + rank, n)
  const int ncl = static_cast<int>(gridDim.x) / CL;
  const int cl_id = static_cast<int>(blockIdx.x) / CL;
  const int num_ct = p.num_tiles / CL;
  auto tile_of = [&](int ct) { return ((ct / p.n_tiles) * CL + cta_rank) * p.n_tiles + (ct % p.n_tiles); };

  const int nx = p.ntaps / ny;
  const int total_k = nx * p.kblocks;                          // groups per tile (each = ny k-iterations of MMAs)
  const int kb_elems = p.row_bytes >> 1;

  if (warp < 4) {
    setmaxnreg_dec<40>();
    // ------------------------------------------------------------ TMA producer (one thread).  The k loop is
    // (tap, kblock)-nested so there is no division, and everything loop-invariant lives in registers: this
    // thread's issue rate bounds the whole pipeline.
    if (warp == 0 && elect_one()) {
      constexpr uint16_t kMask = static_cast<uint16_t>((1u << CL) - 1u);
      constexpr int kBRows = BN / CL;               // rows of the B tile this CTA fetches (and multicasts)
      const int kps = p.kps, kblocks = p.kblocks, stages = p.stages;
      const bool rank5 = (p.rank == 5), banded = (p.b_banded != 0), band_half = (p.band_half != 0);
      const uint32_t smem_base = smem_u32(smem), full0 = smem_u32(full_bar);
      const uint32_t a_sub = static_cast<uint32_t>(p.a_sub_bytes), sub_u = static_cast<uint32_t>(sub_bytes);
      const uint32_t b_sub = static_cast<uint32_t>(p.b_sub_bytes);
      const uint32_t a_tx = static_cast<uint32_t>(p.BD * p.BW * (p.BH * MS + ny - 1)) * p.row_bytes;
      const uint32_t kit_tx = a_tx + static_cast<uint32_t>(ny) * BN * p.row_bytes;
      const uint32_t b_off = static_cast<uint32_t>(cta_rank * kBRows * p.row_bytes);
      const int b_row = cta_rank * kBRows;
      const uint64_t mapA_hi = reinterpret_cast<uint64_t>(&p.tmA), mapB_hi = reinterpret_cast<uint64_t>(&p.tmB);
      const uint64_t mapA_lo = reinterpret_cast<uint64_t>(&p.tmA2), mapB_lo = reinterpret_cast<uint64_t>(&p.tmB2);
      constexpr bool split = SPLIT;          // pseudo-taps pick the hi / lo plane of either operand (tap[.][3])
      int stage = 0;
      uint32_t phase = 0;
      for (int ct = cl_id; ct < num_ct; ct += ncl) {
        const TileCoord t = decode_tile(p, tile_of(ct), BN);
        const int a_c0 = p.a_c_base + (t.n0 / BN) * p.a_c_ntile;
        const int bn0 = t.n0 + b_row;
        int left = total_k, j = 0, n_here = 0;
        uint32_t dst = 0, bar = 0;
        for (int kx = 0; kx < nx; ++kx) {      // tap(ky, kx) = ky*nx + kx; entry kx holds (dx, dy of ky = 0, dz)
          const int cx = t.x0 + p.tap[kx][0], cy = t.y0 + p.tap[kx][1], cz = t.z0 + p.tap[kx][2];
          const uint64_t mapA = (split && (p.tap[kx][3] & 1)) ? mapA_lo : mapA_hi;
          int ac = a_c0, bk = 0;
          for (int kb = 0; kb < kblocks; ++kb) {
            if (band_half) ac = a_c0 + static_cast<int>(p.kb_order[kb]) * kb_elems;   // blocks run in kb_order (B is packed so)
            if (j == 0) {
              n_here = min(kps, left);
              mbar_wait(&empty_bar[stage], phase ^ 1);
              bar = full0 + 8u * stage;
              mbar_expect_tx_a(bar, n_here * kit_tx);
              dst = smem_base + static_cast<uint32_t>(stage) * stage_bytes;
            }
            if (rank5) tma_a_5d(dst, mapA, bar, ac, cz, cx, cy, t.b);
            else tma_a_4d(dst, mapA, bar, ac, cx, cy, t.b);
            uint32_t bdst = dst + a_sub;
            for (int ky = 0; ky < ny; ++ky) {
              int tap = ky * nx + kx;
              const uint64_t mapB = (split && (p.tap[tap][3] & 2)) ? mapB_lo : mapB_hi;
              if (split) tap = p.tap_b[tap];
              if constexpr (CL > 1) {
                if (banded) tma_a_3d_mc(bdst + b_off, mapB, bar, kMask, 0, b_row, tap * kblocks + kb);
                else tma_a_3d_mc(bdst + b_off, mapB, bar, kMask, bk, bn0, tap);
              } else {
                if (banded) tma_a_3d(bdst, mapB, bar, 0, 0, tap * kblocks + kb);
                else tma_a_3d(bdst, mapB, bar, bk, bn0, tap);
              }
              bdst += b_sub;
            }
            ac += kb_elems; bk += kb_elems; dst += sub_u;
            if (++j == n_here) {
              j = 0; left -= n_here;
              if (++stage == stages) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ------------------------------------------------------------ consumers: MMAs of 64 rows, then their epilogue
    const int wg = (warp - 4) >> 2;                 // rows [64 wg, 64 wg + 64) of every M sub-tile
    const int wtid = threadIdx.x - 128 * (1 + wg);
    const int bf16 = p.ab_fmt;
    const int kblocks = p.kblocks;
    const int mma_per_kit = p.row_bytes >> 5;       // 32 B (= 16 elements) per k-step
    const bool wide_k1 = ny == 1 && mma_per_kit == 4;
    const int kps = p.kps, stages = p.stages;
    // descriptor = constant high part | (smem address >> 4); all operand buffers are 1024-byte aligned
    const uint64_t desc_hi = make_smem_desc(0, p.row_bytes);
    const uint32_t base16 = (smem_u32(smem) & 0x3FFFFu) >> 4;
    const uint32_t stage16 = static_cast<uint32_t>(stage_bytes) >> 4, sub16 = static_cast<uint32_t>(sub_bytes) >> 4;
    const uint32_t a16 = static_cast<uint32_t>(p.a_sub_bytes) >> 4, b16 = static_cast<uint32_t>(p.b_sub_bytes) >> 4;
    const uint32_t ady16 = static_cast<uint32_t>(p.BD * p.BW * p.row_bytes) >> 4;   // one image row of the A halo
    const uint32_t ams16 = static_cast<uint32_t>(kTileM * p.row_bytes) >> 4;          // one M sub-tile (BH image rows)
    const uint32_t awg16 = static_cast<uint32_t>(64 * wg * p.row_bytes) >> 4;          // this warpgroup's 64 rows
    const uint32_t bhalf16 = static_cast<uint32_t>((BN / 2) * p.row_bytes) >> 4;        // rows [BN/2, BN) of a B tile
    // epilogue mapping: fragment rows fr, fr + 8 (columns fc, fc + 1 of every 8-column block) are written to the staging
    // panel; thread wtid then reads row er, columns ec..ec+15 of it back and stores them
    float* stg = stg_all + wg * 64 * kStgStride;
    const int fr = 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);
    const int er = wtid / TPR, ec = (wtid % TPR) * 16;
    const int m = 64 * wg + er;
    const int zl = m % p.BD;
    const int xl = (m / p.BD) % p.BW;
    const int yl = m / (p.BD * p.BW);
    const int bar_id = 1 + wg;
    float acc[MS][NP][NACC];
    int stage = 0;
    uint32_t phase = 0;
    // frees smem stage s in every CTA of the cluster (their multicasts write into ours) once its MMAs have retired
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        if constexpr (CL == 1) mbar_arrive(&empty_bar[s]);
        else
          for (int c = 0; c < CL; ++c) mbar_arrive_cluster(&empty_bar[s], static_cast<uint32_t>(c));
      }
    };
    for (int ct = cl_id; ct < num_ct; ct += ncl) {
      int prev = -1;                                // stage whose wgmma group may still be in flight
      uint32_t scale_d = 0;
      int kbi = 0;                                  // K block (in processing order) of the current group
      for (int left = total_k; left > 0;) {
        const int n_here = min(kps, left);
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        uint32_t da = base16 + static_cast<uint32_t>(stage) * stage16;
        for (int j = 0; j < n_here; ++j) {
          uint64_t dak = desc_hi | (da + awg16), dbk = desc_hi | (da + a16);
          // banded filter: an edge K block feeds only half of the N tile -> only that half's MMA (its packed tile holds the
          // needed rows first; the very first block of a tile is always a full one)
          const uint32_t half = HALF ? p.kb_half[kbi] : 0u;
          if (++kbi == kblocks) kbi = 0;
          // One A tile and one B tile of 128-byte rows (no halo sharing; the trunk and most other layers): the four k16 steps
          // are issued back to back from a fully unrolled loop, without the runtime ky / k-step loop and its predicates between
          // the wgmmas.  Same MMAs in the same order as the general loop below, so the results are bit-identical.
          if (!HALF && wide_k1) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
              for (int s = 0; s < MS; ++s) wgmma_ss<BN>(acc[s][0], dak + s * ams16 + 2 * k, dbk + 2 * k, k == 0 ? scale_d : 1u, bf16);
            scale_d = 1;
            da += sub16;
            continue;
          }
          for (int ky = 0; ky < ny; ++ky) {       // operand ky = the halo shifted down by ky image rows
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              if (k < mma_per_kit) {
#pragma unroll
                for (int s = 0; s < MS; ++s) {
                  const uint64_t a = dak + s * ams16 + 2 * k, b = dbk + 2 * k;
                  if constexpr (!HALF) {
                    wgmma_ss<BN>(acc[s][0], a, b, scale_d, bf16);
                  } else {
                    if (half != 2) wgmma_ss<BN / 2>(acc[s][0], a, b, scale_d, bf16);
                    if (half == 0) wgmma_ss<BN / 2>(acc[s][1], a, b + bhalf16, scale_d, bf16);
                    else if (half == 2) wgmma_ss<BN / 2>(acc[s][1], a, b, scale_d, bf16);
                  }
                }
                scale_d = 1;
              }
            }
            dak += ady16;
            dbk += b16;
          }
          da += sub16;
        }
        // one group stays in flight: the previous stage is released once its MMAs have retired
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) release(prev);
        prev = stage;
        left -= n_here;
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      release(prev);
      // epilogue: accumulator fragments -> staging panel (SC columns at a time) -> one row per thread -> epilogue_chunk
      const TileCoord t = decode_tile(p, tile_of(ct), BN);
      const int x = t.x0 + xl, z = t.z0 + zl;
#pragma unroll
      for (int s = 0; s < MS; ++s) {
        const int y = t.y0 + s * p.BH + yl;
        const bool row_valid = (er < 64) && (x < p.W) && (y < p.H) && (z < p.D);
        const long long off = p.o_base + t.b * p.o_b + y * p.o_y + x * p.o_x + z * p.o_z;
#pragma unroll
        for (int c0 = 0; c0 < BN; c0 += SC) {
          named_bar_sync(bar_id, 128);              // the previous pass has read the staging panel
#pragma unroll
          for (int jj = 0; jj < SC / 8; ++jj) {
            const int j = c0 / 8 + jj;
            const float* d = acc[s][j / JP] + 4 * (j % JP);
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
            const int nc = t.n0 + c0 + ec;
            const long long offc = p.o_nsplit > 0 ? off + (nc / p.o_nsplit) * p.o_nhi + (nc % p.o_nsplit) - nc : off;
            epilogue_chunk<16, SPLIT>(p, a, nc, offc, true, t.b);
          }
        }
      }
    }
  }

  __syncthreads();
  if constexpr (CL > 1) cluster_sync();   // no CTA exits while a peer may still multicast into / arrive on it
}

// One explicit instantiation per kernel variant lives in its own object file (rn_igemm_inst.cu compiled with
// -DRN_BN=.. etc., see the Makefile's VARIANTS list); rn_igemm.cu holds the matching dispatch table.
template <int BN, int CL, int MS, bool SPLIT, bool HALF>
cudaError_t launch_ms(const IgemmParams& p, int grid, size_t smem, cudaStream_t stream) {
  // cudaFuncSetAttribute is per DEVICE (and per kernel variant): one flag per device ordinal
  static std::atomic<bool> attr_set[kMaxDevices];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(igemm_kernel<BN, CL, MS, SPLIT, HALF>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
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
  cudaLaunchAttribute attr[2];
  int na = 0;
  if constexpr (CL > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = CL;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (tuning().pdl) {       // this grid may start its prologue before the previous kernel of the stream has drained
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, igemm_kernel<BN, CL, MS, SPLIT, HALF>, p);
}

}  // namespace rn
