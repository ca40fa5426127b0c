// rn_igemm.cu -- implicit-GEMM convolution on Hopper tensor cores (wgmma) for sm_90a.
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
//     shared-memory descriptors; fp32 accumulators live in the registers of two consumer warpgroups (64 rows each).
//   * Warpgroup roles: warpgroup 0 = TMA producer, warpgroups 1-2 = wgmma issue + epilogue
//     (bias/PReLU/residual/sigmoid -> 16B global stores).
//   * Persistent: grid = #SMs, static round-robin tile schedule with N fastest so concurrently running
//     CTAs share the same activation rows in L2.
//
// This file is the host side (argument validation, tile / pipeline sizing, TMA tensor maps); the kernel template lives
// in rn_igemm_kernel.cuh and is instantiated in rn_igemm_inst.cu.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "rn_igemm.cuh"

namespace rn {

// launch_ms<BN, CL, MS, SPLIT, HALF, RAW> is defined in rn_igemm_kernel.cuh and explicitly instantiated once per row of
// RN_IGEMM_VARIANTS (rn_igemm.cuh; rn_igemm_inst.cu x the Makefile's VARIANTS list).
template <int BN, int CL, int MS, bool SPLIT, bool HALF, bool RAW>
cudaError_t launch_ms(const IgemmParams& p, int grid, size_t smem, cudaStream_t stream);

static cudaError_t launch_variant(int BN, int CL, int MS, int SP, int HF, int RW, const IgemmParams& p, int grid, size_t smem,
                                  cudaStream_t stream) {
#define RN_V(bn, cl, ms, sp, hf, rw) \
  if (BN == bn && CL == cl && MS == ms && SP == sp && HF == hf && RW == rw) \
    return launch_ms<bn, cl, ms, (sp != 0), (hf != 0), (rw != 0)>(p, grid, smem, stream);
  RN_IGEMM_VARIANTS(RN_V)
#undef RN_V
  return cudaErrorInvalidDeviceFunction;   // unreachable: plan_conv rejects a plan without a built variant (-25)
}

// ------------------------------------------------------------------------------------------------ host side
PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

static CUtensorMapSwizzle swizzle_of(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

std::atomic<long long> g_launch_count{0};   // kernels launched by this library (bench.py's gpu_launches)

// Library defaults of the launch heuristics.  They can be overridden ONCE per process through the environment variable
// RN_TUNE ("msub=1,kps=4,cluster=4,yhalo=0"; read at first use, immutable
// afterwards -- a tuning / A-B aid, see scripts/ab_step.py) and per call through the 0-means-auto fields of rn_conv_desc.
// There is no mutable global state.
static Tuning parse_tuning() {
  Tuning t;
  const char* e = getenv("RN_TUNE");
  if (e == nullptr) return t;
  auto get = [&](const char* key, int* dst, int lo, int hi) {
    const char* q = strstr(e, key);
    if (q == nullptr || q[strlen(key)] != '=') return;
    const int v = atoi(q + strlen(key) + 1);
    if (v >= lo && v <= hi) *dst = v;
  };
  get("cluster", &t.cluster, 1, 4);
  get("kps", &t.kps, 0, 16);
  get("msub", &t.msub, 0, 2);
  get("yhalo", &t.yhalo, 0, 1);
  get("tiled_tex_conv", &t.tiled_tex_conv, 0, 1);
  get("pdl", &t.pdl, 0, 1);
  get("winograd", &t.winograd, 0, 1);
  get("wino_tile", &t.wino_tile, 2, 4);
  if (t.wino_tile != 2) t.wino_tile = 4;
  return t;
}
const Tuning& tuning() {
  static const Tuning t = parse_tuning();
  return t;
}

// SM count of the CURRENT device (cached per device ordinal); 132 (H100 SXM) when no device is visible (rn_conv_plan on a
// CPU host)
int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    cudaGetLastError();
    return 132;
  }
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      return 132;
    }
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

}  // namespace rn

#include "../../include/rendernet_b200.h"

extern "C" long long rn_launch_count(void) { return rn::g_launch_count.load(std::memory_order_relaxed); }

namespace rn {
struct ConvPlan {
  int BN, CL, grid, sub, KB, D;
  bool raw;   // no bias: plain fp32 output stored straight from the accumulators (no staging panel)
  size_t smem;
};

// Everything rn_conv_igemm decides before it touches the device: N tile, M tile box, halo sharing, M sub-tiles, cluster
// size, pipeline depth, shared-memory size.  Pure host arithmetic on the
// descriptor (pointers are only tested for null / alignment), so rn_conv_plan can report it on a machine without a GPU.
static int plan_conv(const rn_conv_desc* d, IgemmParams& p, ConvPlan& pl) {
  if (d == nullptr || d->x == nullptr || d->w_packed == nullptr) return -1;
  // bias == NULL: raw fp32 output, the accumulators as they are (only out32, every column a real one)
  const bool raw = d->bias == nullptr;
  if (raw && (d->act != ACT_NONE || d->residual != nullptr || d->out16 != nullptr || d->out32 == nullptr ||
              d->phong != nullptr || d->o_nsplit != 0 || d->Cout != d->cout_pad))
    return -24;
  if (d->ndim != 2 && d->ndim != 3) return -2;
  if (d->ntaps < 1 || d->ntaps * (d->fmt == 2 ? 3 : 1) > kMaxTaps) return -3;
  if (d->fmt < 0 || d->fmt > 2) return -17;
  const bool res16 = d->residual != nullptr && !d->residual_is_f32;
  if (d->fmt == 2 && (d->x_plane <= 0 || d->w_plane <= 0 || ((d->out16 != nullptr || res16) && d->o_plane <= 0) ||
                      d->x_plane % 8 != 0 || d->w_plane % 8 != 0 || d->o_plane % 8 != 0))
    return -18;   // fp16 hi/lo pairs: the LO plane of every 16-bit tensor must be given (16-byte aligned offsets)
  if (d->Cin % 16 != 0 || d->cout_pad % 16 != 0 || d->Cout > d->cout_pad || d->Cout < 1) return -4;
  if (d->act == ACT_PRELU && d->alpha == nullptr) return -5;
  if (d->cta_group > 1) return -22;         // sm_90 has no paired (two-CTA) MMA
  if (d->out16 == nullptr && d->out32 == nullptr) return -6;
  const int D = d->ndim == 3 ? d->D : 1;
  if (d->B < 1 || d->H < 1 || d->W < 1 || D < 1) return -7;
  if (d->b_tap_div < 0 || (d->b_tap_div > 0 && (d->ntaps != 1 || d->w_banded || d->B % d->b_tap_div != 0))) return -23;
  if (d->w_unscale != nullptr && (d->fmt != 2 || raw)) return -26;   // only the exact-mode epilogue applies it

  const Tuning& tn = tuning();
  const bool split = d->fmt == 2;
  memset(&p, 0, sizeof(p));
  p.w_unscale = d->w_unscale;
  // K block: as many input channels as fit one 128/64/32-byte swizzle row
  p.row_bytes = (d->Cin % 64 == 0) ? 128 : ((d->Cin % 32 == 0) ? 64 : 32);
  const int KB = p.row_bytes / 2;
  p.kblocks = d->Cin / KB;
  p.ntaps = d->ntaps;
  // N tile
  int BN = 16;
  for (int c : {256, 128, 64, 32, 16})
    if (d->cout_pad % c == 0) { BN = c; break; }
  if (d->force_bn > 0) {
    if (d->cout_pad % d->force_bn != 0) return -9;
    BN = d->force_bn;
  }
  p.n_tiles = d->cout_pad / BN;
  // y-halo sharing of the A operand between the ny taps of a filter column (3x3 convs, banded 3^3)
  p.ny = 1;
  if (d->ny > 1) {
    if (d->ndim != 2 || d->ntaps % d->ny != 0) return -13;
    const int nxh = d->ntaps / d->ny;
    for (int kx = 0; kx < nxh; ++kx)
      for (int ky = 0; ky < d->ny; ++ky) {
        const int8_t* t0 = d->taps + 3 * kx;
        const int8_t* t1 = d->taps + 3 * (ky * nxh + kx);
        if (t1[0] != t0[0] || t1[1] != t0[1] + ky || t1[2] != t0[2]) return -14;
      }
    p.ny = d->ny;
  }
  // M tile box (BD x BW x BH == 128, innermost spatial dim first), launch shape and pipeline sizing.  If the y-halo
  // variant cannot keep >= 3 stages in flight (tiny images -> no CTA pairing -> 3 full-width B tiles per group),
  // fall back to one A load per tap.
  auto pow2_le = [](int v, int cap) { int r = 1; while (r * 2 <= cap && r < v) r *= 2; return r; };
  if (split) {
    p.ntaps = 3 * d->ntaps;
    p.split = 1;
  }
  p.ab_fmt = d->fmt == 1 ? 1 : 0;
  if (d->w_banded && d->band_cin > 0) {     // depth-folded conv3d: K-block order / half-tile blocks (rn_igemm.cuh band_layout)
    if (d->force_bn != 128 || d->band_cout < 8 || 128 % d->band_cout != 0 || d->band_cin < 8 || 64 % d->band_cin != 0 ||
        d->band_sz < 1 || d->band_sz > 2)
      return -19;
    const BandLayout L = band_layout(d->band_cin, d->band_cout, d->band_sz);
    if (L.kblocks != p.kblocks || L.kblocks > 8) return -19;
    p.band_half = 1;                        // the packed filter is in processing order even when no block is a half block
    for (int i = 0; i < L.kblocks; ++i) { p.kb_order[i] = L.order[i]; p.kb_half[i] = L.half[i]; }
  }
  p.b_tap_div = d->b_tap_div;
  p.rank = d->ndim == 3 ? 5 : 4;
  p.W = d->W; p.H = d->H; p.D = D; p.B = d->B;
  int grid = 0, CL = 1, sub = 0;
  // M sub-tiles: two 128-row accumulators per CTA share every weight stage (BN <= 128, so that 2 x BN/2 accumulator
  // registers per consumer thread fit).  Halves the weight bytes per MAC.
  int want_ms = d->msub > 0 ? d->msub : (tn.msub > 0 ? tn.msub : 2);
  if (want_ms > 2) return -16;
  if (BN > 128 || d->ndim != 2) want_ms = 1;
  const int stg_bytes = raw ? 0 : kStgBytes;   // the epilogue's staging panel
  const int budget = kMaxSmem - 1024 - 256 - stg_bytes;
  for (int attempt = 0; attempt < 3; ++attempt) {
    p.ms = want_ms;
    int rem = kTileM;
    p.BD = d->ndim == 3 ? pow2_le(D, rem) : 1;
    rem /= p.BD;
    p.BW = pow2_le(d->W, rem);
    if (p.ny > 1) {   // tall tiles keep the halo overhead low: (BH+ny-1)/BH
      const int tw = d->tile_w > 0 ? d->tile_w : 16;
      if (p.BW > tw) p.BW = tw;
      if (p.BW < 8 || (p.BW * p.row_bytes) % 1024 != 0) p.ny = 1;   // operand ky must start on a swizzle-atom boundary
      if (p.ny == 1) p.BW = pow2_le(d->W, rem);
    }
    rem /= p.BW;
    p.BH = rem;
    p.tiles_x = (d->W + p.BW - 1) / p.BW;
    if (p.ms == 2 && d->H < 2 * p.BH) p.ms = 1;       // nothing to pair
    p.tiles_y = (d->H + p.BH * p.ms - 1) / (p.BH * p.ms);
    p.tiles_z = (D + p.BD - 1) / p.BD;
    p.num_tiles = d->B * p.tiles_x * p.tiles_y * p.tiles_z * p.n_tiles;
    // persistent grid, cluster size CL for the B multicast (split kernels run on single CTAs)
    grid = num_sms();
    if (d->max_ctas > 0 && d->max_ctas < grid) grid = d->max_ctas;
    if (grid > p.num_tiles) grid = p.num_tiles;
    const int m_tiles = p.num_tiles / p.n_tiles;
    CL = 1;
    if (BN >= 128 && !split) {
      const int want = d->cluster > 0 ? d->cluster : tn.cluster;
      if (want >= 4 && m_tiles % 4 == 0 && grid >= 4) CL = 4;
      else if (want >= 2 && m_tiles % 2 == 0 && grid >= 2) CL = 2;
    }
    grid -= grid % CL;
    p.a_sub_bytes = ((p.BD * p.BW * (p.BH * p.ms + p.ny - 1) * p.row_bytes + 1023) / 1024) * 1024;
    p.b_sub_bytes = ((BN * p.row_bytes + 1023) / 1024) * 1024;
    sub = p.a_sub_bytes + p.ny * p.b_sub_bytes;       // one group: A (halo) + ny weight tiles
    const int total_k = (p.ntaps / p.ny) * p.kblocks;
    // groups per stage: ~64 KB stages amortise the per-stage barrier round trips
    p.kps = (65536 + sub / 2) / sub;
    if (p.kps < 1) p.kps = 1;
    if (p.kps > 8) p.kps = 8;
    if (p.kps > total_k) p.kps = total_k;
    if (d->force_kps > 0) p.kps = d->force_kps;
    else if (tn.kps > 0) p.kps = tn.kps < total_k ? tn.kps : total_k;
    p.stages = budget / (p.kps * sub);
    if (p.stages > 12) p.stages = 12;
    while (p.stages < 3 && p.kps > 1) {   // keep at least 3 stages in flight
      --p.kps;
      p.stages = budget / (p.kps * sub);
    }
    if (p.stages >= 3 || (p.ny == 1 && p.ms == 1)) break;
    if (want_ms > 1) want_ms = 1;           // retry with one accumulator per tile,
    else p.ny = 1;                          // then without halo sharing
  }
  if (p.stages < 2) return -10;
  if (!igemm_variant_built(BN, CL, p.ms, p.split, p.band_half, raw ? 1 : 0)) return -25;
  if (!split) {
    for (int t = 0; t < d->ntaps; ++t) {
      p.tap[t][0] = d->taps[3 * t + 0];
      p.tap[t][1] = d->taps[3 * t + 1];
      p.tap[t][2] = d->taps[3 * t + 2];
      p.tap[t][3] = 0;
      p.tap_b[t] = static_cast<uint8_t>(t);
    }
  } else {
    // Split ("exact") mode: tap t = ky*nx0 + kx0 becomes three pseudo-taps with the same input offset:
    // (x_lo, w_hi), (x_hi, w_lo), (x_hi, w_hi).  Order along the k loop: ALL correction terms of the tile first, the hi.hi
    // terms last.  The tensor core's fp32 accumulation truncates (round toward zero, one truncation per MMA step), so the
    // error of a step scales with the magnitude the accumulator has at that moment: while only 2^-11-sized corrections
    // have been summed it is negligible, and only the hi.hi third of the steps runs against the full-size accumulator
    // (DESIGN.md §4).  Within each of the three
    // passes the ky-major order that y-halo sharing needs is preserved: pseudo kx' = j*nx0 + kx0, tap = ky*(3*nx0) + kx'
    // (built from the FINAL ny: without halo sharing nx0 = ntaps and the order is simply j-major).
    const int nx0 = d->ntaps / p.ny;
    for (int t = 0; t < d->ntaps; ++t) {
      const int ky = t / nx0, kx0 = t % nx0;
      for (int j = 0; j < 3; ++j) {          // j = 0: x_lo.w_hi, 1: x_hi.w_lo, 2: x_hi.w_hi
        const int q = ky * (3 * nx0) + j * nx0 + kx0;
        p.tap[q][0] = d->taps[3 * t + 0];
        p.tap[q][1] = d->taps[3 * t + 1];
        p.tap[q][2] = d->taps[3 * t + 2];
        p.tap[q][3] = static_cast<int8_t>(j == 0 ? 1 : (j == 1 ? 2 : 0));
        p.tap_b[q] = static_cast<uint8_t>(t);
      }
    }
  }
  pl.BN = BN; pl.CL = CL; pl.grid = grid; pl.sub = sub; pl.KB = KB; pl.D = D; pl.raw = raw;
  pl.smem = static_cast<size_t>(p.stages) * p.kps * sub + 1024 + 256 + stg_bytes;
  return 0;
}
}  // namespace rn

extern "C" int rn_conv_plan(const rn_conv_desc* d, int* out, int n_out) {
  rn::IgemmParams p;
  rn::ConvPlan pl;
  const int rc = rn::plan_conv(d, p, pl);
  if (rc != 0) return rc;
  // cta_group is always 1 and the epilogue always the two consumer warpgroups' direct stores (mode 0)
  const int v[16] = {pl.BN, pl.CL, 1, p.ms, 2, p.ny, p.BW, p.BH, p.BD, p.kps, p.stages, static_cast<int>(pl.smem),
                     pl.grid, p.num_tiles, 0, p.row_bytes};
  for (int i = 0; i < n_out && i < 16; ++i) out[i] = v[i];
  return 0;
}

extern "C" int rn_conv_igemm(const rn_conv_desc* d, void* stream_v) {
  using namespace rn;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  IgemmParams p;
  ConvPlan pl;
  const int prc = plan_conv(d, p, pl);
  if (prc != 0) return prc;
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return -8;
  const int BN = pl.BN, CL = pl.CL, grid = pl.grid, KB = pl.KB, D = pl.D;
  const size_t smem = pl.smem;

  const CUtensorMapDataType dt = d->fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const bool split = d->fmt == 2;
  const uint16_t* x_lo = split ? static_cast<const uint16_t*>(d->x) + d->x_plane : nullptr;
  const uint16_t* w_lo = split ? static_cast<const uint16_t*>(d->w_packed) + d->w_plane : nullptr;
  const cuuint32_t ones[5] = {1, 1, 1, 1, 1};
  CUresult r;
  const cuuint64_t Cx = d->x_channels > 0 ? d->x_channels : d->Cin;  // channel extent of x (>= K per tap)
  if (Cx % 8 != 0) return -11;
  p.a_c_base = d->a_c_base; p.a_c_ntile = d->a_c_ntile; p.b_banded = d->w_banded;
  if (d->w_banded && (d->force_bn <= 0)) return -12;
  if (p.rank == 4) {
    const cuuint64_t dims[4] = {Cx, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->B};
    const cuuint64_t strides[3] = {Cx * 2, Cx * 2 * d->W, Cx * 2 * d->W * d->H};
    const cuuint32_t box[4] = {(cuuint32_t)KB, (cuuint32_t)p.BW, (cuuint32_t)(p.BH * p.ms + p.ny - 1), 1};
    r = enc(&p.tmA, dt, 4, const_cast<void*>(d->x), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS && split)
      r = enc(&p.tmA2, dt, 4, const_cast<uint16_t*>(x_lo), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
              swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const cuuint64_t dims[5] = {Cx, (cuuint64_t)D, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->B};
    const cuuint64_t strides[4] = {Cx * 2, Cx * 2 * D, Cx * 2 * D * d->W, Cx * 2 * D * d->W * d->H};
    const cuuint32_t box[5] = {(cuuint32_t)KB, (cuuint32_t)p.BD, (cuuint32_t)p.BW, (cuuint32_t)p.BH, 1};
    r = enc(&p.tmA, dt, 5, const_cast<void*>(d->x), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS && split)
      r = enc(&p.tmA2, dt, 5, const_cast<uint16_t*>(x_lo), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
              swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return 1000 + static_cast<int>(r);
  const uint16_t* w_hi = static_cast<const uint16_t*>(d->w_packed);
  if (d->w_banded) {  // [ntaps*kblocks][BN][KB], identical for every N tile
    const cuuint64_t dims[3] = {(cuuint64_t)KB, (cuuint64_t)BN, (cuuint64_t)d->ntaps * p.kblocks};
    const cuuint64_t strides[2] = {(cuuint64_t)KB * 2, (cuuint64_t)KB * 2 * BN};
    const cuuint32_t box[3] = {(cuuint32_t)KB, (cuuint32_t)(BN / CL), 1};  // each CTA of a cluster fetches 1/CL of B
    r = enc(&p.tmB, dt, 3, const_cast<uint16_t*>(w_hi), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS && split)
      r = enc(&p.tmB2, dt, 3, const_cast<uint16_t*>(w_lo), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
              swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const int btaps = d->b_tap_div > 0 ? d->ntaps * (d->B / d->b_tap_div) : d->ntaps;   // taps of the packed filter
    const cuuint64_t dims[3] = {(cuuint64_t)d->Cin, (cuuint64_t)d->cout_pad, (cuuint64_t)btaps};
    const cuuint64_t strides[2] = {(cuuint64_t)d->Cin * 2, (cuuint64_t)d->Cin * 2 * d->cout_pad};
    const cuuint32_t box[3] = {(cuuint32_t)KB, (cuuint32_t)(BN / CL), 1};  // each CTA of a cluster fetches 1/CL of B
    r = enc(&p.tmB, dt, 3, const_cast<uint16_t*>(w_hi), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS && split)
      r = enc(&p.tmB2, dt, 3, const_cast<uint16_t*>(w_lo), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
              swizzle_of(p.row_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return 2000 + static_cast<int>(r);

  p.out16 = d->out16; p.out32 = d->out32; p.res = d->residual; p.res_is_f32 = d->residual_is_f32;
  p.bias = d->bias; p.alpha = d->alpha; p.act = d->act; p.n_valid = d->Cout;
  p.o_base = d->o_base; p.o_b = d->o_b; p.o_y = d->o_y; p.o_x = d->o_x; p.o_z = d->o_z;
  p.o_nsplit = d->o_nsplit; p.o_nhi = d->o_nhi;
  p.o_plane = d->o_plane;
  if (d->phong != nullptr) {      // fused Phong composite (16-column kernels, sigmoid epilogue, direct fp32 / uint8 stores)
    if (BN != 16 || d->act != ACT_SIGMOID || d->Cout % 3 != 0 || d->Cout > 15 || d->o_nsplit != 0 || d->residual != nullptr ||
        d->phong->light_dir == nullptr || d->phong->light_col == nullptr || (d->out32 == nullptr && d->phong->out_u8 == nullptr))
      return -21;
    p.phong_light_dir = d->phong->light_dir; p.phong_light_col = d->phong->light_col; p.out_u8 = d->phong->out_u8;
    p.phong_ambient = d->phong->ambient; p.phong_kd = d->phong->k_diffuse; p.phong_F = d->Cout / 3;
    p.phong_white = d->phong->background_white; p.phong_mask = d->phong->with_mask;
  }
  if (d->o_nsplit > 0 && (d->o_nsplit % 32 != 0 || d->o_nhi % 8 != 0)) return -15;
  const bool strides8 = (d->o_base % 8 == 0) && (d->o_b % 8 == 0) && (d->o_y % 8 == 0) && (d->o_x % 8 == 0) &&
                        (d->o_z % 8 == 0);
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec_ok = strides8 && al16(d->out16) && al16(d->out32) && al16(d->residual) ? 1 : 0;
  if (pl.raw && !p.vec_ok) return -24;    // the raw epilogue stores float2 pairs without a scalar fallback

  const cudaError_t e = launch_variant(BN, CL, p.ms, p.split, p.band_half, pl.raw ? 1 : 0, p, grid, smem, stream);
  return e == cudaSuccess ? 0 : static_cast<int>(e);
}
