// rn_igemm.cuh -- parameter block shared by the host launcher and the wgmma implicit-GEMM kernel.
#pragma once
#include <cstdint>
#include <cuda.h>

namespace rn {

constexpr int kMaxTaps = 48;   // 16 filter taps x 3 operand-split terms (fmt 2)
constexpr int kMaxSmem = 232448;   // opt-in dynamic shared memory per block on sm_90 (227 KB)
constexpr int kStgBytes = 2 * 64 * 36 * 4;   // epilogue staging: 64 rows x (32 + 4 padding) fp32 per consumer warpgroup
constexpr int kTileM = 128;  // rows (pixels / voxels) per CTA (sub-)tile: 64 per consumer warpgroup

enum Act : int { ACT_NONE = 0, ACT_PRELU = 1, ACT_SIGMOID = 2 };

// Every built igemm_kernel variant X(BN, CL, MS, SPLIT, HALF, RAW): N tile, cluster size, M sub-tiles, operand-split exact
// mode, half-tile K blocks of banded filters, raw fp32 output.  rn_igemm_inst.cu is compiled once per row (the Makefile's
// VARIANTS list, which tests/test_igemm_variants_host.py pins equal to this table); launch_variant dispatches over it and
// plan_conv rejects a plan that names no row of it.
#define RN_IGEMM_VARIANTS(X)                                                                                              \
  X(256, 1, 1, 0, 0, 0) X(256, 2, 1, 0, 0, 0) X(256, 4, 1, 0, 0, 0)                                                        \
  X(128, 1, 1, 0, 0, 0) X(128, 2, 1, 0, 0, 0) X(128, 4, 1, 0, 0, 0) X(128, 1, 2, 0, 0, 0) X(128, 2, 2, 0, 0, 0)            \
  X(128, 4, 2, 0, 0, 0)                                                                                                    \
  X(64, 1, 1, 0, 0, 0) X(64, 1, 2, 0, 0, 0) X(32, 1, 1, 0, 0, 0) X(32, 1, 2, 0, 0, 0) X(16, 1, 1, 0, 0, 0)                 \
  X(16, 1, 2, 0, 0, 0)                                                                                                     \
  /* operand-split "exact" mode (fmt 2): single CTAs */                                                                    \
  X(256, 1, 1, 1, 0, 0) X(128, 1, 1, 1, 0, 0) X(128, 1, 2, 1, 0, 0) X(64, 1, 1, 1, 0, 0) X(64, 1, 2, 1, 0, 0)              \
  X(32, 1, 1, 1, 0, 0) X(32, 1, 2, 1, 0, 0) X(16, 1, 1, 1, 0, 0) X(16, 1, 2, 1, 0, 0)                                      \
  /* banded filters (N tile 128) with half-tile K blocks */                                                                \
  X(128, 1, 1, 0, 1, 0) X(128, 2, 1, 0, 1, 0) X(128, 4, 1, 0, 1, 0) X(128, 1, 2, 0, 1, 0) X(128, 2, 2, 0, 1, 0)            \
  X(128, 4, 2, 0, 1, 0) X(128, 1, 1, 1, 1, 0) X(128, 1, 2, 1, 1, 0)                                                        \
  /* raw fp32 output (no bias): the exact-mode Winograd per-position GEMM */                                               \
  X(256, 1, 1, 1, 0, 1)

inline bool igemm_variant_built(int BN, int CL, int MS, int SP, int HF, int RW) {
#define RN_IGEMM_IS(bn, cl, ms, sp, hf, rw) \
  if (BN == bn && CL == cl && MS == ms && SP == sp && HF == hf && RW == rw) return true;
  RN_IGEMM_VARIANTS(RN_IGEMM_IS)
#undef RN_IGEMM_IS
  return false;
}

struct alignas(64) IgemmParams {
  CUtensorMap tmA;  // activations, channel-last: rank 4 {C,W,H,B} or rank 5 {C,D,W,H,B}; box {KB,[BD],BW,BH,1}
  CUtensorMap tmB;  // weights [tap][CoutPad][Cin]: rank 3 {Cin,CoutPad,taps}; box {KB,BN,1}
  CUtensorMap tmA2; // split mode (fmt 2): the LO plane of the activations, same geometry as tmA
  CUtensorMap tmB2; // split mode: the LO plane of the packed weights, same geometry as tmB
  int rank;
  int W, H, D, B;                 // extents of the output (== input) pixel space; D = 1 for rank 4
  int BW, BH, BD;                 // M (sub-)tile box, BW*BH*BD == 128
  int tiles_x, tiles_y, tiles_z;  // per image
  int n_tiles;                    // CoutPad / BN
  int num_tiles;                  // B*tiles_y*tiles_x*tiles_z*n_tiles
  int ntaps, kblocks;             // k-iterations = ntaps * kblocks, each KB = row_bytes/2 input channels
  int row_bytes;                  // 32 / 64 / 128 (== TMA + wgmma swizzle span)
  int kps;                        // k-iterations per pipeline stage
  int stages;
  int a_sub_bytes, b_sub_bytes;   // smem bytes of one k-iteration's A / B sub-buffer (1024-multiples)
  int ab_fmt;                     // 0 = fp16, 1 = bf16 (operands and 16-bit outputs)
  int a_c_base, a_c_ntile;        // A channel coordinate = a_c_base + n_tile*a_c_ntile + kb*KB (depth-folded conv3d)
  int b_banded;                   // 1: B box = (0, 0, tap*kblocks+kb) -- one banded filter shared by all N tiles
  int ms;                         // M sub-tiles per CTA tile (1 or 2): the CTA's tile is BW x (ms*BH) pixels = ms x 128 GEMM rows;
                                  // every weight (B) stage is used for ms accumulators, halving B traffic per MAC (BN <= 128)
  int ny;                         // y-halo sharing: taps are ordered tap = ky*nx + kx with dy consecutive; the ny taps of a
                                  // column share ONE A load of BH+ny-1 image rows (operand ky starts ky*BW rows into it)
  int8_t tap[kMaxTaps][4];        // (dx, dy, dz, sel) input offset of each filter tap; sel bit 0: A operand comes from the
                                  // LO plane (tmA2), bit 1: B operand comes from the LO plane (tmB2) -- split mode only
  uint8_t tap_b[kMaxTaps];        // tap coordinate of pseudo-tap t in the packed filter (== t unless split)
  // Split mode (fmt 2, "exact"): every 16-bit tensor is a PAIR of fp16 planes, hi = fp16(v), lo = fp16(v - hi), ~22
  // mantissa bits together.  Each filter tap becomes three pseudo-taps accumulated into the same accumulator tile:
  // x_hi.w_hi + x_lo.w_hi + x_hi.w_lo (the lo.lo term is below fp32 resolution); the epilogue reads a hi+lo residual and
  // writes hi and lo planes.  The reference computes these convolutions in fp32 (tools/layer_util.py:171,212,253).
  int split;
  long long o_plane;
  // Depth-folded conv3d only: the K blocks of a tap are processed in the order kb_order[0..kblocks) (a block that feeds the
  // whole N tile first, so that it initialises every accumulator column); kb_half[i] says which half of the N tile block i
  // feeds: 0 = all of it, 1 = columns [0, BN/2), 2 = columns [BN/2, BN).  The edge blocks of the band touch only half of
  // the tile's output depths, and their MMAs are issued with N = BN/2 instead of multiplying structural zeros.
  int band_half;                  // 1: kb_order / kb_half are in use
  uint8_t kb_order[8];
  uint8_t kb_half[8];              // element offset of the LO plane of out16 / of a 16-bit residual
  // fused epilogue: v = acc + bias; v = act(v); v += residual; store
  void* out16;                    // 16-bit output or nullptr
  float* out32;                   // fp32 output or nullptr
  const void* res;                // residual (same indexing as the output) or nullptr
  int res_is_f32;
  const float* bias;              // [CoutPad]
  const float* alpha;             // [CoutPad] (PReLU) or nullptr
  int act;
  int n_valid;                    // real Cout (<= CoutPad); columns beyond are dropped
  int vec_ok;                     // output/residual rows are 16B aligned -> vector path
  long long o_base, o_b, o_y, o_x, o_z;  // output element offset = o_base + b*o_b + y*o_y + x*o_x + z*o_z + n
  // Phong composite + uint8 fused into the sigmoid epilogue of the x-folded last up-conv (SURVEY §8 f-2; 16-column kernels only):
  // a GEMM row holds the 3 channels of phong_F adjacent pixels; out32 then receives the SHADED colour and out_u8 its uint8 form.
  const float* phong_light_dir;   // [B,3] or nullptr (off)
  const float* phong_light_col;   // [B,3]
  uint8_t* out_u8;                // [B,H,W,3] uint8, same element indexing as out32
  float phong_ambient, phong_kd;
  int phong_F, phong_white, phong_mask;
  int o_nsplit;                   // > 0: column n lands at (n / o_nsplit) * o_nhi + (n % o_nsplit) instead of n (merged
  long long o_nhi;                //      phases of a stride-2 transposed conv: n = (ay, ax, co))
  int b_tap_div;                  // > 0 (one-tap convs only): image b of the tile reads filter tap b / b_tap_div -- the 16
                                  // per-position GEMMs of a Winograd conv as one launch over [16*B, H/2, W/2, C]
  const float* w_unscale;         // split mode: device fp32 2^-s of a filter packed as 2^s w (the epilogue's acc * 2^-s, exact
                                  // in fp32, comes before the bias), or nullptr (s = 0)
};

// Band structure of the depth-folded 3^3 conv3d (rn_conv3d_banded_same): N tile = 128/Cout output depths x Cout, K per tap =
// the input depths those need, in blocks of 64 elements = 64/Cin depths.  Shared by the filter packer and the launcher.
struct BandLayout {
  int kblocks;
  bool any_half;
  uint8_t order[8];   // processing order of the K blocks (a full block first)
  uint8_t half[8];    // per PROCESSED block: 0 full, 1 lower half of the N tile, 2 upper half
};
inline BandLayout band_layout(int Cin, int Cout, int sz) {
  BandLayout L{};
  const int zo_n = 128 / Cout, dpb = 64 / Cin, nzi = (zo_n - 1) * sz + 3;
  L.kblocks = (nzi * Cin + 63) / 64;
  uint8_t h[8] = {0};
  int first_full = -1;
  for (int kb = 0; kb < L.kblocks && kb < 8; ++kb) {
    const int zi_lo = kb * dpb, zi_hi = (kb + 1) * dpb - 1 < nzi - 1 ? (kb + 1) * dpb - 1 : nzi - 1;
    int zo_min = (zi_lo - 2 + sz - 1) / sz;                 // smallest zo with sz*zo + 2 >= zi_lo
    if (zi_lo - 2 < 0) zo_min = 0;
    int zo_max = zi_hi / sz;                                // largest zo with sz*zo <= zi_hi
    if (zo_max > zo_n - 1) zo_max = zo_n - 1;
    const int c0 = zo_min * Cout, c1 = (zo_max + 1) * Cout; // columns [c0, c1) of the 128-column tile
    h[kb] = c1 <= 64 ? 1 : (c0 >= 64 ? 2 : 0);
    if (h[kb] == 0 && first_full < 0) first_full = kb;
  }
  int n = 0;
  if (first_full >= 0 && L.kblocks <= 8) {
    L.order[n] = static_cast<uint8_t>(first_full); L.half[n++] = 0;
    for (int kb = 0; kb < L.kblocks; ++kb)
      if (kb != first_full) { L.order[n] = static_cast<uint8_t>(kb); L.half[n] = h[kb]; L.any_half |= h[kb] != 0; ++n; }
  } else {
    for (int kb = 0; kb < L.kblocks && kb < 8; ++kb) { L.order[kb] = static_cast<uint8_t>(kb); L.half[kb] = 0; }
  }
  return L;
}

// launch-heuristic defaults (immutable after first use; RN_TUNE environment override -- rn_igemm.cu)
struct Tuning {
  int cluster = 1;        // B-multicast cluster size when the descriptor says 0.  1: on the H100 the weight multicast of a
                          // 2 / 4-CTA cluster made the 3x3 1024->1024 trunk conv 2.6x / 6.5x slower (2.60 vs 6.76 / 17.0
                          // ms per B=24 launch, fp16), the stage releases couple every CTA of the cluster
  int kps = 0;            // k-groups per pipeline stage (0 = heuristic)
  int msub = 0;           // M sub-tiles per CTA tile (0 = heuristic)
  int yhalo = 1;          // y-halo sharing of the activation operand (3x3, banded 3^3, merged / x-folded transposed)
  int tiled_tex_conv = 1; // shared-memory tiled kernel for the texture decoder's 4^3 8->4 conv (0: generic kernel; A/B, tests)
  int pdl = 0;            // programmatic dependent launch: igemm launches carry the programmatic-stream-serialization attribute,
                          // trigger their dependents after the prologue and griddepcontrol.wait before touching global memory
  int winograd = 1;       // exact-mode 3x3 trunk convs as Winograd F(2x2, 3x3) (rn_winograd.cu; 0: the direct kernel, for A/B)
  int wino_tile = 4;      // Winograd output tile: 4 = F(4x4, 3x3) where H and W are multiples of 4, 2 = always F(2x2, 3x3)
};
const Tuning& tuning();

// cuTensorMapEncodeTiled resolved through the runtime (no libcuda link), and the SM count of the current device (rn_igemm.cu)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_fn();
int num_sms();

}  // namespace rn
