/* rendernet_b200.h -- C ABI of librendernet_b200.so: the H100 (sm_90a) kernels behind RenderNet's
 * forward-rendering hot path.
 *
 * The reference (thunguyenphuoc/RenderNet) is pure Python over TensorFlow-1 and has NO FFI of its own;
 * its boundary is the set of graph-building Python functions cited per entry point below (file:line into
 * the reference tree).  A maintainer would bind these with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - Every pointer is a DEVICE pointer unless stated otherwise; the caller owns every buffer (the
 *     library never allocates device memory).  `stream` is a cudaStream_t passed as void*; calls are
 *     asynchronous and stream-ordered and may be issued from any thread on any device.  The library has NO mutable
 *     global state: what it caches is immutable once set (per-device kernel attributes / SM counts, and the launch-
 *     heuristic defaults, which the environment variable RN_TUNE can override once per process -- a tuning aid);
 *     per-call overrides go through the 0-means-auto fields of rn_conv_desc.  The only counter is rn_launch_count().
 *   - Tensors are channel-last and dense: 2-D [B,H,W,C], 3-D [B,H,W,D,C] (D innermost spatial axis),
 *     exactly the reference's layouts (tools/layer_util.py:228,147; SURVEY.md §8b).
 *   - "16-bit" tensors (`fmt`): RN_FMT_F16 = IEEE fp16, RN_FMT_BF16 = bfloat16, RN_FMT_F16X2 = "exact" mode: a PAIR of
 *     fp16 planes stored back to back, [2][numel]: plane 0 = hi = fp16(v), plane 1 = lo = fp16(v - hi), together ~22
 *     significant bits while |v| >= 2^-3 (below, lo is an fp16 subnormal: an absolute step of 2^-25).  In that mode every
 *     convolution evaluates x_hi.w_hi + x_lo.w_hi + x_hi.w_lo on the tensor cores (3x the MMAs) and matches the reference's
 *     fp32 convolutions (tools/layer_util.py:171,212,253) to ~1e-6 relative; packed filters, 16-bit activations, residuals
 *     and outputs are all such pairs (buffers twice the size).  The networks' packed filters carry a per-layer power-of-two
 *     exponent (2^s w, rn_conv_desc::w_unscale), so any filter scale packs to the same bits; activations are not rescaled and hold
 *     the bars for x ~ N(0,1) 2^k from k = -9 (F(4x4): k = -5) up to the range limits (DESIGN.md §4).
 *     Accumulation is always fp32.
 *   - Return value: 0 = ok; <0 = invalid argument (see source for the code); >0 = CUDA / driver error.
 */
#ifndef RENDERNET_B200_H_
#define RENDERNET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RN_FMT_F16 0
#define RN_FMT_BF16 1
#define RN_FMT_F16X2 2 /* fp16 hi/lo pairs, "exact" mode */

#define RN_ACT_NONE 0
#define RN_ACT_PRELU 1   /* max(0,x) + alpha[c]*min(0,x)    tools/layer_util.py:27-45 */
#define RN_ACT_SIGMOID 2 /* tf.nn.sigmoid                   RenderNet_Shader.py:127,130 */
#define RN_ACT_ELU 3     /* tf.nn.elu: x < 0 ? exp(x) - 1 : x   Reconstruct_RenderNet_Face.py:48-69 (rn_conv3d_f32 only) */

int rn_version(void);
const char* rn_error_string(int code);
/* number of kernels this library has launched in this process (host-side counter) */
long long rn_launch_count(void);
/* ---- resampler ----------------------------------------------------------------------------------
 * Replaces tf_resampling + tf_interpolate + tf_voxel_meshgrid (tools/resampling_voxel_grid.py:381-614)
 * fused with tf_transform_voxel_to_match_image (tools/model_util.py:41-49).
 *   vox   [B,size,size,size,C] fp32        minv [B,3,4] fp32 = inverse(T'.S.R.T)[:, :3, :] (:579-602)
 *   out   [B,new,new,new,C] fp32
 * transform=0: out[b,i,j,k,c] = sample(minv . (k,j,i,1))           (tf_resampling output)
 * transform=1: out[b,p,q,r,c] = sample(minv . (r,new-1-p,q,1))     (+ axis transform, the network input)
 * Corner clamp / weight rule of :410-485: points with any source coordinate outside [0,size-1) give 0. */
int rn_resample_f32(const float* vox, const float* minv, float* out, int B, int C, int size, int new_size,
                    int transform, void* stream);
/* A patch window of rn_resample_f32(transform=1) (random-patch training, tools/model_util.py:77-161): rows p in [y0, y0+ph),
 * columns q in [x0, x0+pw), every depth r.  out [B,ph,pw,new_size,C] fp32 = out_full[:, y0:y0+ph, x0:x0+pw], bit for bit.
 * C = 1 or 4; ph, pw multiples of 16, 0 <= y0 <= new_size-ph, 0 <= x0 <= new_size-pw (else -2).  The same window rule holds
 * for every *_window entry point below. */
int rn_resample_window_f32(const float* vox, const float* minv, float* out, int B, int C, int size, int new_size, int y0, int x0,
                           int ph, int pw, void* stream);

/* tf_interpolate (tools/resampling_voxel_grid.py:381-486) at caller-supplied coordinates: x, y, z [B*n_per_item] fp32
 * (sampler x addresses the LAST spatial axis of vox, z the first: flat = b*S^3 + z*S^2 + y*S + x, :427-449),
 * out [B*n_per_item, C] fp32.  Bit-faithful to the reference arithmetic everywhere, including the clamped-corner weight
 * cancellation outside the cube (which rn_resample_f32 replaces by exact zeros). */
int rn_interpolate_f32(const float* vox, const float* x, const float* y, const float* z, float* out, int B, int C, int size,
                       long long n_per_item, void* stream);

/* ---- weight packing -------------------------------------------------------------------------------
 * TF filter (fp32) -> [n_sel][cout_pad][Cin] 16-bit, K-major rows for the tensor-core kernel.
 *   transposed=0: w is [ntaps_total][Cin][Cout]   (tf.nn.conv2d / conv3d filters, layer_util.py:162,243)
 *   transposed=1: w is [ntaps_total][Cout][Cin]   (tf.nn.conv2d_transpose filters, layer_util.py:201)
 * tap_sel (HOST pointer, n_sel ints) selects/reorders source taps; rows co >= Cout are zero. */
int rn_pack_conv_weights(const float* w, void* packed, int ntaps_total, int Cin, int Cout, int cout_pad,
                         int transposed, const int* tap_sel, int n_sel, int fmt, void* stream);
/* fp32 -> 16-bit cast with zero padding of the tail: dst[0..n_pad) */
int rn_cast_f32_to_16(const float* src, void* dst, long long n, long long n_pad, int fmt, void* stream);
int rn_cast_16_to_f32(const void* src, float* dst, long long n, int fmt, void* stream);

/* y = act(x + bias[c]) + residual over a 16-bit channel-last tensor of n elements (c = index % C).
 * Standalone tools/layer_util.py:27-45 prelu / tf.add / tf.nn.sigmoid when not fused into a conv epilogue. */
int rn_bias_act_16(const void* x, const float* bias, const float* alpha, int act, const void* residual,
                   void* out16, float* out32, long long n, int C, int fmt, void* stream);

/* ---- tensor-core implicit-GEMM convolution (wgmma + TMA) ------------------------------------------
 * out[b,y,x,z,n] = act( bias[n] + sum_t sum_ci  x[b, y+dy_t, x+dx_t, z+dz_t, ci] * w_packed[t][n][ci] ) + residual
 * with zero outside the input (TF SAME padding is expressed through the tap offsets).
 * The output element offset is o_base + b*o_b + y*o_y + x*o_x + z*o_z + n, which lets one call write a
 * strided sub-lattice (the 4 phases of a stride-2 transposed convolution). */
/* Phong composite + uint8 quantisation (tools/Phong_shading.py:202-228, RenderNet_demo.py:58) fused into the sigmoid epilogue of
 * the Shader net's last up-conv (rn_conv2d_transpose_s1_xfold with Cout = 3): out32 then receives the SHADED colour instead of
 * the normal map, out_u8 (may be NULL) its clip(255 x) uint8 form; bit-identical to rn_phong_composite applied afterwards. */
typedef struct rn_phong {
  const float* light_dir;   /* [B,3] */
  const float* light_col;   /* [B,3] */
  uint8_t* out_u8;          /* [B,H,W,3] or NULL */
  float ambient, k_diffuse;
  int background_white, with_mask;
} rn_phong;

typedef struct rn_conv_desc {
  int ndim;                 /* 2 or 3 spatial dims */
  int B, H, W, D;           /* extents (D ignored for ndim == 2) */
  int Cin;                  /* multiple of 16 */
  int Cout;                 /* real output channels */
  int cout_pad;             /* rows of w_packed / entries of bias, alpha; multiple of 16 */
  int ntaps;                /* <= 48 (<= 16 for RN_FMT_F16X2: every tap expands to 3 operand-split terms) */
  const int8_t* taps;       /* HOST pointer: ntaps x (dx, dy, dz) */
  const void* x;            /* 16-bit [B,H,W,(D),Cin] */
  const void* w_packed;     /* 16-bit [ntaps][cout_pad][Cin] */
  const float* bias;        /* fp32 [cout_pad], or NULL: the raw fp32 sums, stored straight from the accumulators (out32
                             * only, act none, no residual, Cout = cout_pad, 8-byte aligned rows).  The only kernel built for
                             * it is the exact-mode (fmt 2) one with N tile 256 and no banded filter (rn_winograd_gemm);
                             * any other raw plan is rejected with -25 */
  const float* alpha;       /* fp32 [cout_pad] or NULL */
  int act;                  /* RN_ACT_* */
  const void* residual;     /* NULL, or same indexing as the output */
  int residual_is_f32;
  void* out16;              /* 16-bit output or NULL */
  float* out32;             /* fp32 output or NULL */
  long long o_base, o_b, o_y, o_x, o_z;
  int fmt;                  /* RN_FMT_* */
  int force_bn, force_kps, max_ctas; /* 0 = auto (tuning / tests) */
  /* depth-folded ("banded") conv3d: x is [B,H,W,x_channels] with x_channels = D*C, Cin = K elements read per
   * tap starting at channel a_c_base + n_tile*a_c_ntile (may run out of range: zero filled), and w_packed is one
   * banded filter [ntaps*Cin/KB][force_bn][KB] shared by all N tiles.  All zero for ordinary convolutions. */
  int x_channels, a_c_base, a_c_ntile, w_banded;
  /* geometry of the depth-folded conv3d behind a banded filter (channels per depth of x / of the output, z stride; 0 = not
   * given): lets the launcher issue the edge K blocks of the band, which touch only half of the N tile's output depths,
   * as N = 64 MMAs instead of multiplying structural zeros.  w_packed must then come from rn_pack_conv3d_banded (K blocks in
   * processing order, the rows a half tile needs first). */
  int band_cin, band_cout, band_sz;
  int cluster;              /* thread-block-cluster size for the weight-tile TMA multicast: 0 auto, 1, 2 or 4 */
  int cta_group;            /* 0 auto or 1 (single-CTA MMA); anything else is rejected: sm_90 has no paired MMA */
  /* y-halo sharing (2-D only): taps ordered tap = ky*nx + kx with dy(ky) = dy(0) + ky; the ny taps of a filter column
   * then share one activation load of BH+ny-1 image rows.  0/1 = off.  tile_w: M-tile width override (0 = 16).
   * msub: M sub-tiles per CTA tile -- 2 = two 128-row accumulators share every weight stage (Cout tile <= 128; halves
   * the weight traffic per MAC), 1 = off, 0 = auto (on for banded filters). */
  int ny, tile_w, msub;
  /* column split of the output address: n -> (n / o_nsplit) * o_nhi + (n % o_nsplit); 0 = off (multiple of 32) */
  int o_nsplit;
  long long o_nhi;
  /* fmt == RN_FMT_F16X2: element offsets of the LO plane of x, of w_packed and of out16 / a 16-bit residual (multiples
   * of 8; o_plane > 0 whenever out16 or a 16-bit residual is given, else -18).  The reference-shaped wrappers below
   * derive them from the tensor shapes ([2][numel] pairs). */
  long long x_plane, w_plane, o_plane;
  /* accepted and ignored (kept so that the struct layout stays stable): the sm_90 kernel has a single epilogue form, two
   * consumer warpgroups storing their own rows directly */
  int epi_groups, res_prefetch, tma_store;
  const rn_phong* phong;    /* NULL, or the fused Phong epilogue (act = RN_ACT_SIGMOID, N = F pixels x 3 channels <= 16) */
  /* > 0 (ntaps == 1 only): image b reads filter tap b / b_tap_div of w_packed, which then holds B / b_tap_div taps -- the
   * 16 per-position GEMMs of a Winograd convolution as one launch.  0 = off. */
  int b_tap_div;
  /* RN_FMT_F16X2 only: DEVICE pointer to one fp32 2^-s, where w_packed holds 2^s w (the filter exponent, DESIGN.md §4: s puts
   * max |2^s w| in (2^11, 2^12], so that the LO halves of small filters stay fp16 normals).  The epilogue multiplies the
   * accumulator by it before the bias, which is exact in fp32.  NULL = s = 0, today's bits.  Read on the device, so a re-pack
   * chooses s without a host synchronisation. */
  const float* w_unscale;
} rn_conv_desc;
/* Besides the argument codes of the source, -25 = no kernel variant is built for the plan (N tile, cluster, M sub-tiles,
 * exact mode, banded half blocks, raw output) that the descriptor leads to; rn_conv_plan reports it as well.  -26 = a
 * w_unscale with fmt != RN_FMT_F16X2 or with a raw (bias NULL) plan. */
int rn_conv_igemm(const rn_conv_desc* d, void* stream);
/* Per-call overrides of the launch heuristics for the reference-shaped wrappers below (their last argument before
 * `stream`; NULL = library defaults).  0 = default for every field; cluster 1/2/4; cta_group 1; kps = k-groups per
 * pipeline stage; msub 1/2 M sub-tiles; yhalo: 1 = on, -1 = off; epilogue_groups / res_prefetch / tma_store are ignored.
 * Every combination computes bit-identical results (tests/test_gpu_kernels.py::*_bit_identical). */
typedef struct rn_tuning {
  int cluster, cta_group, kps, msub, epilogue_groups, res_prefetch, tma_store, yhalo;
  int winograd;             /* rn_conv2d_winograd_eligible: 1 = on, -1 = off (the direct kernel), 0 = default (RN_TUNE) */
  int wino_tile;            /* rn_conv2d_winograd_tile: 4 = F(4x4, 3x3) where H, W % 4 == 0, 2 = F(2x2, 3x3), 0 = default
                             * (RN_TUNE wino_tile, else 4) */
} rn_tuning;
/* The launch plan rn_conv_igemm would use for `d`, without touching the device (works on a host without a GPU; the SM
 * count then defaults to 132).  Pointers in `d` are only tested for null / 16-byte alignment.  out[0..n_out) receives
 * {N tile, cluster size, cta_group, M sub-tiles, epilogue warp groups, ny (halo sharing), tile W, tile H, tile D,
 *  k-groups per stage, stages, dynamic shared memory bytes, grid, tiles, epilogue mode (always 0: direct stores),
 *  swizzle row bytes}; n_out <= 16.  Same status codes as rn_conv_igemm. */
int rn_conv_plan(const rn_conv_desc* d, int* out, int n_out);

/* Reference-shaped wrappers over rn_conv_igemm (stride 1, TF SAME), 16-bit in/out:
 * slim.conv2d / layer_util.conv2d (layer_util.py:147, RenderNet_Shader.py:83,87,98,102),
 * layer_util.conv3d (:228), projection_unit's 1x1 conv (:8-22). */
int rn_conv2d_same(const void* x, const void* w_packed, const float* bias, const float* alpha, int act,
                   const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                   int Cin, int Cout, int cout_pad, int kh, int kw, int fmt, const rn_tuning* tune, void* stream);
int rn_conv3d_same(const void* x, const void* w_packed, const float* bias, const float* alpha, int act,
                   const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                   int D, int Cin, int Cout, int cout_pad, int k, int fmt, const rn_tuning* tune, void* stream);
/* Every exact-mode wrapper has a companion rn_*_scaled that takes one more argument right after the packed filter:
 * w_unscale, a DEVICE pointer to the fp32 2^-s of a filter packed as 2^s w (rn_conv_desc::w_unscale; NULL or fmt != 2 with
 * NULL = the plain entry point, bit for bit; non-NULL with fmt != RN_FMT_F16X2 = -26).  The pack functions take the filter as
 * given, so the caller scales it by 2^s first (ops.exact_filter). */
int rn_conv2d_same_scaled(const void* x, const void* w_packed, const float* w_unscale, const float* bias, const float* alpha,
                          int act, const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                          int Cin, int Cout, int cout_pad, int kh, int kw, int fmt, const rn_tuning* tune, void* stream);
int rn_conv3d_same_scaled(const void* x, const void* w_packed, const float* w_unscale, const float* bias, const float* alpha,
                          int act, const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W,
                          int D, int Cin, int Cout, int cout_pad, int k, int fmt, const rn_tuning* tune, void* stream);
/* layer_util.conv3d 3^3 SAME stride 1 (res_block_3d, tools/layer_util.py:60-88; RenderNet_Shader.py:45-64) as a
 * depth-folded 2-D convolution: the D axis is part of the GEMM's N (128 = (128/Cout) output depths x Cout) and K
 * ((128/Cout + 2) input depths x Cin, padded to 64-element blocks), so TMA moves full 128-byte rows and each
 * activation byte is fetched from L2 9x instead of 27x.  w_banded from rn_pack_conv3d_banded
 * ([9][kblocks][128][64] 16-bit, bytes =
 * rn_conv3d_banded_bytes per plane; RN_FMT_F16X2: twice that, LO plane after the HI plane); bias/alpha are per Cout (length Cout) and are
 * expanded over depth internally via bias_full/alpha_full scratch [D*Cout] fp32 supplied by the caller
 * (fill them with rn_expand_channels).  x: [B,H,W,D,Cin]; residual, out: [B,H,W,ceil(D/sz),Cout], 16-bit.
 * sz = stride along D (1: res blocks / e_conv3; 2: e_conv2's stride (1,1,2), RenderNet_Shader.py:41), TF SAME pads. */
long long rn_conv3d_banded_bytes(int Cin, int Cout, int sz);
int rn_pack_conv3d_banded(const float* w, void* packed, int Cin, int Cout, int sz, int fmt, void* stream);
int rn_expand_channels(const float* v, float* v_full, int C, int D, void* stream);
int rn_conv3d_banded_same(const void* x, const void* w_banded, const float* bias_full, const float* alpha_full,
                          int act, const void* residual, int residual_is_f32, void* out16, float* out32, int B,
                          int H, int W, int D, int Cin, int Cout, int sz, int fmt, const rn_tuning* tune, void* stream);
int rn_conv3d_banded_same_scaled(const void* x, const void* w_banded, const float* w_unscale, const float* bias_full,
                                 const float* alpha_full, int act, const void* residual, int residual_is_f32, void* out16,
                                 float* out32, int B, int H, int W, int D, int Cin, int Cout, int sz, int fmt,
                                 const rn_tuning* tune, void* stream);

/* The same 3^3 SAME stride-1 conv3d for Cin = Cout = 32 (res1, res_block_3d at RenderNet_Shader.py:45-64; tools/layer_util.py:60-88)
 * as a depth-sliced kernel (rn_conv3d_sliced.cu): tiles of 8 x 8 pixels x 8 output depths, each input depth issued as
 * N = 96 MMAs into the three output depths it feeds (no band zeros), the whole filter resident in shared memory.
 * w_sliced from rn_pack_conv3d_sliced: [9 = (ky,kx)][96 = (2 - kz)*32 + co][32 = ci] 16-bit (9*96*32 elements per plane;
 * RN_FMT_F16X2: the LO plane follows).  x: [B,H,W,D,32], residual / out: [B,H,W,D,32] (16-bit, residual optionally fp32);
 * bias_full / alpha_full [D*32] as for rn_conv3d_banded_same; act RN none or PReLU; any B, H, W; D a multiple of 8.
 * rn_conv3d_sliced_plan reports {stages, dynamic shared memory bytes, grid, tiles, filter bytes, stage bytes, smem limit}
 * without touching a device. */
int rn_pack_conv3d_sliced(const float* w, void* packed, int fmt, void* stream);
int rn_conv3d_sliced_same(const void* x, const void* w_sliced, const float* bias_full, const float* alpha_full, int act,
                          const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W, int D,
                          int Cin, int Cout, int fmt, void* stream);
int rn_conv3d_sliced_same_scaled(const void* x, const void* w_sliced, const float* w_unscale, const float* bias_full,
                                 const float* alpha_full, int act, const void* residual, int residual_is_f32, void* out16,
                                 float* out32, int B, int H, int W, int D, int Cin, int Cout, int fmt, void* stream);
int rn_conv3d_sliced_plan(int B, int H, int W, int D, int fmt, int* out, int n_out);

/* 3x3 SAME stride-1 conv2d, C -> C channels, RN_FMT_F16X2 only, as Winograd F(2x2, 3x3) (rn_winograd.cu): 16 products per
 * 2x2 output block instead of 36, and 16 accumulations of K = C instead of one of K = 9C.
 *   rn_winograd_in:   x [2][B,H,W,C] hi/lo -> V [2][16][B,H/2,W/2,C] hi/lo, V = B^T d B of every 4x4 input patch (SAME zero
 *                     padding), summed in fp32 from hi + lo and split once.
 *   rn_winograd_gemm: M [16][B,H/2,W/2,C] fp32 = V . U per position: one igemm launch (b_tap_div = B, bias NULL: the raw
 *                     sums, stored straight from the accumulators), C a multiple of 256.
 *                     u [2][16][C][C] hi/lo: U = G g G^T of the filter per position, [position][Cout][Cin] (ops.winograd_filter).
 *   rn_winograd_out:  y = A^T M A of every 2x2 block, then bias, PReLU / none, the residual and the stores exactly as the
 *                     igemm epilogue does them (out16 hi/lo and/or out32).
 * rn_conv2d_winograd runs the three on `workspace` (rn_winograd_workspace_bytes(B, H, W, C) bytes: V then M).
 * rn_conv2d_winograd_eligible says whether ops.conv2d takes the Winograd path for a layer of this shape (fmt 2,
 * 3x3, H and W even, Cin = Cout = a multiple of 256 >= 1024, tune->winograd / RN_TUNE winograd not off; tune->winograd = 1
 * also takes Cin < 1024).  Host-only. */
long long rn_winograd_workspace_bytes(int B, int H, int W, int C);
int rn_conv2d_winograd_eligible(int fmt, int kh, int kw, int H, int W, int Cin, int Cout, int cout_pad, const rn_tuning* tune);
int rn_winograd_in(const void* x, void* v, int B, int H, int W, int C, void* stream);
int rn_winograd_gemm(const void* v, const void* u, float* m, int B, int H, int W, int C, const rn_tuning* tune, void* stream);
int rn_winograd_out(const float* m, const float* bias, const float* alpha, int act, const void* residual, int residual_is_f32,
                    void* out16, float* out32, int B, int H, int W, int C, void* stream);
int rn_conv2d_winograd(const void* x, const void* u, const float* bias, const float* alpha, int act, const void* residual,
                       int residual_is_f32, void* out16, float* out32, int B, int H, int W, int C, void* workspace,
                       long long workspace_bytes, const rn_tuning* tune, void* stream);
/* F(2x2) of a filter packed with an exponent: u = G (2^s g) G^T, and the epilogue multiplies A^T M A by w_unscale = 2^-s. */
int rn_winograd_out_scaled(const float* m, const float* w_unscale, const float* bias, const float* alpha, int act,
                           const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W, int C,
                           void* stream);
int rn_conv2d_winograd_scaled(const void* x, const void* u, const float* w_unscale, const float* bias, const float* alpha,
                              int act, const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H,
                              int W, int C, void* workspace, long long workspace_bytes, const rn_tuning* tune, void* stream);

/* The same convolution as Winograd F(4x4, 3x3): 36 products per 4x4 output block (2.25 per pixel instead of 4), V and M
 * 2.25x the activation instead of 4x.  Interpolation points 0, +-1, +-1/2, infinity; powers of two keep V and U in range
 * without adding a rounding (rn_winograd.cu).  H and W multiples of 4.
 *   rn_winograd4_in:   x [2][B,H,W,C] hi/lo -> V [2][36][B,H/4,W/4,C] hi/lo, V = 1/2 B^T d B of every 6x6 input patch.
 *   rn_winograd4_gemm: M [36][B,H/4,W/4,C] fp32 = V . U per position, one igemm launch as rn_winograd_gemm;
 *                      u [2][36][C][C] hi/lo: U = 2^u_exp G g G^T, [position][Cout][Cin] (ops.winograd_filter(L, 4)).
 *   rn_winograd4_out:  y = 2^(1 - u_exp) A^T M A of every 4x4 block (|u_exp| <= 100), then the igemm epilogue.
 * rn_conv2d_winograd4 runs the three on `workspace` (rn_winograd4_workspace_bytes(B, H, W, C) bytes: V then M).
 * rn_conv2d_winograd_tile: 0 where rn_conv2d_winograd_eligible says no, else the output tile ops.conv2d runs: 4 where H and W
 * are multiples of 4 and tune->wino_tile / RN_TUNE wino_tile is not 2, else 2.  Host-only. */
int rn_conv2d_winograd_tile(int fmt, int kh, int kw, int H, int W, int Cin, int Cout, int cout_pad, const rn_tuning* tune);
long long rn_winograd4_workspace_bytes(int B, int H, int W, int C);
int rn_winograd4_in(const void* x, void* v, int B, int H, int W, int C, void* stream);
int rn_winograd4_gemm(const void* v, const void* u, float* m, int B, int H, int W, int C, const rn_tuning* tune, void* stream);
int rn_winograd4_out(const float* m, const float* bias, const float* alpha, int act, const void* residual, int residual_is_f32,
                     void* out16, float* out32, int B, int H, int W, int C, int u_exp, void* stream);
int rn_conv2d_winograd4(const void* x, const void* u, int u_exp, const float* bias, const float* alpha, int act,
                        const void* residual, int residual_is_f32, void* out16, float* out32, int B, int H, int W, int C,
                        void* workspace, long long workspace_bytes, const rn_tuning* tune, void* stream);

/* slim.conv2d_transpose / layer_util.conv2d_transpose (layer_util.py:186; RenderNet_Shader.py:106-129),
 * SAME, out = in*stride.  w_packed holds the stride^2 phase filters back to back, as produced by
 * rn_pack_conv2d_transpose_weights: [phase = ay*s+ax][taps_of_phase][cout_pad][Cin]. */
int rn_pack_conv2d_transpose_weights(const float* w, void* packed, int kh, int kw, int Cin, int Cout,
                                     int cout_pad, int stride, int fmt, void* stream);
int rn_conv2d_transpose_same(const void* x, const void* w_packed, const float* bias, const float* alpha, int act,
                             void* out16, float* out32, int B, int H, int W, int Cin, int Cout, int cout_pad,
                             int kh, int kw, int stride, int fmt, const rn_tuning* tune, void* stream);
int rn_conv2d_transpose_same_scaled(const void* x, const void* w_packed, const float* w_unscale, const float* bias,
                                    const float* alpha, int act, void* out16, float* out32, int B, int H, int W, int Cin,
                                    int Cout, int cout_pad, int kh, int kw, int stride, int fmt, const rn_tuning* tune,
                                    void* stream);

/* Stride-2, k = 4 SAME transposed conv (e_conv7/8/9, RenderNet_Shader.py:106-119) as ONE launch: rows = input pixels,
 * N = (ay, ax, co) = 4*Cout, 9 taps (dy,dx in {-1,0,1}) with the unused phase/tap combinations zero in the packed
 * filter [9][4*Cout][Cin]; each thread writes two full 2*Cout-element runs of the 2x2 output block.  bias4 / alpha4:
 * per-Cout vectors tiled 4 times.  (The 4-launch phase form is rn_conv2d_transpose_same.) */
int rn_pack_conv2d_transpose_s2_merged(const float* w, void* packed, int Cin, int Cout, int fmt, void* stream);
int rn_conv2d_transpose_s2_merged(const void* x, const void* w_merged, const float* bias4, const float* alpha4, int act,
                                  void* out16, float* out32, int B, int H, int W, int Cin, int Cout, int fmt,
                                  const rn_tuning* tune, void* stream);
int rn_conv2d_transpose_s2_merged_scaled(const void* x, const void* w_merged, const float* w_unscale, const float* bias4,
                                         const float* alpha4, int act, void* out16, float* out32, int B, int H, int W,
                                         int Cin, int Cout, int fmt, const rn_tuning* tune, void* stream);

/* Thin-channel stride-1 transposed conv (e_conv10 32->16, e_conv11 16->3 at 512^2; RenderNet_Shader.py:122-129) with
 * F = 64/Cin adjacent x-pixels folded into the channel axis: rows of the implicit GEMM are pixel groups, K = F*Cin
 * (= one 128-byte TMA row), N = F*Cout, and the kw x-taps collapse into 3 group offsets.  rn_xfold_factor returns F
 * (1 = not applicable).  bias_x / alpha_x: per-Cout vectors tiled F times, zero padded to cout_pad >= F*Cout. */
int rn_xfold_factor(int Cin, int W);
int rn_pack_conv2d_transpose_xfold(const float* w, void* packed, int kh, int kw, int Cin, int Cout, int F, int cout_pad,
                                   int fmt, void* stream);
int rn_conv2d_transpose_s1_xfold(const void* x, const void* w_xfold, const float* bias_x, const float* alpha_x, int act,
                                 void* out16, float* out32, int B, int H, int W, int Cin, int Cout, int kh, int kw, int F,
                                 int cout_pad, int fmt, const rn_phong* phong, const rn_tuning* tune, void* stream);
int rn_conv2d_transpose_s1_xfold_scaled(const void* x, const void* w_xfold, const float* w_unscale, const float* bias_x,
                                        const float* alpha_x, int act, void* out16, float* out32, int B, int H, int W,
                                        int Cin, int Cout, int kh, int kw, int F, int cout_pad, int fmt,
                                        const rn_phong* phong, const rn_tuning* tune, void* stream);

/* ---- thin 3-D convolutions on CUDA cores (too few channels for the tensor pipe) ---------------------
 * tf.nn.conv3d SAME + bias + PReLU (layer_util.py:228-265, RenderNet_Shader.py:36-43): e_conv1 (Cin=1,
 * 5^3, stride 2) and e_conv2 (Cin=8, 3^3, stride (1,1,2)).  x fp32 or 16-bit, w fp32 TF layout
 * [k,k,k,Cin,Cout], out 16-bit [B,H/sy,W/sx,D/sz,Cout]. */
int rn_conv3d_direct(const void* x, int x_is_f32, const float* w, const float* bias, const float* alpha,
                     void* out16, int B, int H, int W, int D, int Cin, int Cout, int k, int sy, int sx, int sz,
                     int fmt, void* stream);

/* ---- resampler (+) e_conv1, fused (SURVEY 8 f-1) -----------------------------------------------------
 * tf_rotation_resampling (tools/resampling_voxel_grid.py:381-614) + tf_transform_voxel_to_match_image
 * (tools/model_util.py:41-49) + conv3d 5^3 stride 2, 1 -> 8 + bias + PReLU (RenderNet_Shader.py:36-39) without
 * materialising the new_size^3 grid; tiles whose inputs are all exactly 0 skip the convolution.  Bit-identical to
 * rn_resample_f32(transform=1) followed by rn_conv3d_direct.  vox fp32 [B,size^3] (C = 1), minv fp32 [B,3,4],
 * w fp32 [5,5,5,1,8], bias/alpha fp32 [8] (alpha NULL = no activation), out16 [B,(new_size/2)^3,8];
 * new_size % 16 == 0. */
int rn_resample_conv1_fused(const float* vox, const float* minv, const float* w, const float* bias,
                            const float* alpha, void* out16, int B, int size, int new_size, int fmt, void* stream);
/* rn_resample_conv1_fused on the window (y0, x0, ph, pw) of the transformed grid (rn_resample_window_f32's rule): e_conv1's SAME
 * padding applies at the window's borders (points outside the window are zero, as when the grid is sliced before the conv).
 * out16 [B,ph/2,pw/2,new_size/2,8]; bit-identical to rn_resample_window_f32 (C = 1) -> rn_conv3d_direct on [B,ph,pw,new,1].
 * The full window (0, 0, new_size, new_size) is rn_resample_conv1_fused. */
int rn_resample_conv1_fused_window(const float* vox, const float* minv, const float* w, const float* bias, const float* alpha,
                                   void* out16, int B, int size, int new_size, int y0, int x0, int ph, int pw, int fmt,
                                   void* stream);

/* The same fusion for the Texture/Normal network's input (BASELINE config 4; RenderNet_Texture_Face_Normal.py:155-179):
 * tf_rotation_resampling of the geometry grid (vox fp32 [B,size^3], C = 1) AND of the decoded texture volume (tex fp32
 * [B,size^3,4], 16-byte aligned) with the same pose + axis transform + tf.concat(axis=4) (:178) + e_conv1 5^3 stride 2,
 * 5 -> 8 (w fp32 [5,5,5,5,8]) + bias + PReLU, one kernel; bit-identical to rn_resample_f32 x2 -> rn_concat_channels_f32 ->
 * rn_conv3d_direct. */
int rn_resample5_conv1_fused(const float* vox, const float* tex, const float* minv, const float* w, const float* bias,
                             const float* alpha, void* out16, int B, int size, int new_size, int fmt, void* stream);
/* rn_resample5_conv1_fused on a window (y0, x0, ph, pw), as rn_resample_conv1_fused_window: out16 [B,ph/2,pw/2,new_size/2,8],
 * bit-identical to rn_resample_window_f32 (C = 1 and C = 4) -> rn_concat_channels_f32 -> rn_conv3d_direct. */
int rn_resample5_conv1_fused_window(const float* vox, const float* tex, const float* minv, const float* w, const float* bias,
                                    const float* alpha, void* out16, int B, int size, int new_size, int y0, int x0, int ph, int pw,
                                    int fmt, void* stream);

/* ---- binvox run-length decode on the device (tools/binvox_rw.py:84-93; SURVEY 8 f-2) ----------------------
 * pairs: the raw (value, count) byte pairs of n_items files back to back; run_start[r] = number of voxels before run r
 * WITHIN its item (exclusive prefix sum of the counts, host-computed); item_first_run[i] = index of item i's first
 * run, item_first_run[n_items] = total runs.  out fp32 [n_items, d0, d2, d1] for fix_coords = 1 (the reference's
 * transpose(0, 2, 1); what RenderNet_demo.py:125-127 feeds as [1,64,64,64,1]) or [n_items, d0, d1, d2] for 0. */
int rn_binvox_decode(const uint8_t* pairs, const int* run_start, const int* item_first_run, float* out, int n_items,
                     int d0, int d1, int d2, int fix_coords, void* stream);

/* ---- texture decoder (BASELINE config 4; RenderNet_Texture_Face_Normal.py:34-46) ----------------------------
 * fully_connected (tools/layer_util.py:311-343): y[B,N] = prelu(x[B,K] . w[K,N] + bias[N]; alpha[N]); fp32 in,
 * 16-bit and/or fp32 out; B <= 32.  alpha NULL -> no activation. */
int rn_fully_connected(const float* x, const float* w, const float* bias, const float* alpha, void* out16,
                       float* out32, int B, int K, int N, int fmt, void* stream);
/* conv3d / conv3d_transpose with <= 8 channels (layer_util.py:228-309), TF SAME, cubic kernel k, isotropic stride,
 * + bias + PReLU.  w in TF layout: forward [k,k,k,Cin,Cout], transposed [k,k,k,Cout,Cin].  x [B,H,W,D,Cin]. */
int rn_conv3d_small(const void* x, int x_is_f32, const float* w, const float* bias, const float* alpha, void* out16,
                    float* out32, int B, int H, int W, int D, int Cin, int Cout, int k, int stride, int transposed,
                    int fmt, void* stream);
/* tf.concat([a, b], axis=4) of fp32 channel-last tensors with n points (RenderNet_Texture_Face_Normal.py:178) */
int rn_concat_channels_f32(const float* a, const float* b, float* out, long long n, int Ca, int Cb, void* stream);

/* ---- Phong composite (tools/Phong_shading.py:138-228, RenderNet_demo.py:54-58) -----------------------
 * img [B,H,W,3] fp32 normal map in [0,1]; light_dir [B,3]; light_col [B,3]; out_f32 [B,H,W,3] and/or
 * out_u8 = clip(255*out,0,255) as uint8.  background: 0 = "Black" (threshold 150), 1 = white (80). */
int rn_phong_composite(const float* img, const float* light_dir, const float* light_col, float ambient,
                       float k_diffuse, int background_white, int with_mask, float* out_f32, uint8_t* out_u8,
                       int B, int H, int W, void* stream);
/* Shaded image of a normal map and an albedo: shade = Phong composite of `normal` [B,H,W,3] fp32, compos = albedo * shade (fp32,
 * one multiply; albedo NULL: compos = shade).  composite = RN_PHONG_NUMPY: rn_phong_composite's arithmetic (tools/Phong_shading.py:
 * 138-228); RN_PHONG_TF: TensorFlow's tf_phong_composite (:24-113), bit-identical to the shading rn_phong_recon_loss_grad
 * measures (white mask sigmoid(255 (sqrt 3 - |n|) - 80), black sigmoid(255 |n| - 80), evaluated in double).  light_dir,
 * light_col [B,3]; background_white selects the mask (and the colour the background is composited to).  Outputs, each NULL or
 * [B,H,W,3]: shade_f32, compos_f32, compos_u8 = clip(255 compos, 0, 255) truncated to uint8 (RenderNet_demo.py:58).  At least
 * one must be given.  rn_phong_composite is this entry with RN_PHONG_NUMPY, no albedo and compos as its output. */
#define RN_PHONG_NUMPY 0
#define RN_PHONG_TF 1
int rn_phong_shade(const float* normal, const float* albedo, const float* light_dir, const float* light_col, float ambient,
                   float k_diffuse, int composite, int background_white, int with_mask, float* shade_f32, float* compos_f32,
                   uint8_t* compos_u8, int B, int H, int W, void* stream);
/* rn_phong_shade with the ambient term per item: ambient [B] fp32 on the device (the fitted shading of
 * rn_phong_shade_backward_params and the fits).  The arithmetic is the scalar entry's, with the value loaded instead of passed:
 * a uniform ambient array gives rn_phong_shade's bits. */
int rn_phong_shade_ambient(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                           const float* ambient, float k_diffuse, int composite, int background_white, int with_mask,
                           float* shade_f32, float* compos_f32, uint8_t* compos_u8, int B, int H, int W, void* stream);

/* ---- backward pass: input gradients of the forward path (SURVEY 8 f-4) --------------------------------------------
 * What inverse rendering differentiates through the frozen network (Reconstruct_RenderNet_Face.py:383-412).  The data
 * gradient of every stride-1 convolution / transposed convolution is itself a convolution and runs through rn_conv_igemm
 * (mirrored taps, filters packed with the channel roles swapped: rendernet_b200/backward.py); these are the remaining pieces. */
/* dL/d(pre) = g * (y > 0 ? 1 : alpha[c]); 16-bit in/out, n elements, C = innermost (channel) extent (tools/layer_util.py:27-45).
 * `y` decides the side of the kink: the stored post-activation output works while every slope is >= 0; with a negative slope
 * (y = alpha*pre > 0 for pre < 0) pass the PRE-activation instead (rendernet_b200/backward.py re-runs the layer without its
 * PReLU in that case, and always in the training step, whose slope gradient needs it anyway). */
int rn_prelu_backward_16(const void* g, const void* y, const float* alpha, void* out, long long n, int C, int fmt, void* stream);
/* Network output img = sigmoid(logits) (RenderNet_Shader.py:127-130): out16[p, c] = scale * g[p,c] * img[p,c] * (1 - img[p,c])
 * for c < C, 0 for C <= c < Cpad (the last up-conv's data-gradient GEMM needs K % 16 == 0).  g, img fp32 [npix, C]. */
int rn_sigmoid_backward(const float* g, const float* img, void* out16, long long npix, int C, int Cpad, float scale, int fmt,
                        void* stream);
/* Data gradient of the thin strided tf.nn.conv3d SAME layers (e_conv1 5^3 s2 1|5->8, e_conv2 3^3 s(1,1,2) 8->16;
 * RenderNet_Shader.py:36-43): g16 [B,Ho,Wo,Do,Cout] 16-bit, w fp32 TF layout [k,k,k,Cin,Cout] -> dx16 (16-bit) and/or
 * dx32 (fp32, multiplied by out_scale) [B,H,W,D,Cin]. */
int rn_conv3d_backward_data_direct(const void* g16, const float* w, void* dx16, float* dx32, int B, int H, int W, int D, int Cin,
                                   int Cout, int k, int sy, int sx, int sz, float out_scale, int fmt, void* stream);
/* Backward of rn_resample_f32: gout = dL/dout [B,new,new,new,C] fp32 -> dvox [B,size^3,C] += (scatter-add of the 8 corner
 * weights; may be NULL) and dminv [B,3,4] += dL/d(inverse sampling matrix) (may be NULL).  Both are ACCUMULATED into: zero
 * them first.  Points outside the cube contribute nothing (the forward writes exact zeros there).  C = 1 or 4. */
int rn_resample_backward_f32(const float* vox, const float* minv, const float* gout, float* dvox, float* dminv, int B, int C,
                             int size, int new_size, int transform, void* stream);
/* Backward of rn_resample5_conv1_fused's input chain (Texture net, RenderNet_Texture_Face_Normal.py:155-179 /
 * Reconstruct_RenderNet_Face.py:367-378: two axis-transformed resamplings with one pose, concatenated): gout = dL/d(concat)
 * [B,new,new,new,5] fp32 -> dvox [B,size^3,1] (channel 0), dtex [B,size^3,4] (channels 1..4, 16-byte aligned) and dminv
 * [B,3,4] (all five channels), each ACCUMULATED into (zero them first) and each may be NULL.  Sample coordinates and in/out
 * decisions are the forward kernel's. */
int rn_resample5_backward_f32(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox, float* dtex,
                              float* dminv, int B, int size, int new_size, void* stream);
/* rn_resample5_backward_f32 for a window (y0, x0, ph, pw; rn_resample_window_f32's rule): gout = dL/d(cropped concat)
 * [B,ph,pw,new_size,5]; only the window's points scatter.  dvox, dtex, dminv as above (accumulated, each may be NULL). */
int rn_resample5_backward_window_f32(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox,
                                     float* dtex, float* dminv, int B, int size, int new_size, int y0, int x0, int ph, int pw,
                                     void* stream);
/* fp32 PReLU derivative (texture decoder, tools/layer_util.py:27-45): out[i] = g[i] * (z[i] > 0 ? 1 : alpha[i % C]) with z the
 * PRE-activation (slopes may be negative). */
int rn_prelu_backward_f32(const float* g, const float* z, const float* alpha, float* out, long long n, int C, void* stream);
/* Data gradient of rn_fully_connected (tools/layer_util.py:311-343): dx[b][k] = sum_n g[b][n] w[k][n], g fp32 [B,N], w fp32 TF
 * layout [K,N] (16-byte aligned, N % 4 == 0), B <= 32.  Split over N with a fixed-order second stage (no float atomics: the
 * result is reproducible bit for bit); `work` holds rn_fully_connected_backward_workspace(B, K, N) floats. */
/* Face reconstruction objective (Reconstruct_RenderNet_Face.py:372-383) over TensorFlow's Phong composite
 * (tools/Phong_shading.py:24-113, tf_phong_composite; not the NumPy composite rn_phong_composite implements): shade =
 * tf_phong_composite(normal, light_dir, light_col, ambient, k_diffuse, black_background, with_mask), loss[b] += mean_{h,w,c}
 * (target - albedo * shade)^2, and in the same pass d_albedo, d_normal (fp32 [B,H,W,3], overwritten) and d_light_dir [B,3]
 * (ACCUMULATED into: zero it first; may be NULL).  loss (double [B]) is accumulated into as well.  TF-1 gradient conventions:
 * tf.maximum passes where x >= y, clip_by_value where lo <= x <= hi, d|x|/dx = x/|x|.  At normal = (0.5, 0.5, 0.5) the pixel
 * is shaded as unlit, only the mask term reaches d_normal and nothing reaches d_light; where |normal| = 0 the mask term is 0, so
 * every output is finite for normal maps in [0, 1].  light_dir, light_col [B,3]. */
int rn_phong_recon_loss_grad(const float* albedo, const float* normal, const float* target, const float* light_dir,
                             const float* light_col, float ambient, float k_diffuse, int black_background, int with_mask,
                             double* loss, float* d_albedo, float* d_normal, float* d_light_dir, int B, int H, int W,
                             void* stream);
/* Shader pose / light fit objective over the demo's NumPy composite (RenderNet_demo.py:54-58, tools/Phong_shading.py:138-228):
 * out = rn_phong_composite(img, light_dir, light_col, ambient, k_diffuse, background_white, with_mask) -- the same device function
 * (rn_phong.cuh phong_pixel), so the image the loss measures is the one rn_phong_composite and the fused epilogue render, bit for
 * bit -- loss[b] += mean_{h,w,c} (target - out)^2 (double [B], ACCUMULATED into), and in the same pass d_img (fp32 [B,H,W,3],
 * overwritten) and d_light_dir [B,3] (ACCUMULATED into: zero it first; may be NULL; the light direction need not be unit: the
 * gradient runs through l / |l|).  img, target [B,H,W,3]; light_dir, light_col [B,3].  The gradient covers n = (img - 0.5) /
 * |img - 0.5|, l / |l| and the soft mask (sigmoid(255 |img| - 150) black, sigmoid(255 |1 - img| - 80) white), whose derivative is
 * evaluated in double from the fp32 pixel.  Conventions as rn_phong_recon_loss_grad: max(x, 0) passes where x >= 0, a clip where
 * lo <= x <= hi.  At img = (0.5, 0.5, 0.5) the normal is 0/0: the forward shades the pixel as unlit (as rn_phong_composite does),
 * and the gradient there is the mask term alone (nothing through the normal, nothing to d_light_dir); at |img| = 0 (black) or
 * |1 - img| = 0 (white) the mask term is 0. */
int rn_phong_composite_loss_grad(const float* img, const float* target, const float* light_dir, const float* light_col,
                                 float ambient, float k_diffuse, int background_white, int with_mask, double* loss, float* d_img,
                                 float* d_light_dir, int B, int H, int W, void* stream);
/* Backward of rn_phong_shade for any loss: g_compos = dL/d(compos) [B,H,W,3] fp32 -> d_normal [B,H,W,3] (overwritten), d_albedo
 * [B,H,W,3] = g_compos * shade (overwritten; written only when albedo is given, and may be NULL) and d_light_dir [B,3]
 * (ACCUMULATED into: zero it first; may be NULL).  The other arguments are rn_phong_shade's, and each composite is differentiated
 * through its own forward device function, recomputed in the same thread: RN_PHONG_TF through tf_phong_pixel (the light
 * normalised by a division by |l|), RN_PHONG_NUMPY through phong_pixel (a multiply by 1 / |l|).  Albedo NULL: compos = shade.
 * Conventions of the fused objectives rn_phong_recon_loss_grad / rn_phong_composite_loss_grad: max(x, 0) passes where x >= 0, a
 * clip where lo <= x <= hi, the mask's derivative in double from the fp32 pixel.  At normal = (0.5, 0.5, 0.5) the direction is
 * 0/0: the forward shades the pixel as unlit, only the mask term reaches d_normal and nothing reaches d_light_dir (finite for
 * both composites).  One thread per pixel, blockIdx.y = item; d_light_dir takes one atomic per block and component. */
int rn_phong_shade_backward(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                            float ambient, float k_diffuse, int composite, int background_white, int with_mask,
                            const float* g_compos, float* d_normal, float* d_albedo, float* d_light_dir, int B, int H, int W,
                            void* stream);
/* Gradients of the shading parameters.  Each *_params entry is the entry above it with ambient read per item from a device array
 * [B] (as rn_phong_shade_ambient) and two more outputs, each ACCUMULATED into (zero them first) and each may be NULL:
 * d_light_col [B,3] and d_ambient [B].  Per pixel, with dx_c the upstream gradient passed through the outer clip(x, 0, 1) and
 * dpre_c the one passed on through the diffuse clip (times the mask m, 1 without a mask):
 *   d_ambient += sum_c m dx_c,   d_light_col_c += dpre_c fl(k_diffuse max(d, 0)),
 * summed over the item's pixels, one atomic per block and component.  k_diffuse has no gradient: the composites see only the
 * product k_diffuse col, which the fitted colour absorbs.  Every other output is the scalar entry's bit for bit when the ambient
 * array holds the scalar. */
int rn_phong_recon_loss_grad_params(const float* albedo, const float* normal, const float* target, const float* light_dir,
                                    const float* light_col, const float* ambient, float k_diffuse, int black_background,
                                    int with_mask, double* loss, float* d_albedo, float* d_normal, float* d_light_dir,
                                    float* d_light_col, float* d_ambient, int B, int H, int W, void* stream);
int rn_phong_composite_loss_grad_params(const float* img, const float* target, const float* light_dir, const float* light_col,
                                        const float* ambient, float k_diffuse, int background_white, int with_mask, double* loss,
                                        float* d_img, float* d_light_dir, float* d_light_col, float* d_ambient, int B, int H,
                                        int W, void* stream);
int rn_phong_shade_backward_params(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                                   const float* ambient, float k_diffuse, int composite, int background_white, int with_mask,
                                   const float* g_compos, float* d_normal, float* d_albedo, float* d_light_dir,
                                   float* d_light_col, float* d_ambient, int B, int H, int W, void* stream);
long long rn_fully_connected_backward_workspace(int B, int K, int N);
int rn_fully_connected_backward_data(const float* g, const float* w, float* work, float* dx, int B, int K, int N, void* stream);

/* ---- face-reconstruction shape decoder (Reconstruct_RenderNet_Face.py:31-75, decoder_3d_pretrained) --------------------------
 * fp32 conv3d / conv3d_transpose with a cubic k = 4 kernel, TF SAME, any channel count up to 512, B <= 32, x [B,H,W,D,Cin] and
 * out channel-last, out = act(conv + bias) with act RN_ACT_NONE / RN_ACT_ELU / RN_ACT_SIGMOID (bias may be NULL).  Replaces
 * the reference's conv3d_transpose k4 s2 + tf.nn.elu (g_conv1..4, :47-69) and conv3d_transpose k4 s1 + tf.nn.sigmoid (g_conv5,
 * :71-74).  transposed = 1: filter [4,4,4,Cout,Cin], out [B,sH,sW,sD,Cout]; transposed = 0: tf.nn.conv3d, filter [4,4,4,Cin,Cout],
 * out [B,ceil(H/s),...,Cout] -- which is also the data gradient of the transposed conv on the same filter array (TF defines
 * conv3d_transpose as conv3d's input gradient).  Implicit GEMM on the CUDA cores; a stride-2 transposed conv runs as its 8 output
 * phases.  Small-M shapes split K; `work` must then hold rn_conv3d_f32_workspace(...) floats (0 = no workspace needed, may be
 * NULL).  No float atomics: the result is reproducible bit for bit.  rc -2: unsupported geometry. */
long long rn_conv3d_f32_workspace(int B, int H, int W, int D, int Cin, int Cout, int stride, int transposed);
int rn_conv3d_f32(const float* x, const float* w, const float* bias, float* out, float* work, int B, int H, int W, int D, int Cin,
                  int Cout, int k, int stride, int transposed, int act, void* stream);
/* fp32 activation derivative from the activation's OUTPUT y (n elements): act RN_ACT_ELU -> TF-1 EluGrad, y < 0 ? g * (y + 1) : g;
 * RN_ACT_SIGMOID -> SigmoidGrad, g * y * (1 - y) (rn_sigmoid_backward writes 16-bit only). */
int rn_act_backward_f32(const float* g, const float* y, float* out, long long n, int act, void* stream);
/* Weight and bias gradients of rn_conv3d_f32's layers, for fine-tuning the shape decoder (decoder_3d_pretrained(trainable=True),
 * :31-75, whose conv3d_transpose layers pass `trainable` to their variables; replaces the filter and bias gradients that
 * tf.gradients computes for them).  x fp32 [B,H,W,D,Cin] (the layer's input), gz = dL/d(pre-activation) fp32 [B,Ho,Wo,Do,Cout]
 * (the layer's output grid: Ho = sH transposed, ceil(H/s) forward; anything else rc -2) ->
 *   transposed = 1:  dw[kidx][co][ci] = sum over b and output voxels o of gz[b,o,co] x[b, i(o, k), ci]   [4,4,4,Cout,Cin]
 *   transposed = 0:  dw[kidx][ci][co], the same sums                                                         [4,4,4,Cin,Cout]
 *   db[co] = sum over b, o of gz[b,o,co]
 * (SAME padding: taps that fall outside the input grid contribute zero), both overwritten.  The geometry rn_conv3d_f32 accepts:
 * k = 4, B <= 32, 1..512 channels (rc -1 / -2).  A stride-2 transposed conv runs as its 8 output phases, each a GEMM over the
 * phase's voxels (M = 8 taps x Cin, N = Cout) writing its own 8 taps of dw; K is split over CTAs.  Transposed stride 1 with
 * Cin = 16, Cout = 1 (g_conv5) and a grid divisible by 4 x 4 x 16 runs a direct kernel.  `work` must hold
 * rn_conv3d_f32_weight_grad_workspace(...) floats (always > 0; NULL: rc -4): the K slices' partial sums, added in a fixed order
 * by a second kernel, which also sums db.  No float atomics: reproducible bit for bit. */
long long rn_conv3d_f32_weight_grad_workspace(int B, int H, int W, int D, int Cin, int Cout, int stride, int transposed);
int rn_conv3d_f32_weight_grad(const float* x, const float* gz, float* dw, float* db, float* work, int B, int H, int W, int D,
                              int Cin, int Ho, int Wo, int Do, int Cout, int k, int stride, int transposed, void* stream);

/* ---- backward pass, stage 2: weight gradients (training step, RenderNet_Shader.py:159-167) -------------------------------
 * dW of a stride-1 SAME conv2d (slim.conv2d / layer_util.conv2d, tools/layer_util.py:147-184) on the tensor cores:
 *   dw[ky][kx][ci][co] = sum_{b,y,x} x[b, y+ky-pb, x+kx-pb, ci] * g[b, y, x, co]        (TF filter layout, fp32)
 * x 16-bit [B,H,W,Cin] (the layer's input), g 16-bit [B,H,W,Cout] (dL/d conv output); both are read as MN-major wgmma
 * operands directly from their channel-last layout (K = pixels).  Cin % 128 == 0, Cout % 128 == 0, kh*kw <= 16,
 * fmt RN_FMT_F16 or RN_FMT_F16X2.  dw is overwritten. */
int rn_conv2d_weight_grad(const void* x, const void* g, float* dw, int B, int H, int W, int Cin, int Cout, int kh, int kw,
                          int fmt, void* stream);
/* db[c] = sum over the npix pixels of g[p][c] (bias gradient of any conv); g 16-bit [npix, C], db fp32 [C], overwritten. */
int rn_bias_grad_16(const void* g, float* db, long long npix, int C, int fmt, void* stream);

/* ---- training step (RenderNet_Shader.py:154-167): remaining weight gradients, PReLU slopes, dropout, loss, Adam -----------
 * Weight gradient of ANY convolution / transposed convolution (2-D: D = kd = 1; 3-D; any stride; TF SAME) as a strided
 * correlation on the CUDA cores, fp32 accumulation (atomics):
 *   dW[tap = (kz*kh + ky)*kw + kx][a][b] = scale * sum_{n,z,y,x} P[n,z,y,x,a] * Q[n, z*sd+kz-pd, y*sh+ky-ph, x*sw+kx-pw, b]
 * (terms whose Q index falls outside the grid are zero padding).  Forward conv (layer_util.conv3d tools/layer_util.py:228-265,
 * slim.conv2d): P = dL/d(conv output), Q = the layer's input, (pd,ph,pw) = TF SAME pad-before -> dW[tap][co][ci].  Transposed
 * conv (slim.conv2d_transpose, RenderNet_Shader.py:106-129; o = i*s + k - pb): P = the layer's input, Q = dL/d(output)
 * -> dW[tap][ci][co].  P is [B,Dp,Hp,Wp,Cap] with Ca <= Cap channels used, Q [B,Dq,Hq,Wq,Cbp]; fmtP / fmtQ: RN_FMT_F16,
 * RN_FMT_BF16, RN_FMT_F16X2 or 3 = fp32.  dW fp32, overwritten.  (Ca,Cb) = (8,1), (16,3), (4,4), (4,8), (8,5) -- e_conv1 and
 * e_conv11 of the Shader; e_tex_conv0, e_tex_conv1 / e_tex_conv2 (fp32 P and Q, RenderNet_Texture_Face_Normal.py:39-44) and
 * e_conv1 (:51-52) of the Texture+Normal network -- run a thin kernel with the whole Ca x Cb block per thread. */
int rn_conv_weight_grad_direct(const void* P, const void* Q, float* dW, int B, int Dp, int Hp, int Wp, int Ca, int Cap, int Dq,
                               int Hq, int Wq, int Cb, int Cbp, int kd, int kh, int kw, int sd, int sh, int sw, int pd, int ph,
                               int pw, int fmtP, int fmtQ, float scale, void* stream);
/* PReLU slope gradient (tools/layer_util.py:27-45: y = max(0,z) + alpha*min(0,z)): dalpha[c] = scale * sum_{z<0} g*z over the
 * n elements (channel-last, n % C == 0) of g = dL/dy and the PRE-activation z, both 16-bit in `fmt`; dalpha fp32 [C], overwritten. */
int rn_prelu_alpha_grad(const void* g, const void* z, float* dalpha, long long n, int C, int fmt, float scale, void* stream);
/* Parameter gradient of the Texture+Normal network's FC + PReLU (e_tex_fc1, RenderNet_Texture_Face_Normal.py:37-38:
 * y = prelu(x W + b; alpha), tools/layer_util.py:27-45,311-343) in one pass: x fp32 [B,K] (the texture vectors), gy = dL/dy,
 * z = x W + b (pre-activation), both fp32 [B,N], alpha [N] ->
 *   gz[b][n] = gy * (z > 0 ? 1 : alpha[n])          (may be NULL: not written)
 *   dw[k][n] = sum_b x[b][k] gz[b][n]               (TF layout [K,N])
 *   db[n]    = sum_b gz[b][n],   dalpha[n] = sum_{b: z<0} gy[b][n] z[b][n]
 * all overwritten.  B <= 32 (rc -2), N % 4 == 0 and 16-byte aligned rows (rc -3).  Sums over b in a fixed order, no atomics:
 * reproducible bit for bit.  z == alpha == dalpha == NULL: an FC without activation (the shape decoder's g_gc1 = fully_connected
 * with no activation, Reconstruct_RenderNet_Face.py:47-50), gz = gy: dw = x^T gy, db = sum_b gy; only some of the three NULL:
 * rc -1. */
int rn_fully_connected_param_grad(const float* x, const float* gy, const float* z, const float* alpha, float* gz, float* dw,
                                  float* db, float* dalpha, int B, int K, int N, void* stream);
/* fp32 PReLU derivative with the bias and slope gradients of a thin texture-decoder conv (e_tex_conv0..2,
 * RenderNet_Texture_Face_Normal.py:39-44, conv3d(_transpose) + bias + prelu): gy = dL/dy, z = pre-activation, channel-last
 * fp32 [n], C = 4 or 8 (rc -2), 16-byte aligned -> gz = gy * (z > 0 ? 1 : alpha[c]) [n], db[c] = sum gz, dalpha[c] =
 * sum_{z<0} gy * z, all overwritten.  Register partials, one fp32 atomic per CTA and channel (db / dalpha: summation order
 * varies between runs; gz is exact). */
int rn_prelu_grad_f32(const float* gy, const float* z, const float* alpha, float* gz, float* db, float* dalpha, long long n, int C,
                      void* stream);
/* tf.nn.dropout (RenderNet_Shader.py:39...123): out[i] = x[i] / keep where hash(seed, salt, i) < keep * 2^32, else 0 (16-bit in
 * `fmt`, out may alias x).  Stateless: the same call on the gradient is the backward pass; rn_dropout_mask_host reproduces the
 * mask on the host (1 = kept).  salt = index of the dropout call within the step. */
int rn_dropout_16(const void* x, void* out, long long n, float keep, unsigned seed, unsigned salt, int fmt, void* stream);
int rn_dropout_mask_host(unsigned char* mask, long long n, float keep, unsigned seed, unsigned salt);
/* Reconstruction loss and its gradient w.r.t. the image (RenderNet_Shader.py:158-163): kind 0 = tf.losses.mean_squared_error
 * (mean over all n elements), kind 1 = binary cross entropy summed per image and averaged over the batch, 1e-6 inside the logs.
 * img / target / dimg fp32 [n] (dimg may be NULL), *loss (device double) is overwritten. */
int rn_image_loss_grad(const float* img, const float* target, float* dimg, double* loss, long long n, int batch, int kind,
                       void* stream);
/* The same losses per item, for a search over several hypotheses (Reconstruct_RenderNet_Face.py:522-534): img / target / dimg fp32
 * [batch, npix, C] (C = 1 or 3), loss double [batch] (overwritten).  kind 0: loss[b] = mean over the item's npix * C elements of
 * (img - target)^2; kind 1: loss[b] = -sum over them of t log(1e-6 + p) + (1 - t) log(1e-6 + 1 - p).  dimg (may be NULL) =
 * d sum_b loss[b] / dimg, overwritten: batch x rn_image_loss_grad's gradient. */
int rn_image_loss_grad_items(const float* img, const float* target, float* dimg, double* loss, long long npix, int C, int batch,
                             int kind, void* stream);
/* One tf.train.AdamOptimizer update of a flat fp32 parameter (RenderNet_Shader.py:167, beta1 = 0.5): m += (g-m)(1-beta1),
 * v += (g^2-v)(1-beta2), param -= lr_t * m / (sqrt(v) + eps), with lr_t = lr * sqrt(1-beta2^t) / (1-beta1^t) passed by the caller. */
int rn_adam_step(float* param, const float* grad, float* m, float* v, long long n, float lr_t, float beta1, float beta2, float eps,
                 void* stream);
/* Shape fit through the Shader network (rendernet_b200/shape_fit.py): the gradient of
 *   L(occ) = sum_v loss_v + lambda_smooth R_s + lambda_bin R_b,
 *   R_s = (1/N) sum over axis-neighbour pairs (i, j) inside the grid (no wrap-around) of (occ_i - occ_j)^2,
 *   R_b = (1/N) sum_i occ_i (1 - occ_i),   N = S^3,
 * w.r.t. one occupancy grid that every view renders.  dvox fp32 [V, S^3]: the per-view dL/dvoxels rn_resample_backward_f32
 * writes; occ fp32 [S^3]; keep uint8 [S^3] or NULL (1 = voxel not carved away).  g fp32 [S^3], overwritten:
 *   g[i] = keep[i] ? sum_v dvox[v][i] + lambda_smooth dR_s/docc_i + lambda_bin dR_b/docc_i : 0
 * (the view sum in double, v = 0..V-1).  reg double [2] = (R_s, R_b), overwritten; both are taken over the whole grid, carved
 * voxels included.  work: rn_voxel_fit_grad_workspace(S) doubles.  The reduction has a fixed order (block partials, then one
 * block; the block count depends on S alone): two launches are bit-identical.  lambda_* >= 0 and finite, else rc -1. */
long long rn_voxel_fit_grad_workspace(int S);
int rn_voxel_fit_grad(const float* dvox, const float* occ, const unsigned char* keep, float* g, double* reg, double* work, int V,
                      int S, float lambda_smooth, float lambda_bin, void* stream);

/* ---- fixed-order twins (what rendernet_b200.ops calls under torch.use_deterministic_algorithms) ------------------------------
 * Twins of the input-gradient kernels that reduce with float atomics.  Each result is a function of its own item's inputs alone:
 * bit-identical from run to run, and for an item whatever batch it is part of.  Each takes a caller-owned workspace of at least
 * the matching *_workspace(...) bytes (rc -4 if smaller), allocates nothing and does not synchronise (a CUDA graph may capture
 * it).  Unlike the atomic kernels, every output is OVERWRITTEN: nothing needs zeroing.  Per-pixel outputs are the atomic
 * kernels' bit for bit; only the reductions differ.
 *   rn_resample_backward_fixed_f32 / rn_resample5_backward_fixed_f32 (whole grid): dvox / dtex are summed in 64-bit fixed point
 *   (per item and channel of gout a power of two 2^k with new_size^3 max|gout| 2^k < 2^62, so no sum can overflow; each fp32
 *   corner contribution w g is scaled by 2^k in double and rounded once to an integer, then added with an integer atomic), dminv
 *   from per-block partial sums added in block order.  An item whose gout holds an Inf or NaN gets NaN in all its outputs.
 *   rn_fixed_point_exponent(max_abs, new_size) is the k the resampler twins use (0 for max_abs 0 or non-finite).
 *   Phong objectives and rn_image_loss_grad_items_fixed: loss and d_light from per-block partials added in block order in double;
 *   the image loss uses a block count per item that does not depend on the batch. */
int rn_fixed_point_exponent(float max_abs, int new_size);
long long rn_resample_backward_fixed_workspace(int B, int C, int size, int new_size, int want_dvox);
int rn_resample_backward_fixed_f32(const float* vox, const float* minv, const float* gout, float* dvox, float* dminv, int B, int C,
                                   int size, int new_size, int transform, void* work, long long work_bytes, void* stream);
long long rn_resample5_backward_fixed_workspace(int B, int size, int new_size, int want_dvox, int want_dtex);
int rn_resample5_backward_fixed_f32(const float* vox, const float* tex, const float* minv, const float* gout, float* dvox,
                                    float* dtex, float* dminv, int B, int size, int new_size, void* work, long long work_bytes,
                                    void* stream);
long long rn_phong_recon_loss_grad_fixed_workspace(int B, int H, int W);
int rn_phong_recon_loss_grad_fixed(const float* albedo, const float* normal, const float* target, const float* light_dir,
                                   const float* light_col, float ambient, float k_diffuse, int black_background, int with_mask,
                                   double* loss, float* d_albedo, float* d_normal, float* d_light_dir, int B, int H, int W,
                                   void* work, long long work_bytes, void* stream);
long long rn_phong_composite_loss_grad_fixed_workspace(int B, int H, int W);
int rn_phong_composite_loss_grad_fixed(const float* img, const float* target, const float* light_dir, const float* light_col,
                                       float ambient, float k_diffuse, int background_white, int with_mask, double* loss,
                                       float* d_img, float* d_light_dir, int B, int H, int W, void* work, long long work_bytes,
                                       void* stream);
/* work may be NULL when d_light_dir is NULL */
long long rn_phong_shade_backward_fixed_workspace(int B, int H, int W);
int rn_phong_shade_backward_fixed(const float* normal, const float* albedo, const float* light_dir, const float* light_col,
                                  float ambient, float k_diffuse, int composite, int background_white, int with_mask,
                                  const float* g_compos, float* d_normal, float* d_albedo, float* d_light_dir, int B, int H, int W,
                                  void* work, long long work_bytes, void* stream);
/* twins of the *_params entries: d_light_col and d_ambient from per-block partials added in block order, like d_light_dir.
 * rn_phong_shade_backward_params_fixed needs no work when d_light_dir, d_light_col and d_ambient are all NULL. */
long long rn_phong_recon_loss_grad_params_fixed_workspace(int B, int H, int W);
int rn_phong_recon_loss_grad_params_fixed(const float* albedo, const float* normal, const float* target, const float* light_dir,
                                          const float* light_col, const float* ambient, float k_diffuse, int black_background,
                                          int with_mask, double* loss, float* d_albedo, float* d_normal, float* d_light_dir,
                                          float* d_light_col, float* d_ambient, int B, int H, int W, void* work,
                                          long long work_bytes, void* stream);
long long rn_phong_composite_loss_grad_params_fixed_workspace(int B, int H, int W);
int rn_phong_composite_loss_grad_params_fixed(const float* img, const float* target, const float* light_dir,
                                              const float* light_col, const float* ambient, float k_diffuse, int background_white,
                                              int with_mask, double* loss, float* d_img, float* d_light_dir, float* d_light_col,
                                              float* d_ambient, int B, int H, int W, void* work, long long work_bytes,
                                              void* stream);
long long rn_phong_shade_backward_params_fixed_workspace(int B, int H, int W);
int rn_phong_shade_backward_params_fixed(const float* normal, const float* albedo, const float* light_dir,
                                         const float* light_col, const float* ambient, float k_diffuse, int composite,
                                         int background_white, int with_mask, const float* g_compos, float* d_normal,
                                         float* d_albedo, float* d_light_dir, float* d_light_col, float* d_ambient, int B, int H,
                                         int W, void* work, long long work_bytes, void* stream);
long long rn_image_loss_grad_items_fixed_workspace(long long npix, int C, int batch);
int rn_image_loss_grad_items_fixed(const float* img, const float* target, float* dimg, double* loss, long long npix, int C,
                                   int batch, int kind, void* work, long long work_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RENDERNET_B200_H_ */
