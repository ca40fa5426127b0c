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
 *     significant bits.  In that mode every convolution evaluates x_hi.w_hi + x_lo.w_hi + x_hi.w_lo on the tensor cores
 *     (3x the MMAs) and matches the reference's fp32 convolutions (tools/layer_util.py:171,212,253) to ~1e-6 relative;
 *     packed filters, 16-bit activations, residuals and outputs are all such pairs (buffers twice the size).
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
  const float* bias;        /* fp32 [cout_pad] */
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
   * of 8).  The reference-shaped wrappers below derive them from the tensor shapes ([2][numel] pairs). */
  long long x_plane, w_plane, o_plane;
  /* accepted and ignored (kept so that the struct layout stays stable): the sm_90 kernel has a single epilogue form, two
   * consumer warpgroups storing their own rows directly */
  int epi_groups, res_prefetch, tma_store;
  const rn_phong* phong;    /* NULL, or the fused Phong epilogue (act = RN_ACT_SIGMOID, N = F pixels x 3 channels <= 16) */
} rn_conv_desc;
int rn_conv_igemm(const rn_conv_desc* d, void* stream);
/* Per-call overrides of the launch heuristics for the reference-shaped wrappers below (their last argument before
 * `stream`; NULL = library defaults).  0 = default for every field; cluster 1/2/4; cta_group 1; kps = k-groups per
 * pipeline stage; msub 1/2 M sub-tiles; yhalo: 1 = on, -1 = off; epilogue_groups / res_prefetch / tma_store are ignored.
 * Every combination computes bit-identical results (tests/test_gpu_kernels.py::*_bit_identical). */
typedef struct rn_tuning {
  int cluster, cta_group, kps, msub, epilogue_groups, res_prefetch, tma_store, yhalo;
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

/* slim.conv2d_transpose / layer_util.conv2d_transpose (layer_util.py:186; RenderNet_Shader.py:106-129),
 * SAME, out = in*stride.  w_packed holds the stride^2 phase filters back to back, as produced by
 * rn_pack_conv2d_transpose_weights: [phase = ay*s+ax][taps_of_phase][cout_pad][Cin]. */
int rn_pack_conv2d_transpose_weights(const float* w, void* packed, int kh, int kw, int Cin, int Cout,
                                     int cout_pad, int stride, int fmt, void* stream);
int rn_conv2d_transpose_same(const void* x, const void* w_packed, const float* bias, const float* alpha, int act,
                             void* out16, float* out32, int B, int H, int W, int Cin, int Cout, int cout_pad,
                             int kh, int kw, int stride, int fmt, const rn_tuning* tune, void* stream);

/* Stride-2, k = 4 SAME transposed conv (e_conv7/8/9, RenderNet_Shader.py:106-119) as ONE launch: rows = input pixels,
 * N = (ay, ax, co) = 4*Cout, 9 taps (dy,dx in {-1,0,1}) with the unused phase/tap combinations zero in the packed
 * filter [9][4*Cout][Cin]; each thread writes two full 2*Cout-element runs of the 2x2 output block.  bias4 / alpha4:
 * per-Cout vectors tiled 4 times.  (The 4-launch phase form is rn_conv2d_transpose_same.) */
int rn_pack_conv2d_transpose_s2_merged(const float* w, void* packed, int Cin, int Cout, int fmt, void* stream);
int rn_conv2d_transpose_s2_merged(const void* x, const void* w_merged, const float* bias4, const float* alpha4, int act,
                                  void* out16, float* out32, int B, int H, int W, int Cin, int Cout, int fmt,
                                  const rn_tuning* tune, void* stream);

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

/* The same fusion for the Texture/Normal network's input (BASELINE config 4; RenderNet_Texture_Face_Normal.py:155-179):
 * tf_rotation_resampling of the geometry grid (vox fp32 [B,size^3], C = 1) AND of the decoded texture volume (tex fp32
 * [B,size^3,4], 16-byte aligned) with the same pose + axis transform + tf.concat(axis=4) (:178) + e_conv1 5^3 stride 2,
 * 5 -> 8 (w fp32 [5,5,5,5,8]) + bias + PReLU, one kernel; bit-identical to rn_resample_f32 x2 -> rn_concat_channels_f32 ->
 * rn_conv3d_direct. */
int rn_resample5_conv1_fused(const float* vox, const float* tex, const float* minv, const float* w, const float* bias,
                             const float* alpha, void* out16, int B, int size, int new_size, int fmt, void* stream);

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
 * tf.maximum passes where x >= y, clip_by_value where lo <= x <= hi, d|x|/dx = x/|x|.  light_dir, light_col [B,3]. */
int rn_phong_recon_loss_grad(const float* albedo, const float* normal, const float* target, const float* light_dir,
                             const float* light_col, float ambient, float k_diffuse, int black_background, int with_mask,
                             double* loss, float* d_albedo, float* d_normal, float* d_light_dir, int B, int H, int W,
                             void* stream);
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
 * reproducible bit for bit. */
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
/* One tf.train.AdamOptimizer update of a flat fp32 parameter (RenderNet_Shader.py:167, beta1 = 0.5): m += (g-m)(1-beta1),
 * v += (g^2-v)(1-beta2), param -= lr_t * m / (sqrt(v) + eps), with lr_t = lr * sqrt(1-beta2^t) / (1-beta1^t) passed by the caller. */
int rn_adam_step(float* param, const float* grad, float* m, float* v, long long n, float lr_t, float beta1, float beta2, float eps,
                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RENDERNET_B200_H_ */
