// rn_phong.cuh -- one pixel of the demo's Phong composite (tools/Phong_shading.py:138-228 np_mask / np_phong_shading /
// np_phong_composite, RenderNet_demo.py:54-58), shared by the stand-alone kernel (rn_ops.cu), the fused epilogue of the
// last up-conv (rn_igemm_kernel.cuh) and the Shader fit's loss kernel (rn_backward.cu) so that all three produce the same bits;
// and one pixel of TensorFlow's composite
// (tf_phong_pixel), which the stand-alone kernel renders for face reconstruction and the reconstruction loss (rn_backward.cu)
// measures.  Next to each, its backward for an arbitrary upstream gradient (phong_pixel_backward, tf_phong_pixel_backward), which
// rn_phong_shade_backward and, for tf_phong_pixel, the reconstruction loss (rn_backward.cu) run on the terms their own forward
// call recorded.
#pragma once
#include <cstdint>

namespace rn {

// The intermediate values of one phong_pixel call, for its backward (phong_composite_loss_grad_kernel, rn_backward.cu).
struct PhongTerms {
  float L[3];      // the normalised light l / |l|
  float linv;      // 1 / |l|
  float inv;       // 1 / |img - 0.5|
  float d;         // (img - 0.5) . L / |img - 0.5|, before max(., 0)
  float mask;      // the fp32 mask (1 without mask)
  float pre[3];    // k_d max(d, 0) col_c, before the clip to [0, 1]
  float diff[3];   // the clipped diffuse term
  float x[3];      // the composite, before the clip to [0, 1]
};

// (r,g,b) = normal map in [0,1]; l = light direction (not normalised), col = light colour.  Returns the shaded colour and, if
// `t` is not NULL, the intermediates the gradient needs (the same values: recorded, not recomputed).
__device__ __forceinline__ void phong_pixel(float r, float g, float bl, float lx, float ly, float lz, const float* col,
                                            float ambient, float k_diffuse, int white, int with_mask, float* out,
                                            PhongTerms* t = nullptr) {
  // np_phong_shading (:162-200): n = (img-0.5)/|img-0.5| ; diffuse = k_d * max(n.l, 0) * light_col, clipped
  const float nx = r - 0.5f, ny = g - 0.5f, nz = bl - 0.5f;
  const float inv = 1.0f / sqrtf(nx * nx + ny * ny + nz * nz);
  const float linv = 1.0f / sqrtf(lx * lx + ly * ly + lz * lz);
  lx *= linv; ly *= linv; lz *= linv;
  const float d = (nx * lx + ny * ly + nz * lz) * inv;
  const float ndl = fmaxf(d, 0.f);
  float mask = 1.f;
  if (with_mask) {  // np_mask (:138-148) / np_mask_white (:150-160)
    const float nrm = white ? sqrtf((1.f - r) * (1.f - r) + (1.f - g) * (1.f - g) + (1.f - bl) * (1.f - bl))
                            : sqrtf(r * r + g * g + bl * bl);
    mask = 1.f / (1.f + expf(-(255.f * nrm - (white ? 80.f : 150.f))));
  }
  if (t != nullptr) {
    t->L[0] = lx; t->L[1] = ly; t->L[2] = lz;
    t->linv = linv; t->inv = inv; t->d = d; t->mask = mask;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float pre = k_diffuse * ndl * col[c];
    const float diff = fminf(fmaxf(pre, 0.f), 1.f);
    float v = with_mask ? mask * (ambient + diff) + (1.f - mask) : ambient + diff;
    if (t != nullptr) { t->pre[c] = pre; t->diff[c] = diff; t->x[c] = v; }
    out[c] = fminf(fmaxf(v, 0.f), 1.f);
  }
}
__device__ __forceinline__ uint8_t phong_u8(float v) { return static_cast<uint8_t>(fminf(fmaxf(255.f * v, 0.f), 255.f)); }

// Backward of one phong_pixel call for an arbitrary upstream gradient ds = dL/d(out) (rn_phong_shade_backward): di = dL/d(r,g,b)
// and dl = dL/dL, L = l / |l| the normalised light (the caller maps it through (I - L L^T) / |l|).  t: the call's own terms.
// Conventions of phong_composite_loss_grad_kernel: max(x, 0) passes where x >= 0, a clip where lo <= x <= hi; the mask's
// derivative m (1 - m) 255 (+-a / |a|) runs in double from the fp32 pixel.  At img = (0.5, 0.5, 0.5) t.d is NaN, max(d, 0)
// passes nothing, and only the mask term reaches di (dl stays 0); where |a| = 0 the mask term is 0.
__device__ __forceinline__ void phong_pixel_backward(float r, float g, float bl, const PhongTerms& t, const float* col,
                                                     float ambient, float k_diffuse, int white, int with_mask, const float* ds,
                                                     float* di, float* dl) {
  float dndl = 0.f, dm = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float dx = (t.x[c] >= 0.f && t.x[c] <= 1.f) ? ds[c] : 0.f;              // clip(compos, 0, 1)
    if (with_mask) dm += dx * (ambient + t.diff[c] - 1.f);
    const float ddiff = with_mask ? dx * t.mask : dx;
    const float dpre = (t.pre[c] >= 0.f && t.pre[c] <= 1.f) ? ddiff : 0.f;         // clip(diffuse, 0, 1)
    dndl += dpre * k_diffuse * col[c];
  }
  const float dd = t.d >= 0.f ? dndl : 0.f;                                         // max(d, 0); false for a NaN d
#pragma unroll
  for (int i = 0; i < 3; ++i) di[i] = dl[i] = 0.f;
  if (dd != 0.f) {
    const float u[3] = {(r - 0.5f) * t.inv, (g - 0.5f) * t.inv, (bl - 0.5f) * t.inv};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      di[i] = dd * (t.L[i] - t.d * u[i]) * t.inv;
      dl[i] = dd * u[i];
    }
  }
  if (with_mask && dm != 0.f) {
    const double a[3] = {white ? 1.0 - r : static_cast<double>(r), white ? 1.0 - g : static_cast<double>(g),
                         white ? 1.0 - bl : static_cast<double>(bl)};
    const double nrm = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    if (nrm > 0.0) {
      const double md = 1.0 / (1.0 + exp(-(255.0 * nrm - (white ? 80.0 : 150.0))));
      const double dsg = static_cast<double>(dm) * md * (1.0 - md) * (white ? -255.0 : 255.0) / nrm;
#pragma unroll
      for (int i = 0; i < 3; ++i) di[i] += static_cast<float>(dsg * a[i]);
    }
  }
}

// The intermediate values of one tf_phong_pixel call, for its backward (tf_phong_pixel_backward).
struct TfPhongTerms {
  float u[3];      // (n - 0.5) / |n - 0.5|
  float vn;        // |n - 0.5|
  float d;         // u . L, before max(., 0)
  float m;         // the fp32 mask (1 without mask)
  double md, nnd;  // the mask and |n| in double
  float pre[3];    // k_d max(d, 0) col_c, before the clip to [0, 1]
  float dif[3];    // the clipped diffuse term
  float x[3];      // the composite, before the clip to [0, 1]
};

// TensorFlow's composite (tools/Phong_shading.py:24-113 tf_mask / tf_mask_white / tf_phong_shading / tf_phong_composite), the
// shading Reconstruct_RenderNet_Face.py:372-378 multiplies the albedo by.  (n0,n1,n2) = normal map in [0,1]; L = the light
// direction ALREADY normalised as l / |l| (division, not a reciprocal); col = light colour.  phong_recon_loss_grad_kernel
// (rn_backward.cu) shades with this function, so the image it returns is the one the reconstruction loss measures, bit for bit.
// The mask's argument multiplies |n|'s rounding by 255 (and its derivative by another 255), so the mask runs in double.  At
// n = (0.5, 0.5, 0.5) u and d are NaN and fmaxf shades the pixel as unlit.  Unlike phong_pixel: the normal is not clamped
// away from |n - 0.5| = 0, the white mask is sigmoid(255 (sqrt 3 - |n|) - 80) and the black one sigmoid(255 |n| - 80).  If `t` is
// not NULL it receives the intermediates the gradient needs (recorded, not recomputed).
__device__ __forceinline__ void tf_phong_pixel(float n0, float n1, float n2, const float* L, const float* col, float ambient,
                                               float k_diffuse, int black, int with_mask, float* out, TfPhongTerms* t = nullptr) {
  // Every rounding is spelled out (the _rn intrinsics are never contracted or reassociated): left to the compiler, a sum of
  // products is contracted into FMAs in an order that depends on the calling kernel, and the callers would differ in the last bit.
  const float v[3] = {n0 - 0.5f, n1 - 0.5f, n2 - 0.5f};
  const float vn = __fsqrt_rn(__fmaf_rn(v[2], v[2], __fmaf_rn(v[0], v[0], __fmul_rn(v[1], v[1]))));
  const float u[3] = {__fdiv_rn(v[0], vn), __fdiv_rn(v[1], vn), __fdiv_rn(v[2], vn)};
  const float d = __fmaf_rn(u[2], L[2], __fmaf_rn(u[0], L[0], __fmul_rn(u[1], L[1])));
  const float dmax = fmaxf(d, 0.f);
  float m = 1.f;
  double md = 1.0, nnd = 1.0;
  if (with_mask) {
    const double e[3] = {n0, n1, n2};
    nnd = __dsqrt_rn(__fma_rn(e[2], e[2], __fma_rn(e[0], e[0], __dmul_rn(e[1], e[1]))));
    const double s = __fma_rn(black ? nnd : __dsub_rn(1.7320508075688772, nnd), 255.0, -80.0);
    md = __drcp_rn(__dadd_rn(1.0, exp(-s)));
    m = static_cast<float>(md);
  }
  if (t != nullptr) {
    t->u[0] = u[0]; t->u[1] = u[1]; t->u[2] = u[2];
    t->vn = vn; t->d = d; t->m = m; t->md = md; t->nnd = nnd;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float pre = __fmul_rn(__fmul_rn(k_diffuse, dmax), col[c]);
    const float dif = fminf(fmaxf(pre, 0.f), 1.f);
    const float x = with_mask ? __fmaf_rn(m, __fadd_rn(ambient, dif), __fsub_rn(1.f, m)) : __fadd_rn(ambient, dif);
    if (t != nullptr) { t->pre[c] = pre; t->dif[c] = dif; t->x[c] = x; }
    out[c] = fminf(fmaxf(x, 0.f), 1.f);
  }
}

// Backward of one tf_phong_pixel call for an arbitrary upstream gradient ds = dL/d(out) (rn_phong_shade_backward,
// phong_recon_loss_grad_kernel): dn = dL/dn and dl = dL/dL (L already normalised; the caller maps dl through (I - L L^T) / |l|).
// n: the pixel, t: the call's own terms.  TF-1's conventions (max(x, 0) passes where x >= 0, a clip where lo <= x <= hi,
// d|x|/dx = x / |x|), the mask's derivative in double.  The normal's term is skipped where nothing passes max(d, 0): at
// n = (0.5, 0.5, 0.5) u = 0/0 and d are NaN, and dn gets the mask term alone, dl nothing.  At |n| = 0 the mask term is 0.
__device__ __forceinline__ void tf_phong_pixel_backward(const float* n, const float* L, const TfPhongTerms& t, const float* col,
                                                        float ambient, float k_diffuse, int black, int with_mask, const float* ds,
                                                        float* dn, float* dl) {
  float ddmax = 0.f, dm = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float dx = (t.x[c] >= 0.f && t.x[c] <= 1.f) ? ds[c] : 0.f;              // clip_by_value(compos, 0, 1)
    const float ddif = with_mask ? dx * t.m : dx;
    if (with_mask) dm += dx * (ambient + t.dif[c] - 1.f);
    const float dpre = (t.pre[c] >= 0.f && t.pre[c] <= 1.f) ? ddif : 0.f;         // clip_by_value(diffuse, 0, 1)
    ddmax += dpre * k_diffuse * col[c];
  }
  const float dd = t.d >= 0.f ? ddmax : 0.f;                                        // tf.maximum(d, 0); false for a NaN d
#pragma unroll
  for (int i = 0; i < 3; ++i) dn[i] = dl[i] = 0.f;
  if (dd != 0.f) {
    float du[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      du[i] = dd * L[i];
      dl[i] = dd * t.u[i];
    }
    const float udu = t.u[0] * du[0] + t.u[1] * du[1] + t.u[2] * du[2];           // d (v/|v|) = (du - u (u.du)) / |v|
#pragma unroll
    for (int i = 0; i < 3; ++i) dn[i] = (du[i] - t.u[i] * udu) / t.vn;
  }
  if (with_mask && dm != 0.f && t.nnd > 0.0) {                                     // sigmoid, then d|n|/dn = n/|n|
    const double dsg = static_cast<double>(dm) * t.md * (1.0 - t.md) * (black ? 255.0 : -255.0) / t.nnd;
#pragma unroll
    for (int i = 0; i < 3; ++i) dn[i] += static_cast<float>(dsg * n[i]);
  }
}

// Gradients of the shading parameters for one pixel of either composite, from the terms its forward recorded (PhongTerms:
// d, mask; TfPhongTerms: d, m; both: pre, x).  Both composites form x_c = m (ambient + clip(pre_c)) + (1 - m) (x_c = ambient +
// clip(pre_c) without a mask) with pre_c = fl(k_d max(d, 0)) col_c, so with dx_c = ds_c where 0 <= x_c <= 1 and dpre_c = m dx_c
// where 0 <= pre_c <= 1:  dL/d ambient += sum_c m dx_c,  dL/d col_c += dpre_c fl(k_d max(d, 0)).  At a NaN d (n = (0.5, 0.5, 0.5))
// max(d, 0) is 0 and the colour gets nothing.  A helper of its own, so phong_pixel_backward / tf_phong_pixel_backward and the
// kernels that inline them are untouched; dcol[3] and *damb are accumulated into.
__device__ __forceinline__ void phong_param_backward(float d, float m, const float* pre, const float* x, float k_diffuse,
                                                     int with_mask, const float* ds, float* dcol, float* damb) {
  const float kd = k_diffuse * fmaxf(d, 0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float dx = (x[c] >= 0.f && x[c] <= 1.f) ? ds[c] : 0.f;                   // clip(compos, 0, 1)
    const float ddiff = with_mask ? dx * m : dx;
    *damb += ddiff;
    const float dpre = (pre[c] >= 0.f && pre[c] <= 1.f) ? ddiff : 0.f;             // clip(diffuse, 0, 1)
    dcol[c] += dpre * kd;
  }
}

}  // namespace rn
