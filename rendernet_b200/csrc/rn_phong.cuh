// rn_phong.cuh -- one pixel of the demo's Phong composite (tools/Phong_shading.py:138-228 np_mask / np_phong_shading /
// np_phong_composite, RenderNet_demo.py:54-58), shared by the stand-alone kernel (rn_ops.cu), the fused epilogue of the
// last up-conv (rn_igemm_kernel.cuh) and the Shader fit's loss kernel (rn_backward.cu) so that all three produce the same bits;
// and one pixel of TensorFlow's composite
// (tf_phong_pixel), which the stand-alone kernel renders for face reconstruction.
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

// TensorFlow's composite (tools/Phong_shading.py:24-113 tf_mask / tf_mask_white / tf_phong_shading / tf_phong_composite), the
// shading Reconstruct_RenderNet_Face.py:372-378 multiplies the albedo by.  (n0,n1,n2) = normal map in [0,1]; L = the light
// direction ALREADY normalised as l / |l| (division, not a reciprocal); col = light colour.  The operation order, the fp32
// rounding points and the mask in double are those of the forward half of phong_recon_loss_grad_kernel (rn_backward.cu), so the
// image this returns is the one the reconstruction loss measures, bit for bit.  Unlike phong_pixel: the normal is not clamped
// away from |n - 0.5| = 0, the white mask is sigmoid(255 (sqrt 3 - |n|) - 80) and the black one sigmoid(255 |n| - 80).
__device__ __forceinline__ void tf_phong_pixel(float n0, float n1, float n2, const float* L, const float* col, float ambient,
                                               float k_diffuse, int black, int with_mask, float* out) {
  const float v[3] = {n0 - 0.5f, n1 - 0.5f, n2 - 0.5f};
  const float vn = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const float u[3] = {v[0] / vn, v[1] / vn, v[2] / vn};
  const float d = u[0] * L[0] + u[1] * L[1] + u[2] * L[2];
  const float dmax = fmaxf(d, 0.f);
  float m = 1.f;
  if (with_mask) {
    const double nnd = sqrt(static_cast<double>(n0) * n0 + static_cast<double>(n1) * n1 + static_cast<double>(n2) * n2);
    const double s = black ? 255.0 * nnd - 80.0 : 255.0 * (1.7320508075688772 - nnd) - 80.0;
    m = static_cast<float>(1.0 / (1.0 + exp(-s)));
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float pre = k_diffuse * dmax * col[c];
    const float dif = fminf(fmaxf(pre, 0.f), 1.f);
    const float x = with_mask ? m * (ambient + dif) + (1.f - m) : ambient + dif;
    out[c] = fminf(fmaxf(x, 0.f), 1.f);
  }
}

}  // namespace rn
