// Per-element arithmetic of the elevation read-out primitives, shared by the single-plane entry points of tdx_post.cu
// and the batched evaluation read-out of tdx_eval.cu, so both compute every output element with the same explicitly
// rounded operations in the same order (and so agree bit for bit).
#pragma once
#include <math.h>

namespace tdx {

// laplacian_encoder.py:6-40: rows are extrapolated first, then the columns of the row-padded tensor.  ld(r, c) reads
// element (r, c) of the unpadded [h][w] plane.
template <class Load>
__device__ __forceinline__ float row_padded(const Load& ld, int h, int r, int c) {   // r in [-1, h], c in [0, w)
  if (r >= 0 && r < h) return ld(r, c);
  if (h == 1) return ld(0, c);
  if (r < 0) return __fsub_rn(__fmul_rn(2.0f, ld(0, c)), ld(1, c));
  return __fsub_rn(__fmul_rn(2.0f, ld(h - 1, c)), ld(h - 2, c));
}
// Element (oy, ox) of the (h+2) x (w+2) linear-extrapolation padding.
template <class Load>
__device__ __forceinline__ float pad_extrapolate_at(const Load& ld, int h, int w, int oy, int ox) {
  const int r = oy - 1, c = ox - 1;
  if (c >= 0 && c < w) return row_padded(ld, h, r, c);
  if (w == 1) return row_padded(ld, h, r, 0);
  if (c < 0) return __fsub_rn(__fmul_rn(2.0f, row_padded(ld, h, r, 0)), row_padded(ld, h, r, 1));
  return __fsub_rn(__fmul_rn(2.0f, row_padded(ld, h, r, w - 1)), row_padded(ld, h, r, w - 2));
}

// Element (oy, ox) of one axis of torch's interpolate(mode="bilinear", antialias=True) of x [h][w] (ATen
// UpSampleKernel.cpp, _compute_indices_min_size_weights_aa with the triangle filter): weights are normalised first,
// then accumulated in tap order.  axis 1: out[y][i] over rows of x;  axis 0: out[i][x] over columns.
__device__ __forceinline__ float resize_aa_at(const float* __restrict__ x, int h, int w, int out_size, int axis, int oy,
                                              int ox) {
  const int in_size = axis == 1 ? w : h;
  const int i = axis == 1 ? ox : oy;
  const float scale = __fdiv_rn((float)in_size, (float)out_size);
  const float support = scale >= 1.0f ? scale : 1.0f;
  const float invscale = scale >= 1.0f ? __fdiv_rn(1.0f, scale) : 1.0f;
  const float center = __fmul_rn(scale, (float)i + 0.5f);
  int lo = (int)__fadd_rn(__fsub_rn(center, support), 0.5f);
  lo = lo > 0 ? lo : 0;
  int hi = (int)__fadd_rn(__fadd_rn(center, support), 0.5f);
  hi = hi < in_size ? hi : in_size;
  const int n = hi - lo;
  auto weight = [&](int j) {
    float t = __fmul_rn(__fadd_rn(__fsub_rn((float)(j + lo), center), 0.5f), invscale);
    t = t < 0.f ? -t : t;
    return t < 1.0f ? __fsub_rn(1.0f, t) : 0.0f;
  };
  float total = 0.f;
  for (int j = 0; j < n; ++j) total = __fadd_rn(total, weight(j));
  const long stride = axis == 1 ? 1 : w;
  const float* src = axis == 1 ? x + (long)oy * w + lo : x + (long)lo * w + ox;
  float acc = 0.f;
  for (int j = 0; j < n; ++j) {
    float wj = weight(j);
    if (total != 0.f) wj = __fdiv_rn(wj, total);
    const float term = __fmul_rn(src[(long)j * stride], wj);
    acc = j == 0 ? term : __fadd_rn(acc, term);
  }
  return acc;
}

struct BlurParams {
  float k[32];
  int ksize;
};
// torchvision _get_gaussian_kernel1d in float32: taps on linspace(-(k-1)/2, (k-1)/2, k), normalised by their sum.
// ksize odd and <= 31 (callers check).
inline BlurParams gaussian_blur_params(int ksize, float sigma) {
  BlurParams bp;
  bp.ksize = ksize;
  const float half = (ksize - 1) * 0.5f;
  float sum = 0.f;
  for (int i = 0; i < ksize; ++i) {
    const float t = (-half + (float)i) / sigma;
    bp.k[i] = expf(-0.5f * (t * t));
    sum += bp.k[i];
  }
  for (int i = 0; i < ksize; ++i) bp.k[i] /= sum;
  return bp;
}
// Element (oy, ox) of torchvision gaussian_blur: reflect padding ksize/2, 2-D kernel = outer(k, k), taps accumulated
// row-major.
__device__ __forceinline__ float gaussian_blur_at(const float* __restrict__ x, int h, int w, const BlurParams& bp,
                                                  int oy, int ox) {
  const int p = bp.ksize / 2;
  float acc = 0.f;
  for (int dy = 0; dy < bp.ksize; ++dy) {
    int yy = oy + dy - p;
    yy = yy < 0 ? -yy : (yy >= h ? 2 * h - 2 - yy : yy);
    for (int dx = 0; dx < bp.ksize; ++dx) {
      int xx = ox + dx - p;
      xx = xx < 0 ? -xx : (xx >= w ? 2 * w - 2 - xx : xx);
      acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(bp.k[dy], bp.k[dx]), x[(long)yy * w + xx]));
    }
  }
  return acc;
}

// sign(v) * v^2 (world_pipeline.py:1312)
__device__ __forceinline__ float signed_square(float v) { return v == 0.f ? 0.f : copysignf(__fmul_rn(v, v), v); }

// One element of laplacian_decode on a normalised residual: f(r * scale + offset + up), rounded as torch rounds
// `residual * std + mean` (a multiply, then an add) followed by tdx_post_combine's add; f = sign(v) v^2 with signed_sq,
// else the identity.
__device__ __forceinline__ float denorm_combine(float r, float scale, float offset, float up, int signed_sq) {
  const float v = __fadd_rn(__fadd_rn(__fmul_rn(r, scale), offset), up);
  return signed_sq ? signed_square(v) : v;
}

}  // namespace tdx
