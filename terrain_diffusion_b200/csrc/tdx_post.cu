// Elevation read-out ("post step", SURVEY.md section 8(f) rank 3): the reference does this on the CPU with torchvision
// on every WorldPipeline.get() (world_pipeline.py:1277-1313, data/laplacian_encoder.py:6-137).  Here each primitive is
// one small fp32 kernel, thread per output element, so the read-out stays on the device next to the canvases:
//   normalise-on-read, linear-extrapolation padding, torch's anti-aliased separable bilinear resize (one axis per
//   launch), torchvision's reflect-padded Gaussian blur, and add + crop + signed square (+ int16 pack, api.py:73-77).
// All arithmetic is written with explicitly rounded operations in the order of the CPU restatement (oracle/postproc.py,
// pinned against the reference), so results agree to float32 round-off.  HBM-bound and tiny (a few hundred KB per call).
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

__global__ void post_normalize_kernel(const float* __restrict__ num, const float* __restrict__ den, long pitch,
                                      float* __restrict__ out, int h, int w, float scale, float offset) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w || y >= h) return;
  const float q = __fdiv_rn(num[(long)y * pitch + x], den[(long)y * pitch + x]);
  out[(long)y * w + x] = __fadd_rn(__fmul_rn(q, scale), offset);
}

// laplacian_encoder.py:6-40: rows are extrapolated first, then the columns of the row-padded tensor.
__device__ __forceinline__ float row_padded(const float* x, int h, int w, int r, int c) {   // r in [-1, h], c in [0, w)
  if (r >= 0 && r < h) return x[(long)r * w + c];
  if (h == 1) return x[c];
  if (r < 0) return __fsub_rn(__fmul_rn(2.0f, x[c]), x[(long)w + c]);
  return __fsub_rn(__fmul_rn(2.0f, x[(long)(h - 1) * w + c]), x[(long)(h - 2) * w + c]);
}
__global__ void post_pad_extrapolate_kernel(const float* __restrict__ x, int h, int w, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= w + 2 || oy >= h + 2) return;
  const int r = oy - 1, c = ox - 1;
  float v;
  if (c >= 0 && c < w) v = row_padded(x, h, w, r, c);
  else if (w == 1) v = row_padded(x, h, w, r, 0);
  else if (c < 0) v = __fsub_rn(__fmul_rn(2.0f, row_padded(x, h, w, r, 0)), row_padded(x, h, w, r, 1));
  else v = __fsub_rn(__fmul_rn(2.0f, row_padded(x, h, w, r, w - 1)), row_padded(x, h, w, r, w - 2));
  out[(long)oy * (w + 2) + ox] = v;
}

// One axis of torch's interpolate(mode="bilinear", antialias=True) (ATen UpSampleKernel.cpp,
// _compute_indices_min_size_weights_aa with the triangle filter): weights are normalised first, then accumulated in
// tap order.  axis 1: out[y][i] over rows of x;  axis 0: out[i][x] over columns.
__global__ void resize_aa_axis_kernel(const float* __restrict__ x, int h, int w, float* __restrict__ out, int out_size,
                                      int axis) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  const int oh = axis == 0 ? out_size : h, ow = axis == 1 ? out_size : w;
  if (ox >= ow || oy >= oh) return;
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
  out[(long)oy * ow + ox] = acc;
}

struct BlurParams {
  float k[32];
  int ksize;
};
// torchvision gaussian_blur: reflect padding ksize/2, 2-D kernel = outer(k, k), taps accumulated row-major.
__global__ void gaussian_blur_kernel(const float* __restrict__ x, int h, int w, float* __restrict__ out,
                                     const BlurParams bp) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= w || oy >= h) return;
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
  out[(long)oy * w + ox] = acc;
}

// api.py:73-77: floor, clip, '<i2'.  numpy's clip keeps a NaN and its cast to int16 gives 0 on x86 (fmaxf would drop
// the NaN and pack -32768), so NaN packs as 0; +-inf clip to 32767 / -32768.
__device__ __forceinline__ int16_t elev_to_i16(float v) {
  const float f = v != v ? 0.f : fminf(fmaxf(floorf(v), -32768.f), 32767.f);
  return (int16_t)f;
}

__global__ void post_combine_kernel(const float* __restrict__ a, long a_pitch, const float* __restrict__ b, long b_pitch,
                                    float* __restrict__ out, int16_t* __restrict__ out_i16, int h, int w,
                                    int signed_square) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w || y >= h) return;
  float v = __fadd_rn(a[(long)y * a_pitch + x], b[(long)y * b_pitch + x]);
  if (signed_square) v = v == 0.f ? 0.f : copysignf(__fmul_rn(v, v), v);   // sign(v) * v^2 (world_pipeline.py:1312)
  if (out) out[(long)y * w + x] = v;
  if (out_i16) out_i16[(long)y * w + x] = elev_to_i16(v);
}

// The HTTP API's terrain read-out (api.py:103-166 _get_terrain + :80-100 _binary_response): torch's CPU
// upsample_bilinear2d (align_corners=False, scale factor given) of the padded native window, evaluated only at the kept
// output pixels, then the wire packing.  torch takes one of two CPU kernels by the size of the WHOLE upsampled window
// (ATen UpSampleKernel.cpp, _use_vectorized_kernel_cond_2d: out_h + out_w <= 128 picks the per-pixel-weight kernel),
// and the two round differently; both are restated here operation for operation (fma = the contraction x86 builds do):
//   per axis:  src = max(fma(r, d + 0.5, -0.5), 0), r = fp32(1/scale);  i0 = min(floor(src), n-1), i1 = i0 + (i0 < n-1);
//              l1 = clamp(src - i0, 0, 1), l0 = 1 - l1
//   wide  (separable):   t_a = fma(wl0, x[a][j0], wl1 * x[a][j1]);  out = fma(hl0, t_i0, hl1 * t_i1)
//   small (out_h + out_w <= 128):  w_ab = hl_a * wl_b;  out = fma(w11, x11, fma(w10, x10, fma(w00, x00, w01 * x01)))
// scale == 1 is no interpolation at all (the reference returns get()'s window as is): a plain copy, so an inf does not
// meet a zero weight.
struct UpsampleParams {
  const float* elev;      // [h][w]
  const float* climate;   // [5][h][w] or NULL
  float* elev_out;        // [H][W] or NULL
  float* climate_out;     // [5][H][W] or NULL
  uint16_t* payload;      // H*W int16 + H*W*4 fp32 (channels 0..3 interleaved), as 16-bit words, or NULL
  int h, w, scale, oi, oj, H, W, small;
  float r;
};
struct AxisTap {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ AxisTap upsample_axis(int d, int n, float r) {
  const float src = fmaxf(__fmaf_rn(r, __fadd_rn((float)d, 0.5f), -0.5f), 0.0f);
  AxisTap t;
  t.i0 = min((int)floorf(src), n - 1);
  t.i1 = t.i0 + (t.i0 < n - 1 ? 1 : 0);
  t.l1 = fminf(fmaxf(__fsub_rn(src, (float)t.i0), 0.0f), 1.0f);
  t.l0 = __fsub_rn(1.0f, t.l1);
  return t;
}
__global__ void terrain_upsample_kernel(const UpsampleParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.W || y >= p.H) return;
  AxisTap ty, tx;
  if (p.scale == 1) {
    ty.i0 = ty.i1 = p.oi + y;
    tx.i0 = tx.i1 = p.oj + x;
  } else {
    ty = upsample_axis(p.oi + y, p.h, p.r);
    tx = upsample_axis(p.oj + x, p.w, p.r);
  }
  float w00 = 0.f, w01 = 0.f, w10 = 0.f, w11 = 0.f;
  if (p.small) {
    w00 = __fmul_rn(ty.l0, tx.l0); w01 = __fmul_rn(ty.l0, tx.l1);
    w10 = __fmul_rn(ty.l1, tx.l0); w11 = __fmul_rn(ty.l1, tx.l1);
  }
  const long r0 = (long)ty.i0 * p.w, r1 = (long)ty.i1 * p.w;
  auto sample = [&](const float* f) {
    if (p.scale == 1) return f[r0 + tx.i0];
    const float x00 = f[r0 + tx.i0], x01 = f[r0 + tx.i1], x10 = f[r1 + tx.i0], x11 = f[r1 + tx.i1];
    if (p.small)
      return __fmaf_rn(w11, x11, __fmaf_rn(w10, x10, __fmaf_rn(w00, x00, __fmul_rn(w01, x01))));
    const float t0 = __fmaf_rn(tx.l0, x00, __fmul_rn(tx.l1, x01));
    const float t1 = __fmaf_rn(tx.l0, x10, __fmul_rn(tx.l1, x11));
    return __fmaf_rn(ty.l0, t0, __fmul_rn(ty.l1, t1));
  };
  const long o = (long)y * p.W + x, plane_in = (long)p.h * p.w, plane_out = (long)p.H * p.W;
  const float e = sample(p.elev);
  if (p.elev_out) p.elev_out[o] = e;
  if (p.payload) p.payload[o] = (uint16_t)elev_to_i16(e);
  if (!p.climate) return;
  // channel 4 (the lapse rate) is in get_terrain's climate but not on the wire
  const int n_ch = p.climate_out ? 5 : 4;
  uint16_t* wire = p.payload ? p.payload + plane_out + 8 * o : nullptr;   // 2*H*W bytes in: only 2-byte aligned
  for (int c = 0; c < n_ch; ++c) {
    const float v = sample(p.climate + c * plane_in);
    if (p.climate_out) p.climate_out[c * plane_out + o] = v;
    if (wire && c < 4) {
      const uint32_t bits = __float_as_uint(v);
      wire[2 * c] = (uint16_t)(bits & 0xFFFFu);                            // little-endian fp32
      wire[2 * c + 1] = (uint16_t)(bits >> 16);
    }
  }
}

// Land-weighted windowed regression of temperature on elevation (inference/postprocessing.py:262-326, called by
// WorldPipeline._compute_climate with win = 15): one thread per valid-window output, window sums in row-major tap order.
// e = sign(c0) * max(0, c0)^2 is the de-normalised coarse elevation (world_pipeline.py:1329), land mask = e > 0.
struct LapseParams {
  int h, w, win;
  float beta_lo, beta_hi, fallback_beta, eps, fallback_threshold;
};
__global__ void lapse_rate_kernel(const float* __restrict__ temp, const float* __restrict__ c0, float* __restrict__ t_sea,
                                  float* __restrict__ beta_out, const LapseParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  const int oh = p.h - p.win + 1, ow = p.w - p.win + 1;
  if (ox >= ow || oy >= oh) return;
  float s_w = 0.f, s_T = 0.f, s_e = 0.f, s_e2 = 0.f, s_eT = 0.f;
  for (int dy = 0; dy < p.win; ++dy) {
    for (int dx = 0; dx < p.win; ++dx) {
      const long idx = (long)(oy + dy) * p.w + ox + dx;
      const float c = c0[idx], T = temp[idx];
      const float e = c > 0.f ? __fmul_rn(c, c) : 0.f;
      const float m = e > 0.f ? 1.f : 0.f;
      s_w = __fadd_rn(s_w, m);
      s_T = __fadd_rn(s_T, __fmul_rn(T, m));
      s_e = __fadd_rn(s_e, __fmul_rn(e, m));
      s_e2 = __fadd_rn(s_e2, __fmul_rn(__fmul_rn(e, e), m));
      s_eT = __fadd_rn(s_eT, __fmul_rn(__fmul_rn(e, T), m));
    }
  }
  const float n = (float)(p.win * p.win);
  const float den = __fdiv_rn(s_w, n);
  const float dd = __fadd_rn(den, p.eps);
  const float mu_T = __fdiv_rn(__fdiv_rn(s_T, n), dd), mu_e = __fdiv_rn(__fdiv_rn(s_e, n), dd);
  const float mu_e2 = __fdiv_rn(__fdiv_rn(s_e2, n), dd), mu_eT = __fdiv_rn(__fdiv_rn(s_eT, n), dd);
  const float var_e = __fsub_rn(mu_e2, __fmul_rn(mu_e, mu_e));
  const float cov = __fsub_rn(mu_eT, __fmul_rn(mu_e, mu_T));
  float b = __fdiv_rn(cov, __fadd_rn(var_e, p.eps));
  if (var_e < 1.0f || den < p.fallback_threshold) b = p.fallback_beta;
  b = fminf(fmaxf(b, p.beta_lo), p.beta_hi);
  const int pad = (p.win - 1) / 2;
  const long cidx = (long)(oy + pad) * p.w + ox + pad;
  const float cc = c0[cidx];
  const float ec = cc > 0.f ? __fmul_rn(cc, cc) : 0.f;
  t_sea[(long)oy * ow + ox] = __fsub_rn(temp[cidx], __fmul_rn(b, ec));
  beta_out[(long)oy * ow + ox] = b;
}

// grid_sample(bilinear, border, align_corners=False) of [t_sea, beta, central coarse channels] at the pixel centres of
// the requested window + the lapse-rate correction (world_pipeline.py:1333-1365).  One thread per output pixel.
struct ClimateParams {
  const float* t_sea;
  const float* beta;
  const float* coarse;   // [n_ch][hc][wc] normalised coarse planes; the sampled "central" part starts at (crop, crop)
  const float* elev;     // [h][w]
  float* out;            // [5][h][w]
  int hc, wc, crop, hs, ws, i1, j1, h, w, S, ci1, cj1;
};
__device__ __forceinline__ float unnormalize_border(float g, int size) {
  float c = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.0f), (float)size), 1.0f), 2.0f);
  return fminf(fmaxf(c, 0.0f), (float)(size - 1));
}
__global__ void climate_sample_kernel(const ClimateParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.w || y >= p.h) return;
  const float S = (float)p.S;
  const float u = __fadd_rn(__fsub_rn(__fdiv_rn((float)(p.i1 + y) + 0.5f, S), (float)p.ci1), 0.5f);
  const float v = __fadd_rn(__fsub_rn(__fdiv_rn((float)(p.j1 + x) + 0.5f, S), (float)p.cj1), 0.5f);
  const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(__fadd_rn(u, 0.5f), 2.0f), (float)p.hs), 1.0f);
  const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(__fadd_rn(v, 0.5f), 2.0f), (float)p.ws), 1.0f);
  const float sy = unnormalize_border(gy, p.hs), sx = unnormalize_border(gx, p.ws);
  const float fy = floorf(sy), fx = floorf(sx);
  const float wy1 = __fsub_rn(sy, fy), wx1 = __fsub_rn(sx, fx);
  const float wy0 = __fsub_rn(1.0f, wy1), wx0 = __fsub_rn(1.0f, wx1);
  const int y0 = (int)fy, x0 = (int)fx, y1 = y0 + 1, x1 = x0 + 1;
  const bool oky1 = y1 < p.hs, okx1 = x1 < p.ws;   // (y0, x0 are inside after the border clamp)
  const float w00 = __fmul_rn(wy0, wx0), w01 = __fmul_rn(wy0, wx1), w10 = __fmul_rn(wy1, wx0), w11 = __fmul_rn(wy1, wx1);
  auto sample = [&](const float* f, long pitch) {   // f = first element of the sampled [hs][ws] window
    float o = __fmul_rn(f[(long)y0 * pitch + x0], w00);
    o = __fadd_rn(o, okx1 ? __fmul_rn(f[(long)y0 * pitch + x1], w01) : 0.f);
    o = __fadd_rn(o, oky1 ? __fmul_rn(f[(long)y1 * pitch + x0], w10) : 0.f);
    o = __fadd_rn(o, (oky1 && okx1) ? __fmul_rn(f[(long)y1 * pitch + x1], w11) : 0.f);
    return o;
  };
  const float tb = sample(p.t_sea, p.ws), be = sample(p.beta, p.ws);
  const long cplane = (long)p.hc * p.wc;
  const float* central = p.coarse + (long)p.crop * p.wc + p.crop;
  const long plane = (long)p.h * p.w, o = (long)y * p.w + x;
  const float e = p.elev[o];                        // torch.maximum(elev, 0) keeps a NaN elevation (fmaxf would not)
  p.out[o] = __fadd_rn(tb, __fmul_rn(be, e != e ? e : fmaxf(e, 0.0f)));
  p.out[plane + o] = sample(central + 3 * cplane, p.wc);
  p.out[2 * plane + o] = sample(central + 4 * cplane, p.wc);
  p.out[3 * plane + o] = sample(central + 5 * cplane, p.wc);
  p.out[4 * plane + o] = be;
}

static int launch2d(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int h, int w, cudaStream_t stream) {
  fill_launch_config(cfg, attr, dim3((w + 127) / 128, h), dim3(128), 0, stream);
  return TDX_OK;
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_post_normalize(const float* num, const float* den, int64_t pitch, float* out, int32_t h, int32_t w,
                                  float scale, float offset, void* stream) {
  TDX_REQUIRE(num && den && out, "post_normalize: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && h <= 65535 && pitch >= w, "post_normalize: bad shape %d x %d (pitch %lld)", h, w,
              (long long)pitch);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, h, w, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, post_normalize_kernel, num, den, (long)pitch, out, (int)h, (int)w, scale,
                                    offset));
  return TDX_OK;
}

extern "C" int tdx_post_pad_extrapolate(const float* x, int32_t h, int32_t w, float* out, void* stream) {
  TDX_REQUIRE(x && out, "post_pad_extrapolate: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && h + 2 <= 65535, "post_pad_extrapolate: bad shape %d x %d", h, w);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, h + 2, w + 2, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, post_pad_extrapolate_kernel, x, (int)h, (int)w, out));
  return TDX_OK;
}

extern "C" int tdx_resize_aa_axis(const float* x, int32_t h, int32_t w, float* out, int32_t out_size, int32_t axis,
                                  void* stream) {
  TDX_REQUIRE(x && out, "resize_aa_axis: null pointer");
  TDX_REQUIRE(axis == 0 || axis == 1, "resize_aa_axis: axis=%d (0 = height, 1 = width)", axis);
  TDX_REQUIRE(h >= 1 && w >= 1 && out_size >= 1, "resize_aa_axis: bad shape %d x %d -> %d", h, w, out_size);
  const int oh = axis == 0 ? out_size : h, ow = axis == 1 ? out_size : w;
  TDX_REQUIRE(oh <= 65535, "resize_aa_axis: more than 65535 output rows");
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, oh, ow, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, resize_aa_axis_kernel, x, (int)h, (int)w, out, (int)out_size, (int)axis));
  return TDX_OK;
}

extern "C" int tdx_gaussian_blur(const float* x, int32_t h, int32_t w, float* out, int32_t ksize, float sigma,
                                 void* stream) {
  TDX_REQUIRE(x && out && x != out, "gaussian_blur: null or aliased pointers");
  TDX_REQUIRE(ksize >= 1 && ksize <= 31 && (ksize & 1), "gaussian_blur: kernel size %d (odd, <= 31)", ksize);
  TDX_REQUIRE(sigma > 0.f, "gaussian_blur: sigma must be positive");
  TDX_REQUIRE(h > ksize / 2 && w > ksize / 2 && h <= 65535,
              "gaussian_blur: reflect padding of %d needs both dimensions larger than that (got %d x %d)", ksize / 2, h, w);
  BlurParams bp;
  bp.ksize = ksize;
  // torchvision _get_gaussian_kernel1d in float32: taps on linspace(-(k-1)/2, (k-1)/2, k), normalised by their sum
  const float half = (ksize - 1) * 0.5f;
  float sum = 0.f;
  for (int i = 0; i < ksize; ++i) {
    const float t = (-half + (float)i) / sigma;
    bp.k[i] = expf(-0.5f * (t * t));
    sum += bp.k[i];
  }
  for (int i = 0; i < ksize; ++i) bp.k[i] /= sum;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, h, w, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gaussian_blur_kernel, x, (int)h, (int)w, out, bp));
  return TDX_OK;
}

extern "C" int tdx_post_combine(const float* a, int64_t a_pitch, const float* b, int64_t b_pitch, float* out,
                                int16_t* out_i16, int32_t h, int32_t w, int32_t signed_square, void* stream) {
  TDX_REQUIRE(a && b && (out || out_i16), "post_combine: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && h <= 65535 && a_pitch >= w && b_pitch >= w, "post_combine: bad shape %d x %d", h, w);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, h, w, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, post_combine_kernel, a, (long)a_pitch, b, (long)b_pitch, out, out_i16, (int)h,
                                    (int)w, (int)signed_square));
  return TDX_OK;
}

extern "C" int tdx_terrain_upsample(const float* elev, const float* climate, int32_t h, int32_t w, int32_t scale,
                                    int32_t oi, int32_t oj, int32_t H, int32_t W, float* elev_out, float* climate_out,
                                    void* payload, void* stream) {
  TDX_REQUIRE(elev && (elev_out || climate_out || payload), "terrain_upsample: null input or no output");
  TDX_REQUIRE(!climate_out || climate, "terrain_upsample: climate_out without a climate window");
  TDX_REQUIRE(((uintptr_t)payload & 1) == 0, "terrain_upsample: payload must be 2-byte aligned");
  TDX_REQUIRE(scale >= 1 && h >= 1 && w >= 1 && H >= 1 && W >= 1 && H <= 65535,
              "terrain_upsample: bad shape %d x %d x%d -> %d x %d", h, w, scale, H, W);
  TDX_REQUIRE(oi >= 0 && oj >= 0 && (int64_t)oi + H <= (int64_t)h * scale && (int64_t)oj + W <= (int64_t)w * scale,
              "terrain_upsample: crop %d x %d at (%d, %d) outside the %d x %d upsampled window", H, W, oi, oj, h * scale,
              w * scale);
  UpsampleParams p;
  p.elev = elev; p.climate = climate; p.elev_out = elev_out; p.climate_out = climate_out;
  p.payload = static_cast<uint16_t*>(payload);
  p.h = h; p.w = w; p.scale = scale; p.oi = oi; p.oj = oj; p.H = H; p.W = W;
  p.small = ((int64_t)h + w) * scale <= 128;
  p.r = (float)(1.0 / scale);                          // compute_scales_value: static_cast<float>(1.0 / scale)
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, H, W, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, terrain_upsample_kernel, p));
  return TDX_OK;
}

extern "C" int tdx_lapse_rate(const float* temp, const float* coarse_elev_sqrt, int32_t h, int32_t w, int32_t win,
                              float beta_lo, float beta_hi, float fallback_beta, float eps, float fallback_threshold,
                              float* t_sea, float* beta, void* stream) {
  TDX_REQUIRE(temp && coarse_elev_sqrt && t_sea && beta, "lapse_rate: null pointer");
  TDX_REQUIRE(win >= 3 && (win & 1) && h >= win && w >= win && h <= 65535, "lapse_rate: bad shape %d x %d, window %d", h,
              w, win);
  LapseParams p;
  p.h = h; p.w = w; p.win = win;
  p.beta_lo = beta_lo; p.beta_hi = beta_hi; p.fallback_beta = fallback_beta; p.eps = eps;
  p.fallback_threshold = fallback_threshold;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, h - win + 1, w - win + 1, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, lapse_rate_kernel, temp, coarse_elev_sqrt, t_sea, beta, p));
  return TDX_OK;
}

extern "C" int tdx_climate_sample(const float* t_sea, const float* beta, const float* coarse, int32_t n_ch, int32_t hc,
                                  int32_t wc, int32_t crop, const float* elev, int32_t i1, int32_t j1, int32_t h,
                                  int32_t w, int32_t coarse_stride, int32_t ci1, int32_t cj1, float* out, void* stream) {
  TDX_REQUIRE(t_sea && beta && coarse && elev && out, "climate_sample: null pointer");
  TDX_REQUIRE(n_ch >= 6, "climate_sample: the coarse map needs >= 6 channels (3, 4, 5 are sampled), got %d", n_ch);
  TDX_REQUIRE(crop >= 0 && hc > 2 * crop && wc > 2 * crop, "climate_sample: coarse window %d x %d too small for crop %d",
              hc, wc, crop);
  TDX_REQUIRE(h >= 1 && w >= 1 && h <= 65535 && coarse_stride >= 1, "climate_sample: bad shape %d x %d", h, w);
  ClimateParams p;
  p.t_sea = t_sea; p.beta = beta; p.coarse = coarse; p.elev = elev; p.out = out;
  p.hc = hc; p.wc = wc; p.crop = crop; p.hs = hc - 2 * crop; p.ws = wc - 2 * crop;
  p.i1 = i1; p.j1 = j1; p.h = h; p.w = w; p.S = coarse_stride; p.ci1 = ci1; p.cj1 = cj1;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  launch2d(&cfg, attr, h, w, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, climate_sample_kernel, p));
  return TDX_OK;
}
