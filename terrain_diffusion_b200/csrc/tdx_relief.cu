// Shaded relief map (get_relief_map, inference/relief_map.py:64-199): the picture the explorer and the evaluation
// scripts show of an elevation window.  The reference runs it on the CPU after copying the elevation to the host:
// scipy.ndimage.gaussian_filter at two scales, np.gradient + a GDAL-style hillshade per scale, matplotlib's `terrain`
// colormap and an ocean blend.  Here it is three calls on the device:
//   tdx_relief_stats     NaN count and nanmin / nanmax of max(0, elev) into a small device buffer (:135-140),
//   tdx_relief_gaussian  both Gaussian filters, one launch per axis (:125-126),
//   tdx_relief_shade     gradients, hillshades, colormap, intensity, NaN mask and ocean blend, one thread per pixel
//                        (:111-122, :128-199); it reads the statistics from the device buffer, so no host round trip.
// Arithmetic follows the dtypes numpy uses: fp32 where the reference's arrays are fp32, fp64 where a float64 scalar
// promotes (the hillshade sum) or scipy accumulates in double (the filter), each op explicitly rounded so that FMA
// contraction cannot change a result.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

constexpr int kReliefMaxRadius = 96;   // int(4 sigma + 0.5) <= 96: sigma < 24
constexpr int kReliefLut = 256;        // matplotlib rcParams['image.lut']

// scipy's mode='reflect' (half-sample symmetric, period 2n), also when the filter reaches past the far edge.
__device__ __forceinline__ int reflect_index(int i, int n) {
  int m = i % (2 * n);
  if (m < 0) m += 2 * n;
  return m >= n ? 2 * n - 1 - m : m;
}

struct ReliefTaps {
  double w[2][kReliefMaxRadius + 1];   // w[s][k]: weight at distance k from the centre (symmetric filter)
  int radius[2];
};

// One axis of scipy.ndimage.correlate1d with a symmetric odd filter (NI_Correlate1D): the line is read in double,
// out = x[i]*w[0], then for k = r..1: out += (x[i-k] + x[i+k]) * w[k]; the result is stored as fp32, as scipy writes
// the float32 output array between the two axes.  blockIdx.z selects the sigma.
__global__ void relief_gauss_kernel(const float* __restrict__ in, long in_sigma_stride, float* __restrict__ out, int h,
                                    int w, int axis, int replace_nan, float nan_fill, const ReliefTaps t) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y, s = blockIdx.z;
  if (ox >= w) return;
  const int r = t.radius[s];
  const double* wt = t.w[s];
  const int n = axis == 0 ? h : w, i = axis == 0 ? oy : ox;
  const long step = axis == 0 ? w : 1;
  const float* line = in + s * in_sigma_stride + (axis == 0 ? (long)ox : (long)oy * w);
  auto at = [&](int j) {
    float v = line[(long)j * step];
    if (replace_nan && isnan(v)) v = nan_fill;
    return (double)v;
  };
  double acc = __dmul_rn(at(i), wt[0]);
  if (i - r >= 0 && i + r < n) {
    for (int k = r; k >= 1; --k) acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(at(i - k), at(i + k)), wt[k]));
  } else {
    for (int k = r; k >= 1; --k)
      acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(at(reflect_index(i - k, n)), at(reflect_index(i + k, n))), wt[k]));
  }
  out[(long)s * h * w + (long)oy * w + ox] = __double2float_rn(acc);
}

// stats[0] = NaN count; stats[1] = ~bits(nanmin), stats[2] = bits(nanmax) of max(0, x).  The values are >= +0, so
// their bit patterns order like the floats and both extrema are atomicMax on a zeroed buffer.  With no finite value
// stats[1] decodes to +inf (or NaN bits), which the shade kernel treats like the reference's non-finite range.
__global__ void relief_stats_kernel(const float* __restrict__ x, long n, unsigned* __restrict__ stats) {
  pdl_launch_dependents();
  pdl_wait();
  unsigned cnt = 0;
  float mn = __int_as_float(0x7f800000), mx = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float v = x[i];
    if (isnan(v)) {
      ++cnt;
    } else {
      const float l = v > 0.f ? v : 0.f;
      mn = fminf(mn, l);
      mx = fmaxf(mx, l);
    }
  }
  unsigned nmn = ~__float_as_uint(mn), bmx = __float_as_uint(mx);
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    nmn = max(nmn, __shfl_xor_sync(0xffffffffu, nmn, o));
    bmx = max(bmx, __shfl_xor_sync(0xffffffffu, bmx, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (cnt) atomicAdd(&stats[0], cnt);
    atomicMax(&stats[1], nmn);
    atomicMax(&stats[2], bmx);
  }
}

// numpy's fp32 transcendental ufuncs, evaluated in double and rounded once.
__device__ __forceinline__ float pow_f32(float x, float e) { return __double2float_rn(pow((double)x, (double)e)); }
__device__ __forceinline__ float clip01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }   // keeps NaN

struct ShadeParams {
  const float* elev;
  const float* blurred;    // [2][h][w]: sigma_large, sigma_small
  const unsigned* stats;   // tdx_relief_stats output
  const float* lut;        // [256][3]
  float* out;              // [h][w][3]
  int h, w;
  int replace_nan, user_range, vmin_is_zero;
  float nan_fill, grad_div, relief, one_minus_relief, vmin, denom;
  double az, sin_alt, cos_alt;
};

// compute_hillshade (relief_map.py:111-122) at one pixel: np.gradient (edge order 1), / (15*resolution/90), slope and
// aspect in fp32, then the sin/cos mix in fp64 (np.deg2rad returns a float64 scalar, which promotes under NEP 50),
// clip, cast to fp32.
__device__ __forceinline__ float hillshade(const float* __restrict__ p, const ShadeParams& q, int y, int x) {
  const int h = q.h, w = q.w;
  const long o = (long)y * w + x;
  float dy, dx;
  if (y == 0) dy = __fsub_rn(p[o + w], p[o]);
  else if (y == h - 1) dy = __fsub_rn(p[o], p[o - w]);
  else dy = __fmul_rn(__fsub_rn(p[o + w], p[o - w]), 0.5f);
  if (x == 0) dx = __fsub_rn(p[o + 1], p[o]);
  else if (x == w - 1) dx = __fsub_rn(p[o], p[o - 1]);
  else dx = __fmul_rn(__fsub_rn(p[o + 1], p[o - 1]), 0.5f);
  dy = __fdiv_rn(dy, q.grad_div);
  dx = __fdiv_rn(dx, q.grad_div);
  const double ddx = dx, ddy = dy;
  const float hyp = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(ddx, ddx), __dmul_rn(ddy, ddy))));
  const float slope = __fsub_rn(1.57079637f, __double2float_rn(atan((double)hyp)));   // fp32(pi/2) - arctan
  const float aspect = __double2float_rn(atan2(ddy, -ddx));
  const double sin_s = __double2float_rn(sin((double)slope)), cos_s = __double2float_rn(cos((double)slope));
  double hs = __dadd_rn(__dmul_rn(q.sin_alt, sin_s),
                        __dmul_rn(__dmul_rn(q.cos_alt, cos_s), cos(__dsub_rn(q.az, (double)aspect))));
  hs = hs < 0.0 ? 0.0 : (hs > 1.0 ? 1.0 : hs);
  return __double2float_rn(hs);
}

__global__ void relief_shade_kernel(const ShadeParams q) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= q.w) return;
  const long o = (long)y * q.w + x, plane = (long)q.h * q.w;
  const float raw = q.elev[o];
  const bool is_nan = isnan(raw);
  const float filled = is_nan && q.replace_nan ? q.nan_fill : raw;

  // multi-scale hillshade (:128-131)
  const float hs_l = hillshade(q.blurred, q, y, x), hs_s = hillshade(q.blurred + plane, q, y, x);
  const float hill = pow_f32(clip01(__fadd_rn(__fmul_rn(0.75f, hs_l), __fmul_rn(0.25f, hs_s))), 0.85f);

  // elevation colour (:134-151): norm in fp32 against the fp32-rounded range; Python-float scalars rounded once
  float vmin = q.vmin, denom = q.denom;
  bool zero = q.vmin_is_zero;
  if (!q.user_range) {
    const float lo = __uint_as_float(~q.stats[1]), hi = __uint_as_float(q.stats[2]);
    const bool fallback = !isfinite(lo) || !isfinite(hi) || hi == lo;
    const double dlo = fallback ? 0.0 : (double)lo, dhi = fallback ? 1.0 : (double)hi;
    vmin = (float)dlo;
    denom = __double2float_rn(__dadd_rn(__dsub_rn(dhi, dlo), 1e-8));
    zero = dlo == 0.0;
  }
  const float land = is_nan ? raw : (raw > 0.f ? raw : 0.f);
  const float norm = __fdiv_rn(__fsub_rn(land, vmin), denom);
  float c = clip01(pow_f32(norm, 0.7f));
  if (zero) c = __fadd_rn(0.25f, __fmul_rn(c, 0.75f));
  // Colormap.__call__: x*N, x == N -> N-1, under -> first, over -> last, NaN -> bad colour (0, 0, 0)
  const float xa = __fmul_rn(c, (float)kReliefLut);
  float base[3] = {0.f, 0.f, 0.f};
  if (!isnan(xa)) {
    const int idx = xa < 0.f ? 0 : (xa >= (float)kReliefLut ? kReliefLut - 1 : (int)xa);
    for (int k = 0; k < 3; ++k) base[k] = q.lut[idx * 3 + k];
  }

  // GDAL-like intensity blend (:167-169)
  const float m = __fadd_rn(__fmul_rn(q.relief, __fadd_rn(0.35f, __fmul_rn(0.65f, hill))), q.one_minus_relief);
  float rgb[3];
  for (int k = 0; k < 3; ++k) rgb[k] = is_nan ? __int_as_float(0x7fc00000) : clip01(__fmul_rn(base[k], m));

  // ocean (:183-197), keyed on the NaN-filled elevation: a NaN pixel filled with a negative median turns ocean-blue
  if (filled < 0.f) {
    const float t = pow_f32(clip01(__fdiv_rn(-filled, 10000.0f)), 0.7f), u = __fsub_rn(1.0f, t);
    const float coast[3] = {0.68f, 0.88f, 1.00f}, deep[3] = {0.00f, 0.10f, 0.45f};
    for (int k = 0; k < 3; ++k) rgb[k] = __fadd_rn(__fmul_rn(u, coast[k]), __fmul_rn(t, deep[k]));
  }
  for (int k = 0; k < 3; ++k) q.out[o * 3 + k] = rgb[k];
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_relief_stats(const float* elev, int64_t n, uint32_t* stats, void* stream) {
  TDX_REQUIRE(elev && stats, "relief_stats: null pointer");
  TDX_REQUIRE(n >= 1, "relief_stats: empty input");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TDX_CHECK_CUDA(cudaMemsetAsync(stats, 0, 3 * sizeof(uint32_t), st));
  const long blocks = (n + 255) / 256;
  const int grid = (int)(blocks < 4L * sm_count() ? blocks : 4L * sm_count());
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3(grid), dim3(256), 0, st);
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, relief_stats_kernel, elev, (long)n, reinterpret_cast<unsigned*>(stats)));
  return TDX_OK;
}

extern "C" int tdx_relief_gaussian(const float* x, int32_t h, int32_t w, int32_t replace_nan, float nan_fill,
                                   int32_t n_sigma, const double* weights, const int32_t* radius, float* tmp,
                                   float* out, void* stream) {
  TDX_REQUIRE(x && weights && radius && tmp && out, "relief_gaussian: null pointer");
  TDX_REQUIRE(x != tmp && x != out && tmp != out, "relief_gaussian: aliased buffers");
  TDX_REQUIRE(h >= 1 && w >= 1 && h <= 65535, "relief_gaussian: bad shape %d x %d", h, w);
  TDX_REQUIRE(n_sigma == 1 || n_sigma == 2, "relief_gaussian: n_sigma=%d (1 or 2)", n_sigma);
  ReliefTaps t = {};
  const double* wk = weights;
  for (int s = 0; s < n_sigma; ++s) {
    const int r = radius[s];
    TDX_REQUIRE(r >= 0 && r <= kReliefMaxRadius, "relief_gaussian: radius %d outside [0, %d]", r, kReliefMaxRadius);
    for (int k = 0; k <= r; ++k) {
      TDX_REQUIRE(wk[r - k] == wk[r + k], "relief_gaussian: filter %d is not symmetric", s);
      t.w[s][k] = wk[r - k];
    }
    t.radius[s] = r;
    wk += 2 * r + 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long plane = (long)h * w;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3((w + 127) / 128, h, n_sigma), dim3(128), 0, st);
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, relief_gauss_kernel, x, 0L, tmp, (int)h, (int)w, 0, (int)replace_nan,
                                    nan_fill, t));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, relief_gauss_kernel, (const float*)tmp, plane, out, (int)h, (int)w, 1, 0,
                                    0.f, t));
  return TDX_OK;
}

extern "C" int tdx_relief_shade(const float* elev, const float* blurred, const uint32_t* stats, const float* lut,
                                int32_t h, int32_t w, int32_t replace_nan, float nan_fill, float grad_div, double az_rad,
                                double sin_alt, double cos_alt, float relief, float one_minus_relief,
                                int32_t user_range, float vmin, float denom, int32_t vmin_is_zero, float* out,
                                void* stream) {
  TDX_REQUIRE(elev && blurred && lut && out && (stats || user_range), "relief_shade: null pointer");
  TDX_REQUIRE(h >= 2 && w >= 2 && h <= 65535, "relief_shade: bad shape %d x %d (np.gradient needs >= 2 per axis)", h,
              w);
  ShadeParams q;
  q.elev = elev; q.blurred = blurred; q.stats = reinterpret_cast<const unsigned*>(stats); q.lut = lut; q.out = out;
  q.h = h; q.w = w;
  q.replace_nan = replace_nan; q.user_range = user_range; q.vmin_is_zero = vmin_is_zero;
  q.nan_fill = nan_fill; q.grad_div = grad_div; q.relief = relief; q.one_minus_relief = one_minus_relief;
  q.vmin = vmin; q.denom = denom;
  q.az = az_rad; q.sin_alt = sin_alt; q.cos_alt = cos_alt;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3((w + 127) / 128, h), dim3(128), 0, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, relief_shade_kernel, q));
  return TDX_OK;
}
