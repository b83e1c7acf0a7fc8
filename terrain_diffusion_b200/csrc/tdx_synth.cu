// The coarse stage's synthetic conditioning map (terrain_diffusion/inference/synthetic_map.py:182-271 and
// perlin_transform.py:42-45) and the FastNoiseLite noise planes of the Minecraft read-out (minecraft_api.py:127-186).
// The reference evaluates both with pyfastnoiselite on the host.  Here:
//   tdx_fbm_perlin     up to TDX_FBM_MAX_PLANES planes of FastNoiseLite Perlin + FBm, one thread per cell and plane,
//   tdx_synthetic_map  one thread per cell of a [5, h, w] window: the five FBm fields, np.interp through each channel's
//                      quantile tables in fp64, the cast to fp32, then the import merge, `finalize` and the signed
//                      square root of channel 0 as `mode` asks.
//
// Numerical contract: every fp32 and fp64 operation is explicitly rounded (__fmul_rn, __fadd_rn, __dmul_rn, ...), so
// nvcc contracts nothing into an FMA.  FastNoiseLite is restated from its published C source (FastNoiseLite.h, MIT)
// under the assumption that the pyfastnoiselite 0.0.6 wheel was compiled for baseline x86-64, where there is no FMA
// and every float expression rounds at each operation.  No fixture here comes from pyfastnoiselite itself: the kernel is
// pinned to the numpy restatement in oracle/synthetic_map.py.  Cells whose scaled coordinate reaches 2^31 in magnitude
// (|x * frequency * lacunarity^(octaves-1)|) are outside the contract: C's float-to-int conversion is undefined there.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {
namespace {

constexpr int kThreads = 256;
constexpr int kFields = 5;
constexpr int kPrimeX = 501125321;
constexpr int kPrimeY = 1136930381;
constexpr unsigned kHashMul = 0x27d4eb2du;

// FastNoiseLite's Gradients2D: the 24 unit directions (cos t, sin t), t = 82.5 - 15 k degrees; the library's 256-float
// table is these 24 pairs five times over, then the first 8 again, so pair p of the table is pair p % 24 here.
__device__ const float kGrad24[48] = {
    0.130526192f,  0.991444861f,  0.382683432f,  0.923879533f,  0.608761429f,  0.793353340f,  0.793353340f,  0.608761429f,
    0.923879533f,  0.382683432f,  0.991444861f,  0.130526192f,  0.991444861f,  -0.130526192f, 0.923879533f,  -0.382683432f,
    0.793353340f,  -0.608761429f, 0.608761429f,  -0.793353340f, 0.382683432f,  -0.923879533f, 0.130526192f,  -0.991444861f,
    -0.130526192f, -0.991444861f, -0.382683432f, -0.923879533f, -0.608761429f, -0.793353340f, -0.793353340f, -0.608761429f,
    -0.923879533f, -0.382683432f, -0.991444861f, -0.130526192f, -0.991444861f, 0.130526192f,  -0.923879533f, 0.382683432f,
    -0.793353340f, 0.608761429f,  -0.608761429f, 0.793353340f,  -0.382683432f, 0.923879533f,  -0.130526192f, 0.991444861f,
};

// the five generators of synthetic_map.py:219-225: frequency 0.05 * frequency_mult[k] (the caller's), lacunarity 2, gain
// 0.5 and these octaves
__device__ const int kFieldOctaves[kFields] = {4, 2, 4, 4, 4};

// the 256-float Gradients2D table in shared memory, filled by the whole block
__device__ __forceinline__ void load_gradients(float* g) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) g[i] = kGrad24[((i >> 1) % 24) * 2 + (i & 1)];
}

// np.arange(a, b, dtype=np.float32)[k]: numpy stores fp32(a) and fp32(a + 1) and fills the rest as
// fp32(a) + fp32(k) * (fp32(a + 1) - fp32(a)) in fp32.  Only differs from fp32(a + k) where |a| >= 2^24.
__device__ __forceinline__ float arange_f32(long long a, int k) {
  const float first = __ll2float_rn(a);
  if (k == 0) return first;
  const float second = __ll2float_rn(a + 1);
  if (k == 1) return second;
  return __fadd_rn(first, __fmul_rn(__int2float_rn(k), __fsub_rn(second, first)));
}

__device__ __forceinline__ int fast_floor(float f) {           // _fnlFastFloor: (int)f, minus 1 for f < 0
  const int t = __float2int_rz(f);
  return f >= 0.f ? t : t - 1;
}

__device__ __forceinline__ float lerp(float a, float b, float t) {   // a + t * (b - a)
  return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a)));
}

__device__ __forceinline__ float interp_quintic(float t) {     // t * t * t * (t * (t * 6 - 15) + 10), left to right
  const float t3 = __fmul_rn(__fmul_rn(t, t), t);
  return __fmul_rn(t3, __fadd_rn(__fmul_rn(t, __fsub_rn(__fmul_rn(t, 6.f), 15.f)), 10.f));
}

__device__ __forceinline__ float grad_coord(const float* g, int seed, int xp, int yp, float xd, float yd) {
  int hash = (int)((unsigned)(seed ^ xp ^ yp) * kHashMul);     // int32 wrap
  hash ^= hash >> 15;                                          // arithmetic shift, as on a signed int
  hash &= 127 << 1;
  return __fadd_rn(__fmul_rn(xd, g[hash]), __fmul_rn(yd, g[hash | 1]));
}

// _fnlSinglePerlin2D
__device__ __forceinline__ float single_perlin(const float* g, int seed, float x, float y) {
  int x0 = fast_floor(x), y0 = fast_floor(y);
  const float xd0 = __fsub_rn(x, __int2float_rn(x0)), yd0 = __fsub_rn(y, __int2float_rn(y0));
  const float xd1 = __fsub_rn(xd0, 1.f), yd1 = __fsub_rn(yd0, 1.f);
  const float xs = interp_quintic(xd0), ys = interp_quintic(yd0);
  x0 = (int)((unsigned)x0 * (unsigned)kPrimeX);
  y0 = (int)((unsigned)y0 * (unsigned)kPrimeY);
  const int x1 = (int)((unsigned)x0 + (unsigned)kPrimeX), y1 = (int)((unsigned)y0 + (unsigned)kPrimeY);
  const float xf0 = lerp(grad_coord(g, seed, x0, y0, xd0, yd0), grad_coord(g, seed, x1, y0, xd1, yd0), xs);
  const float xf1 = lerp(grad_coord(g, seed, x0, y1, xd0, yd1), grad_coord(g, seed, x1, y1, xd1, yd1), xs);
  return __fmul_rn(lerp(xf0, xf1, ys), 1.4247691104677813f);
}

// fnlGetNoise2D with FNL_FRACTAL_FBM: the coordinate scaled by the frequency, then _fnlGenFractalFBM2D.  The weighted
// strength is 0, so the per-octave `amp *= Lerp(1, ..., 0)` multiplies by exactly 1 and is left out.
__device__ __forceinline__ float fbm_perlin(const float* g, int seed, float frequency, int octaves, float lacunarity,
                                            float gain, float x, float y) {
  x = __fmul_rn(x, frequency);
  y = __fmul_rn(y, frequency);
  // _fnlCalculateFractalBounding: 1 / (1 + g + g^2 + ...), accumulated in float
  const float ag = fabsf(gain);
  float a = ag, fractal = 1.f;
  for (int i = 1; i < octaves; ++i) {
    fractal = __fadd_rn(fractal, a);
    a = __fmul_rn(a, ag);
  }
  float amp = __fdiv_rn(1.f, fractal), sum = 0.f;
  for (int i = 0; i < octaves; ++i) {
    const float noise = single_perlin(g, seed, x, y);
    seed = (int)((unsigned)seed + 1u);
    sum = __fadd_rn(sum, __fmul_rn(noise, amp));
    x = __fmul_rn(x, lacunarity);
    y = __fmul_rn(y, lacunarity);
    amp = __fmul_rn(amp, gain);
  }
  return sum;
}

struct FbmParams {
  int n;
  int seed[TDX_FBM_MAX_PLANES], octaves[TDX_FBM_MAX_PLANES];
  float frequency[TDX_FBM_MAX_PLANES], lacunarity[TDX_FBM_MAX_PLANES], gain[TDX_FBM_MAX_PLANES];
};

// one thread per cell of plane blockIdx.y; x = arange(j0, j0 + w)[c], y = arange(i0, i0 + h)[r]
__global__ void __launch_bounds__(kThreads) fbm_kernel(FbmParams p, long long i0, long long j0, int h, int w,
                                                       float* __restrict__ out) {
  __shared__ float g[256];
  load_gradients(g);
  pdl_launch_dependents();
  pdl_wait();
  __syncthreads();
  const int k = blockIdx.y;
  const long n = (long)h * w;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = (int)(i / w), c = (int)(i % w);
  out[(long)k * n + i] = fbm_perlin(g, p.seed[k], p.frequency[k], p.octaves[k], p.lacunarity[k], p.gain[k],
                                    arange_f32(j0, c), arange_f32(i0, r));
}

// np.interp(x, xp, fp, left=fp[0], right=fp[-1]) in fp64 (numpy/core/src/multiarray/compiled_base.c): the end values
// outside the table and at x == xp[-1], fp[j] on a knot, else slope * (x - xp[j]) + fp[j] for xp[j] <= x < xp[j+1],
// retried from xp[j+1] when that is NaN.
__device__ __forceinline__ double np_interp(double x, const double* xp, const double* fp, int n) {
  if (x == xp[n - 1]) return fp[n - 1];
  if (x > xp[n - 1]) return fp[n - 1];
  if (x < xp[0]) return fp[0];
  int lo = 0, hi = n - 1;                                      // xp[lo] <= x < xp[hi] (NaN: lo stays 0)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (xp[mid] <= x) lo = mid; else hi = mid;
  }
  if (xp[lo] == x) return fp[lo];
  const double slope = __ddiv_rn(__dsub_rn(fp[lo + 1], fp[lo]), __dsub_rn(xp[lo + 1], xp[lo]));
  double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xp[lo])), fp[lo]);
  if (isnan(r)) {
    r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xp[lo + 1])), fp[lo + 1]);
    if (isnan(r) && fp[lo] == fp[lo + 1]) r = fp[lo];
  }
  return r;
}

// np.maximum / np.minimum on fp32: NaN if either is NaN, else the larger (smaller) one, the second on a tie
__device__ __forceinline__ float np_max(float a, float b) { return isnan(a) || isnan(b) ? a + b : (a > b ? a : b); }
__device__ __forceinline__ float np_min(float a, float b) { return isnan(a) || isnan(b) ? a + b : (a < b ? a : b); }

// np.sign(x) * np.sqrt(np.abs(x)) in fp32: +0 for either zero, NaN stays NaN
__device__ __forceinline__ float signed_sqrt(float x) {
  if (x > 0.f) return __fsqrt_rn(x);
  if (x < 0.f) return -__fsqrt_rn(-x);
  return x == 0.f ? 0.f : x;
}

struct SynthImports {
  const float* values[kFields];    // DEVICE fp32 [rows][cols] or NULL
  long long oi[kFields], oj[kFields];
  int rows[kFields], cols[kFields];
  float deflt[kFields];
  unsigned has_default;            // bit c: channel c has a default value
};

struct SynthParams {
  int seed[kFields];
  float frequency[kFields];
  float a, b, p1, p99, span;       // fp32(a_temp_std), fp32(b_temp_std), fp32(p1), fp32(p99), fp32(p99 - p1 in fp64)
};

// synthetic_map.py:232-254 on one cell, in fp32 with every Python scalar rounded to fp32 at its op (NumPy >= 2)
__device__ __forceinline__ void finalize(float v[kFields], const SynthParams& p) {
  const float elev = v[0], precip = v[3];
  float temp = v[1];
  // lapse_rate = (-6.5 + 0.0015 * precip).clip(-9.8, -4.0) / 1000
  const float lapse = __fdiv_rn(np_min(np_max(__fadd_rn(-6.5f, __fmul_rn(0.0015f, precip)), -9.8f), -4.0f), 1000.f);
  temp = __fadd_rn(temp, __fmul_rn(lapse, np_max(0.f, elev)));
  temp = np_min(np_max(temp, -10.f), 40.f);
  temp = temp > 20.f ? temp : __fadd_rn(__fmul_rn(__fsub_rn(temp, 20.f), 1.25f), 20.f);
  const float t = __fdiv_rn(__fsub_rn(v[2], p.p1), p.span);
  const float fit = __fadd_rn(__fmul_rn(p.a, temp), p.b);
  const float baseline = np_max(p.p1, -fit);
  float tstd = __fadd_rn(__fmul_rn(t, __fsub_rn(p.p99, baseline)), baseline);
  tstd = np_max(__fadd_rn(tstd, fit), 20.f);
  const float pcv = __fmul_rn(v[4], np_max(0.f, __fdiv_rn(__fsub_rn(185.f, __fmul_rn(0.04111f, precip)), 185.f)));
  v[1] = temp;
  v[2] = tstd;
  v[4] = pcv;
}

// window origins of a batched call (one per blockIdx.y)
struct SynthOrigins {
  long long i0[TDX_SYNTH_MAX_IMAGES], j0[TDX_SYNTH_MAX_IMAGES];
};

// one thread per cell (r, c) of the [5, h, w] window blockIdx.y at x = arange(j0, j0 + w)[c], y = arange(i0, i0 + h)[r]
__global__ void __launch_bounds__(kThreads) synth_kernel(SynthParams p, SynthImports imp, const double* __restrict__ tables,
                                                         int n_knots, SynthOrigins org, int h, int w,
                                                         const float* __restrict__ input, int mode,
                                                         float* __restrict__ out) {
  extern __shared__ double tab[];                 // [5][2][n_knots], then the 256 gradients
  float* g = reinterpret_cast<float*>(tab + 2 * kFields * n_knots);
  const bool raw_input = mode & TDX_SYNTH_RAW_INPUT;
  if (!input) load_gradients(g);
  pdl_launch_dependents();
  pdl_wait();
  if (!raw_input)
    for (int k = threadIdx.x; k < 2 * kFields * n_knots; k += blockDim.x) tab[k] = tables[k];
  __syncthreads();
  const long n = (long)h * w;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = (int)(i / w), c = (int)(i % w);
  const long long i0 = org.i0[blockIdx.y], j0 = org.j0[blockIdx.y];
  out += (size_t)blockIdx.y * kFields * n;
  float v[kFields];
  if (raw_input) {
#pragma unroll
    for (int f = 0; f < kFields; ++f) v[f] = input[(long)f * n + i];
  } else {
    const float x = input ? 0.f : arange_f32(j0, c), y = input ? 0.f : arange_f32(i0, r);
#pragma unroll
    for (int f = 0; f < kFields; ++f) {
      const float noise = input ? input[(long)f * n + i]
                                : fbm_perlin(g, p.seed[f], p.frequency[f], kFieldOctaves[f], 2.f, 0.5f, x, y);
      const double* xp = tab + 2 * f * n_knots;
      v[f] = __double2float_rn(np_interp((double)noise, xp, xp + n_knots, n_knots));
    }
  }
  if (mode & TDX_SYNTH_IMPORT) {                  // world_pipeline.py:829-880, on absolute cells (i0 + r, j0 + c)
    const long long ci = i0 + r, cj = j0 + c;
#pragma unroll
    for (int f = 0; f < kFields; ++f) {
      const long long di = ci - imp.oi[f], dj = cj - imp.oj[f];
      if (imp.values[f] && di >= 0 && di < imp.rows[f] && dj >= 0 && dj < imp.cols[f])
        v[f] = imp.values[f][di * imp.cols[f] + dj];
      else if ((imp.has_default >> f) & 1u)
        v[f] = imp.deflt[f];
    }
  }
  if (mode & TDX_SYNTH_FINALIZE) finalize(v, p);
  if (mode & TDX_SYNTH_SQRT0) v[0] = signed_sqrt(v[0]);
#pragma unroll
  for (int f = 0; f < kFields; ++f) out[(long)f * n + i] = v[f];
}

int check_window(int32_t h, int32_t w, const char* who) {
  TDX_REQUIRE(h >= 1 && w >= 1, "%s: empty window %d x %d", who, (int)h, (int)w);
  TDX_REQUIRE(h <= (1 << 24) && w <= (1 << 24) && (long)h * w <= (1L << 31),
              "%s: window %d x %d too large (at most 2^24 per axis and 2^31 cells)", who, (int)h, (int)w);
  return TDX_OK;
}

}  // namespace
}  // namespace tdx

using namespace tdx;

extern "C" int tdx_fbm_perlin(int32_t n_planes, const int32_t* seeds, const float* frequency, const int32_t* octaves,
                              const float* lacunarity, const float* gain, int64_t i0, int64_t j0, int32_t h, int32_t w,
                              float* out, void* stream) {
  TDX_REQUIRE(seeds && frequency && octaves && lacunarity && gain && out, "fbm_perlin: null pointer");
  TDX_REQUIRE(n_planes >= 1 && n_planes <= TDX_FBM_MAX_PLANES, "fbm_perlin: %d planes, 1..%d allowed", (int)n_planes,
              TDX_FBM_MAX_PLANES);
  int rc = check_window(h, w, "fbm_perlin");
  if (rc != TDX_OK) return rc;
  TDX_REQUIRE(i0 > -(1LL << 62) && i0 < (1LL << 62) && j0 > -(1LL << 62) && j0 < (1LL << 62),
              "fbm_perlin: window origin out of range");
  FbmParams p{};
  p.n = n_planes;
  for (int k = 0; k < n_planes; ++k) {
    TDX_REQUIRE(octaves[k] >= 1 && octaves[k] <= 16, "fbm_perlin: plane %d has %d octaves, 1..16 allowed", k,
                (int)octaves[k]);
    p.seed[k] = seeds[k];
    p.octaves[k] = octaves[k];
    p.frequency[k] = frequency[k];
    p.lacunarity[k] = lacunarity[k];
    p.gain[k] = gain[k];
  }
  TDX_CHECK_CUDA(launch(fbm_kernel, dim3((unsigned)(((long)h * w + kThreads - 1) / kThreads), (unsigned)n_planes),
                        kThreads, 0, stream, p, (long long)i0, (long long)j0, (int)h, (int)w, out));
  return TDX_OK;
}

// the checks and the launch of tdx_synthetic_map / tdx_synthetic_maps; origins: n_img (i0, j0) pairs on the host
static int synthetic_map_launch(const double* tables, int32_t n_knots, const int32_t* seeds, const float* frequency,
                                const float* scalars, int32_t n_img, const int64_t* origins, int32_t h, int32_t w,
                                const float* input, int32_t mode, const float* const* imp_values,
                                const int64_t* imp_boxes, const float* imp_defaults, uint32_t imp_has_default,
                                float* out, void* stream) {
  TDX_REQUIRE(out, "synthetic_map: null output");
  TDX_REQUIRE((mode & ~(TDX_SYNTH_FINALIZE | TDX_SYNTH_SQRT0 | TDX_SYNTH_IMPORT | TDX_SYNTH_RAW_INPUT)) == 0,
              "synthetic_map: unknown mode bits 0x%x", (unsigned)mode);
  const bool raw_input = mode & TDX_SYNTH_RAW_INPUT;
  TDX_REQUIRE(!raw_input || input, "synthetic_map: TDX_SYNTH_RAW_INPUT without an input");
  TDX_REQUIRE(raw_input || (tables && n_knots >= 2 && n_knots <= TDX_SYNTH_MAX_KNOTS),
              "synthetic_map: tables missing or %d knots (2..%d allowed)", (int)n_knots, TDX_SYNTH_MAX_KNOTS);
  TDX_REQUIRE(input || (seeds && frequency), "synthetic_map: no input and no seeds / frequencies");
  TDX_REQUIRE(!(mode & TDX_SYNTH_FINALIZE) || scalars, "synthetic_map: TDX_SYNTH_FINALIZE without scalars");
  TDX_REQUIRE(!(mode & TDX_SYNTH_IMPORT) || (imp_values && imp_boxes && (imp_defaults || imp_has_default == 0)),
              "synthetic_map: TDX_SYNTH_IMPORT without the import tables");
  TDX_REQUIRE((imp_has_default & ~0x1Fu) == 0, "synthetic_map: default bits 0x%x, 5 channels", (unsigned)imp_has_default);
  int rc = check_window(h, w, "synthetic_map");
  if (rc != TDX_OK) return rc;
  SynthOrigins org{};
  for (int k = 0; k < n_img; ++k) {
    const int64_t i0 = origins[2 * k], j0 = origins[2 * k + 1];
    TDX_REQUIRE(i0 > -(1LL << 62) && i0 < (1LL << 62) && j0 > -(1LL << 62) && j0 < (1LL << 62),
                "synthetic_map: window origin out of range");
    org.i0[k] = (long long)i0;
    org.j0[k] = (long long)j0;
  }
  SynthParams p{};
  for (int f = 0; f < kFields && !input; ++f) {
    p.seed[f] = seeds[f];
    p.frequency[f] = frequency[f];
  }
  if (mode & TDX_SYNTH_FINALIZE) {
    p.a = scalars[0];
    p.b = scalars[1];
    p.p1 = scalars[2];
    p.p99 = scalars[3];
    p.span = scalars[4];
  }
  SynthImports imp{};
  if (mode & TDX_SYNTH_IMPORT) {
    for (int f = 0; f < kFields; ++f) {
      imp.values[f] = imp_values[f];
      imp.oi[f] = imp_boxes[4 * f];
      imp.oj[f] = imp_boxes[4 * f + 1];
      TDX_REQUIRE(!imp_values[f] || (imp_boxes[4 * f + 2] >= 1 && imp_boxes[4 * f + 3] >= 1 &&
                                     imp_boxes[4 * f + 2] <= (1 << 30) && imp_boxes[4 * f + 3] <= (1 << 30)),
                  "synthetic_map: import %d has a bad shape", f);
      imp.rows[f] = (int)imp_boxes[4 * f + 2];
      imp.cols[f] = (int)imp_boxes[4 * f + 3];
      imp.deflt[f] = ((imp_has_default >> f) & 1u) ? imp_defaults[f] : 0.f;
    }
    imp.has_default = imp_has_default;
  }
  const size_t smem = (raw_input ? 0 : 2 * kFields * (size_t)n_knots * sizeof(double)) + 256 * sizeof(float);
  TDX_CHECK_CUDA(launch(synth_kernel, dim3((unsigned)(((long)h * w + kThreads - 1) / kThreads), (unsigned)n_img),
                        kThreads, smem, stream, p, imp, tables, raw_input ? 0 : (int)n_knots, org, (int)h, (int)w, input,
                        (int)mode, out));
  return TDX_OK;
}

extern "C" int tdx_synthetic_map(const double* tables, int32_t n_knots, const int32_t* seeds, const float* frequency,
                                 const float* scalars, int64_t i0, int64_t j0, int32_t h, int32_t w, const float* input,
                                 int32_t mode, const float* const* imp_values, const int64_t* imp_boxes,
                                 const float* imp_defaults, uint32_t imp_has_default, float* out, void* stream) {
  const int64_t origin[2] = {i0, j0};
  return synthetic_map_launch(tables, n_knots, seeds, frequency, scalars, 1, origin, h, w, input, mode, imp_values,
                              imp_boxes, imp_defaults, imp_has_default, out, stream);
}

extern "C" int tdx_synthetic_maps(const double* tables, int32_t n_knots, const int32_t* seeds, const float* frequency,
                                  const float* scalars, int32_t n_img, const int64_t* origins, int32_t h, int32_t w,
                                  int32_t mode, const float* const* imp_values, const int64_t* imp_boxes,
                                  const float* imp_defaults, uint32_t imp_has_default, float* out, void* stream) {
  TDX_REQUIRE(n_img >= 1 && n_img <= TDX_SYNTH_MAX_IMAGES, "synthetic_maps: %d windows, 1..%d allowed", (int)n_img,
              TDX_SYNTH_MAX_IMAGES);
  TDX_REQUIRE(origins, "synthetic_maps: null origins");
  TDX_REQUIRE(!(mode & TDX_SYNTH_RAW_INPUT), "synthetic_maps: TDX_SYNTH_RAW_INPUT is not batched");
  return synthetic_map_launch(tables, n_knots, seeds, frequency, scalars, n_img, origins, h, w, nullptr, mode,
                              imp_values, imp_boxes, imp_defaults, imp_has_default, out, stream);
}
