// The Minecraft API's read-out (inference/minecraft_api.py: _get_upsampled :265-355, _compute_climate_vars :189-263,
// _classify_biome :358-688, _binary_response :90-99) in one launch, thread per output pixel.  The reference runs it on
// the host after get(): torch's CPU bilinear upsample of a native window padded by 2 pixels, a Sobel slope over a
// 1-pixel ring, optional slope-scaled "detail" noise, and a rule-based classifier written as ~150 full-frame mask
// operations with "last write wins".  Here every pixel evaluates its own 3x3 neighbourhood of the upsampled window and
// one decision function that yields what the mask chain leaves behind, quirks included.
//
// The 9 elevation samples of a pixel are recomputed from the native window rather than staged as a halo in shared
// memory: the native window is a few KB and stays in L1/L2, each sample is 4 loads and 3 fused ops, and recomputing
// keeps the small/separable kernel choice and the scale-1 two-window case free of any tiling logic.
//
// Rounding follows the reference's torch / numpy ops one by one: every torch op rounds to fp32 (Python scalars are cast
// to fp32 at each op; comparisons are against fp32(c)), numpy 2 keeps fp32 arrays fp32 under Python scalars (NEP 50),
// so nothing here is contracted except where torch's bilinear kernels themselves fuse (tdx_upsample.cuh).  asin and
// pow(., 1.5) are not correctly rounded in torch (Sleef) nor here (CUDA asinf / powf); tests bound their effect.
#include "tdx_common.h"
#include "tdx_ptx.cuh"
#include "tdx_upsample.cuh"

namespace tdx {

struct McParams {
  const float* elev;      // [h][w]: scale >= 2 the native window padded by 2; scale 1 the slope window [H+2][W+2]
  const float* centre;    // scale 1: [H][W], the pixel's own elevation (the second get()); NULL for scale >= 2
  const float* climate;   // scale >= 2: [5][h][w] native; scale 1: [5][H][W]; NULL: every pixel is plains
  const float* noise;     // [5][H][W]: temp/snow coarse, temp/snow fine, precip, elev coarse, elev fine
  float* elev_out;        // [H][W] or NULL
  float* smooth_out;      // [H][W] or NULL
  float* climate_out;     // [5][H][W] or NULL
  int16_t* biome_out;     // [H][W] or NULL
  uint16_t* payload;      // H*W int16 elevation + H*W int16 biome ids, as 16-bit words, or NULL
  int h, w, scale, oi, oj, H, W, small, sobel_small, detail;
  float r, amp_c, amp_f, psm, native_res, slope_div;
};

// torch.clamp: NaN stays NaN (fminf / fmaxf alone would drop it).
__device__ __forceinline__ float clamp_nan(float v, float lo, float hi) { return v != v ? v : fminf(fmaxf(v, lo), hi); }
__device__ __forceinline__ float clamp_min_nan(float v, float lo) { return v != v ? v : fmaxf(v, lo); }
__device__ __forceinline__ float clamp_max_nan(float v, float hi) { return v != v ? v : fminf(v, hi); }

// torch's CPU conv2d of the 3x3 Sobel taps over a 1-channel window (products are exact: the taps are 0, +-1/8, +-1/4,
// so only the order of the additions matters).  Measured on torch 2.11 (x86, AVX512 dispatch):
//   input numel > 20480 (oneDNN):            ((((p0 + p1) + p2) + ... ) + p8), from 0, row-major
//   otherwise (im2col + MKL gemm, K = 9), by the pixel's flat index n in the H*W output:
//     n < N - N % 16:  ((p0 + p2) + (p1 + p3)) + ((p4 + p6) + (p5 + p7)), then + p8
//     the N % 16 tail: row-major sequential as above
//     N == 1:          v_j = p_j + p_{j+4};  v0 + ((v1 + v3) + (v2 + p8))
enum { SOBEL_SEQ = 0, SOBEL_PAIR = 1, SOBEL_ONE = 2 };
__device__ __forceinline__ float sobel9(const float* v, const float* k, int order) {
  float p[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) p[i] = __fmul_rn(k[i], v[i]);
  if (order == SOBEL_PAIR) {
    const float a = __fadd_rn(__fadd_rn(p[0], p[2]), __fadd_rn(p[1], p[3]));
    const float b = __fadd_rn(__fadd_rn(p[4], p[6]), __fadd_rn(p[5], p[7]));
    return __fadd_rn(__fadd_rn(a, b), p[8]);
  }
  if (order == SOBEL_ONE) {
    const float v0 = __fadd_rn(p[0], p[4]), v1 = __fadd_rn(p[1], p[5]);
    const float v2 = __fadd_rn(p[2], p[6]), v3 = __fadd_rn(p[3], p[7]);
    return __fadd_rn(v0, __fadd_rn(__fadd_rn(v1, v3), __fadd_rn(v2, p[8])));
  }
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 9; ++i) acc = __fadd_rn(acc, p[i]);
  return acc;
}

enum : int16_t {
  B_PLAINS = 1, B_SNOWY_PLAINS = 3, B_DESERT = 5, B_SWAMP = 6, B_FOREST = 8, B_TAIGA = 15, B_SNOWY_TAIGA = 16,
  B_SAVANNA = 17, B_WINDSWEPT_HILLS = 19, B_JUNGLE = 23, B_GROVE = 31, B_SNOWY_SLOPES = 32, B_FROZEN_PEAKS = 33,
  B_STONY_PEAKS = 35, B_FOREST_SPARSE = 108, B_TAIGA_SPARSE = 115, B_SNOWY_TAIGA_SPARSE = 116,
  B_WARM_OCEAN = 41, B_OCEAN = 44, B_COLD_OCEAN = 46, B_FROZEN_OCEAN = 48
};

// What _classify_biome's mask chain (:525-686) leaves in one pixel.  e: the classified elevation (elev_smooth), temp /
// precip: the noised climate, snow_t: temp + snow noise.  Every comparison is false on NaN, as the masks are.
__device__ int16_t classify(float e, float temp, float precip, float tm, float gs, bool tropical, float sr,
                            float snow_t) {
  const bool ocean = e < 0.0f;
  const bool frozen = temp < -5.0f, cold = temp >= -5.0f && temp < 5.0f, cool = temp >= 5.0f && temp < 12.0f;
  const bool temperate = temp >= 12.0f && temp < 20.0f, warm = temp >= 20.0f && temp < 26.0f, hot = temp >= 26.0f;
  if (ocean) return frozen ? B_FROZEN_OCEAN : cold ? B_COLD_OCEAN : (warm || hot) ? B_WARM_OCEAN : B_OCEAN;

  const float gs_factor = clamp_nan(__fdiv_rn(__fsub_rn(gs, 60.0f), 90.0f), 0.0f, 1.0f);
  const float eff = __fmul_rn(tm, gs_factor);
  const float mf = clamp_nan(__fdiv_rn(__fsub_rn(tm, 0.35f), 0.45f), 0.0f, 1.0f);
  const float bare_t = __fadd_rn(0.7f, __fmul_rn((float)(1.19 - 0.7), mf));
  const bool slope_medium = sr >= 0.62f && sr < bare_t;
  const bool slope_bare = sr >= bare_t;
  const bool has_snow = snow_t < 0.0f && precip > 150.0f && !(sr > 0.78f);
  // The bare-slope override (:684-686) runs last over every non-ocean pixel; mountains (:552-556) give the same ids.
  if (slope_bare) return has_snow ? B_FROZEN_PEAKS : B_STONY_PEAKS;

  // tree classes (:466-499) without the bare-slope demotion, which cannot apply past the return above.  A NaN eff is
  // in none of them.
  const bool none0 = eff < 0.2f;
  const bool had_trees = !none0 && eff >= 0.5f;
  const bool none = none0;
  const bool sparse = (!none0 && eff < 0.5f) || (slope_medium && had_trees);
  const bool forest = !none0 && eff >= 0.5f && eff < 0.8f && !slope_medium;
  const bool dense = !none0 && eff >= 0.8f && eff < 1.3f && !slope_medium;
  const bool rain = !none0 && eff >= 1.3f && !slope_medium;
  const bool barren = tm < 0.05f || gs < 60.0f;
  const bool steppe = tm < 0.35f || precip < 350.0f;

  const float alt = clamp_min_nan(e, 0.0f);
  if (alt > 2500.0f) {                                     // mountains (:549-590), no slope_bare here
    if (has_snow) {
      if (none) return B_SNOWY_SLOPES;
      if (sparse || forest) return B_SNOWY_TAIGA_SPARSE;
      if (dense || rain) return B_SNOWY_TAIGA;
      return B_PLAINS;
    }
    if (none) return barren ? B_WINDSWEPT_HILLS : steppe ? B_GROVE : B_PLAINS;
    if (sparse || forest) return B_TAIGA_SPARSE;
    if (dense || rain) return B_TAIGA;
    return B_PLAINS;
  }
  const bool lowland = alt < 200.0f;                       // false for a NaN elevation
  if (has_snow) {                                          // 3A / 3B; a snowy pixel in no tree class falls to 3I
    if (none) return B_SNOWY_PLAINS;
    if (sparse || forest) return B_SNOWY_TAIGA_SPARSE;
    if (dense || rain) return B_SNOWY_TAIGA;
    return B_PLAINS;
  }
  if (none) {                                              // 3D: cold_steppe is written after desert and wins
    if (steppe && !barren) return B_GROVE;
    if ((cold || cool || temperate) && !lowland && barren) return B_GROVE;
    if (warm || hot) return B_DESERT;
    return B_PLAINS;
  }
  if (sparse || forest) {                                  // 3E: no leaf for a slope-demoted warm sparse pixel
    if (hot) return B_JUNGLE;
    if (warm) return sparse ? (slope_medium ? B_PLAINS : B_SAVANNA) : B_FOREST_SPARSE;
    if (temperate) return B_FOREST_SPARSE;
    if (cool || cold) return B_TAIGA_SPARSE;
    return B_PLAINS;
  }
  if (dense) {                                             // 3G
    if (hot) return B_JUNGLE;
    if (warm && lowland) return B_SWAMP;
    if (cool || cold) return B_TAIGA;
    return B_FOREST;
  }
  if (rain) {                                              // 3H
    if (hot || (warm && tropical)) return B_JUNGLE;
    if (lowland) return B_SWAMP;
    if (cool || cold) return B_TAIGA;
    return B_FOREST;
  }
  return B_PLAINS;                                         // 3I
}

__global__ void minecraft_readout_kernel(const McParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.W || y >= p.H) return;
  const long o = (long)y * p.W + x, plane_out = (long)p.H * p.W;

  // 3x3 neighbourhood in the upsampled window (scale 1: the slope window itself)
  float nb[9];
  AxisTap ty[3], tx[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    if (p.scale == 1) {
      ty[d].i0 = ty[d].i1 = p.oi + y + d - 1;
      tx[d].i0 = tx[d].i1 = p.oj + x + d - 1;
    } else {
      ty[d] = upsample_axis(p.oi + y + d - 1, p.h, p.r);
      tx[d] = upsample_axis(p.oj + x + d - 1, p.w, p.r);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
      nb[a * 3 + b] = p.scale == 1 ? p.elev[(long)ty[a].i0 * p.w + tx[b].i0] : bilinear_at(p.elev, p.w, ty[a], tx[b], p.small);
  const float es = p.scale == 1 ? p.centre[o] : nb[4];

  const float kx[9] = {-0.125f, 0.f, 0.125f, -0.25f, 0.f, 0.25f, -0.125f, 0.f, 0.125f};
  const float ky[9] = {-0.125f, -0.25f, -0.125f, 0.f, 0.f, 0.f, 0.125f, 0.25f, 0.125f};
  int order = SOBEL_SEQ;
  if (p.sobel_small) {
    const long n = plane_out;
    order = n == 1 ? SOBEL_ONE : (o < n - n % 16 ? SOBEL_PAIR : SOBEL_SEQ);
  }
  const float sdx = sobel9(nb, kx, order), sdy = sobel9(nb, ky, order);
  const float grad = __fsqrt_rn(__fadd_rn(__fmul_rn(sdx, sdx), __fmul_rn(sdy, sdy)));

  const float* nz = p.noise;
  float e_out = es;
  if (p.detail) {                                          // :335-351
    const float sf = powf(clamp_nan(__fdiv_rn(grad, p.slope_div), 0.0f, 1.0f), 1.5f);
    const float ac = __fdiv_rn(__fmul_rn(__fmul_rn(p.amp_c, sf), p.psm), p.native_res);
    const float af = __fdiv_rn(__fmul_rn(__fmul_rn(p.amp_f, sf), p.psm), p.native_res);
    const float d = __fadd_rn(__fmul_rn(nz[3 * plane_out + o], ac), __fmul_rn(nz[4 * plane_out + o], af));
    e_out = __fadd_rn(es, __fmul_rn(d, es >= 0.0f ? 1.0f : 0.0f));
  }

  int16_t biome = B_PLAINS;
  if (p.climate) {
    float c[5];
    if (p.scale == 1) {
#pragma unroll
      for (int k = 0; k < 5; ++k) c[k] = p.climate[k * plane_out + o];
    } else {
      const long plane_in = (long)p.h * p.w;
#pragma unroll
      for (int k = 0; k < 5; ++k) c[k] = bilinear_at(p.climate + k * plane_in, p.w, ty[1], tx[1], p.small);
    }
    if (p.climate_out)
#pragma unroll
      for (int k = 0; k < 5; ++k) p.climate_out[k * plane_out + o] = c[k];
    // :393-407, numpy fp32
    const float n0 = nz[o], n1 = nz[plane_out + o], n2 = nz[2 * plane_out + o];
    const float temp = __fadd_rn(c[0], __fadd_rn(__fmul_rn(0.4f, n0), __fmul_rn(0.2f, n1)));
    const float precip = __fmul_rn(clamp_min_nan(c[2], 0.0f), __fadd_rn(1.0f, __fmul_rn(0.2f, n2)));
    const float snow = __fadd_rn(__fmul_rn(3.0f, n0), __fmul_rn(2.0f, n1));
    // _compute_climate_vars (:208-252)
    const float t_std = __fdiv_rn(c[1], 100.0f);
    const float t_eff = clamp_min_nan(__fadd_rn(temp, __fmul_rn(0.5f, t_std)), 0.0f);
    const float pet = clamp_min_nan(__fadd_rn(__fadd_rn(250.0f, __fmul_rn(25.0f, t_eff)),
                                              __fmul_rn(0.7f, __fmul_rn(t_eff, t_eff))), 250.0f);
    const float aridity = __fdiv_rn(precip, clamp_min_nan(pet, 1.0f));
    const float penalty = __fsub_rn(1.0f, __fmul_rn(0.35f, clamp_max_nan(__fdiv_rn(c[3], 100.0f), 1.0f)));
    const float tm = __fmul_rn(aridity, penalty);
    const float amplitude = __fmul_rn(t_std, 1.414f);
    const float xs = __fdiv_rn(__fsub_rn(5.0f, temp), clamp_min_nan(amplitude, 0.1f));
    const float gs = xs <= -1.0f ? 365.0f
                     : xs >= 1.0f ? 0.0f
                     : __fmul_rn(365.0f, __fsub_rn(0.5f, __fdiv_rn(asinf(clamp_nan(xs, -1.0f, 1.0f)), 3.14159f)));
    const bool tropical = temp >= 18.0f && t_std < 5.0f;
    biome = classify(es, temp, precip, tm, gs, tropical, __fdiv_rn(grad, p.psm), __fadd_rn(temp, snow));
  }

  if (p.elev_out) p.elev_out[o] = e_out;
  if (p.smooth_out) p.smooth_out[o] = es;
  if (p.biome_out) p.biome_out[o] = biome;
  if (p.payload) {
    p.payload[o] = (uint16_t)elev_to_i16(e_out);
    p.payload[plane_out + o] = (uint16_t)biome;
  }
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_minecraft_readout(const float* elev, int32_t h, int32_t w, int32_t scale, int32_t oi, int32_t oj,
                                     const float* centre, const float* climate, const float* noise, int32_t H,
                                     int32_t W, int32_t detail, float amp_c, float amp_f, float pixel_size_m,
                                     float native_res, float slope_div, float* elev_out, float* smooth_out,
                                     float* climate_out, int16_t* biome_out, void* payload, void* stream) {
  TDX_REQUIRE(elev && (elev_out || smooth_out || climate_out || biome_out || payload),
              "minecraft_readout: null elevation or no output");
  TDX_REQUIRE(!climate_out || climate, "minecraft_readout: climate_out without a climate window");
  TDX_REQUIRE(noise || (!climate && !detail), "minecraft_readout: noise planes are needed");
  TDX_REQUIRE(((uintptr_t)payload & 1) == 0 && ((uintptr_t)biome_out & 1) == 0,
              "minecraft_readout: payload / biome_out must be 2-byte aligned");
  TDX_REQUIRE(scale >= 1 && h >= 3 && w >= 3 && H >= 1 && W >= 1 && H <= 65535,
              "minecraft_readout: bad shape %d x %d x%d -> %d x %d", h, w, scale, H, W);
  TDX_REQUIRE(oi >= 1 && oj >= 1 && (int64_t)oi + H + 1 <= (int64_t)h * scale && (int64_t)oj + W + 1 <= (int64_t)w * scale,
              "minecraft_readout: crop %d x %d at (%d, %d) and its 1-pixel ring outside the %d x %d upsampled window", H, W,
              oi, oj, h * scale, w * scale);
  TDX_REQUIRE(scale == 1 ? (centre && oi == 1 && oj == 1 && h == H + 2 && w == W + 2 && !detail) : !centre,
              "minecraft_readout: scale 1 takes the [H+2][W+2] slope window at (1, 1), the [H][W] centre window and no "
              "detail noise; scale >= 2 takes no centre window");
  McParams p;
  p.elev = elev; p.centre = centre; p.climate = climate; p.noise = noise;
  p.elev_out = elev_out; p.smooth_out = smooth_out; p.climate_out = climate_out; p.biome_out = biome_out;
  p.payload = static_cast<uint16_t*>(payload);
  p.h = h; p.w = w; p.scale = scale; p.oi = oi; p.oj = oj; p.H = H; p.W = W;
  p.small = ((int64_t)h + w) * scale <= 128;                  // the whole upsampled window, padded by 2 native pixels
  p.sobel_small = ((int64_t)H + 2) * (W + 2) <= 20480;        // conv2d's input is the crop plus its 1-pixel ring
  p.detail = detail != 0;
  p.r = (float)(1.0 / scale);
  p.amp_c = amp_c; p.amp_f = amp_f; p.psm = pixel_size_m; p.native_res = native_res; p.slope_div = slope_div;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3((W + 127) / 128, H), dim3(128), 0, reinterpret_cast<cudaStream_t>(stream));
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, minecraft_readout_kernel, p));
  return TDX_OK;
}
