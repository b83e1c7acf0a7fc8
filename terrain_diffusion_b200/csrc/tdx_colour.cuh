// Device pieces of matplotlib's colour pipeline shared by the explorer's detail view (tdx_explorer.cu) and its coarse
// map (tdx_coarse_view.cu): the order-preserving keys of the NaN-ignoring range buffers, Normalize + Colormap's index
// rule with the range read from such a buffer, and ScalarMappable.to_rgba(bytes=True)'s 8-bit step.
#pragma once
#include <cuda_runtime.h>

namespace tdx {

constexpr int kColourLut = 256;   // rcParams['image.lut']

// A float's bits mapped to an unsigned key that orders like the float (-inf < ... < -0 < +0 < ... < +inf), never 0.
__device__ __forceinline__ unsigned ordered_key(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ScalarMappable.to_rgba(bytes=True) of one fp32 channel in [0, 1]: uint8(trunc(fp32(x * 255))).
__device__ __forceinline__ unsigned quantise(float c) { return (unsigned)__fmul_rn(c, 255.f); }
__device__ __forceinline__ float clip01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }   // keeps NaN

// The table entry that Normalize(vmin, vmax) + Colormap pick for x, or -1 for the bad colour (0, 0, 0, 0).  `range` is
// a {~key(nanmin), key(nanmax)} pair (both 0 when every value was NaN): vmin, vmax = float(nanmin), float(nanmax), NaN
// when empty, and vmax = vmin + 1 in fp64 when equal.  Normalize fills 0 when vmin == vmax still (|vmin| >= 2^53 or
// inf), NaN x included; otherwise `resdat -= vmin; resdat /= (vmax - vmin)` run in fp64 and round once into the fp32
// array (NEP 50: the float64 scalars promote them).  Colormap: x*N in fp32, N -> N-1, under -> first, over -> last,
// NaN -> bad.
__device__ __forceinline__ int colour_index(float x, const unsigned* __restrict__ range) {
  const float fnan = __int_as_float(0x7fc00000);
  const double vmin = range[1] ? (double)key_to_float(~range[0]) : (double)fnan;
  double vmax = range[1] ? (double)key_to_float(range[1]) : (double)fnan;
  if (vmax == vmin) vmax = __dadd_rn(vmin, 1.0);
  float t;
  if (vmin == vmax) {
    t = 0.f;
  } else {
    const float r = __double2float_rn(__dsub_rn((double)x, vmin));
    t = __double2float_rn(__ddiv_rn((double)r, __dsub_rn(vmax, vmin)));
  }
  float xa = __fmul_rn(t, (float)kColourLut);
  if (xa == (float)kColourLut) xa = (float)(kColourLut - 1);
  if (isnan(xa)) return -1;
  return xa < 0.f ? 0 : (xa >= (float)kColourLut ? kColourLut - 1 : (int)xa);
}

}  // namespace tdx
