// The int16 elevation packing of the HTTP read-outs, and torch's CPU upsample_bilinear2d (align_corners=False, integer
// scale factor given) evaluated at one output pixel of the upsampled window, bit for bit.  Shared by the terrain API read-out (tdx_post.cu) and the Minecraft API read-out
// (tdx_biome.cu).  torch picks one of two CPU kernels by the size of the WHOLE upsampled window (ATen
// UpSampleKernel.cpp, _use_vectorized_kernel_cond_2d: out_h + out_w <= 128 picks the per-pixel-weight kernel), and the
// two round differently; both are restated here operation for operation (fma = the contraction x86 builds do):
//   per axis:  src = max(fma(r, d + 0.5, -0.5), 0), r = fp32(1/scale);  i0 = min(floor(src), n-1), i1 = i0 + (i0 < n-1);
//              l1 = clamp(src - i0, 0, 1), l0 = 1 - l1
//   wide  (separable):   t_a = fma(wl0, x[a][j0], wl1 * x[a][j1]);  out = fma(hl0, t_i0, hl1 * t_i1)
//   small (out_h + out_w <= 128):  w_ab = hl_a * wl_b;  out = fma(w11, x11, fma(w10, x10, fma(w00, x00, w01 * x01)))
#pragma once

namespace tdx {

// api.py:73-77 (and minecraft_api.py:83-87): floor, clip, '<i2'.  numpy's clip keeps a NaN and its cast to int16 gives
// 0 on x86 (fmaxf would drop the NaN and pack -32768), so NaN packs as 0; +-inf clip to 32767 / -32768.
__device__ __forceinline__ int16_t elev_to_i16(float v) {
  const float f = v != v ? 0.f : fminf(fmaxf(floorf(v), -32768.f), 32767.f);
  return (int16_t)f;
}

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

// One plane f [.][w] at the output pixel with taps (ty, tx); `small` selects the per-pixel-weight kernel.
__device__ __forceinline__ float bilinear_at(const float* f, int w, const AxisTap& ty, const AxisTap& tx, bool small) {
  const long r0 = (long)ty.i0 * w, r1 = (long)ty.i1 * w;
  const float x00 = f[r0 + tx.i0], x01 = f[r0 + tx.i1], x10 = f[r1 + tx.i0], x11 = f[r1 + tx.i1];
  if (small) {
    const float w00 = __fmul_rn(ty.l0, tx.l0), w01 = __fmul_rn(ty.l0, tx.l1);
    const float w10 = __fmul_rn(ty.l1, tx.l0), w11 = __fmul_rn(ty.l1, tx.l1);
    return __fmaf_rn(w11, x11, __fmaf_rn(w10, x10, __fmaf_rn(w00, x00, __fmul_rn(w01, x01))));
  }
  const float t0 = __fmaf_rn(tx.l0, x00, __fmul_rn(tx.l1, x01));
  const float t1 = __fmaf_rn(tx.l0, x10, __fmul_rn(tx.l1, x11));
  return __fmaf_rn(ty.l0, t0, __fmul_rn(ty.l1, t1));
}

}  // namespace tdx
