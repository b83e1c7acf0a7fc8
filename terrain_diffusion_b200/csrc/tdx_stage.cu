// Elementwise glue of the consistency stages of the product pipeline (fp32, HBM-bound, float4 where the shape allows):
// what the reference does with a dozen small torch ops per tile around the U-Net
// (inference/world_pipeline.py:1097-1098,1128-1131,1223-1226,1235-1242).
#include "tdx_common.h"

namespace tdx {

// x_t = a * sample + b * noise   (TrigFlow re-noising: a = cos t, b = sin t * sigma_data; sample == nullptr: 0)
__global__ void trig_mix_kernel(float* out, const float* sample, const float* noise, int64_t n, float a, float b) {
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (; i + 3 < n; i += stride) {
    const float4 z = *reinterpret_cast<const float4*>(noise + i);
    float4 s = sample ? *reinterpret_cast<const float4*>(sample + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    s.x = __fadd_rn(__fmul_rn(a, s.x), __fmul_rn(b, z.x));
    s.y = __fadd_rn(__fmul_rn(a, s.y), __fmul_rn(b, z.y));
    s.z = __fadd_rn(__fmul_rn(a, s.z), __fmul_rn(b, z.z));
    s.w = __fadd_rn(__fmul_rn(a, s.w), __fmul_rn(b, z.w));
    *reinterpret_cast<float4*>(out + i) = s;
  }
}

// out[img][c] = x[img][c] * scale * w ; out[img][C] = w        (packed window output cat([x*w, w]))
__global__ void pack_weighted_kernel(float* out, const float* x, const float* w, int channels, int64_t plane,
                                     float scale) {
  const int img = blockIdx.y;
  const float* xi = x + (size_t)img * channels * plane;
  float* oi = out + (size_t)img * (channels + 1) * plane;
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (; i + 3 < plane; i += stride) {
    const float4 ww = *reinterpret_cast<const float4*>(w + i);
    for (int c = 0; c < channels; ++c) {
      float4 v = *reinterpret_cast<const float4*>(xi + (size_t)c * plane + i);
      v.x = __fmul_rn(__fmul_rn(v.x, scale), ww.x);
      v.y = __fmul_rn(__fmul_rn(v.y, scale), ww.y);
      v.z = __fmul_rn(__fmul_rn(v.z, scale), ww.z);
      v.w = __fmul_rn(__fmul_rn(v.w, scale), ww.w);
      *reinterpret_cast<float4*>(oi + (size_t)c * plane + i) = v;
    }
    *reinterpret_cast<float4*>(oi + (size_t)channels * plane + i) = ww;
  }
}

// cond[img][c][Y][X] = packed[img][c][Y/f][X/f] / packed[img][last][Y/f][X/f]   for c < keep: normalise-on-read of a
// packed (sum x*w, sum w) window + nearest-neighbour upsampling by f, one pass
__global__ void window_to_cond_kernel(float* out, const float* packed, int packed_ch, int keep, int h, int w, int f) {
  const int img = blockIdx.z, c = blockIdx.y;
  const int H = h * f, W = w * f;
  const float* pv = packed + ((size_t)img * packed_ch + c) * h * w;
  const float* pw = packed + ((size_t)img * packed_ch + packed_ch - 1) * h * w;
  float* o = out + ((size_t)img * keep + c) * H * W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < H * W; i += gridDim.x * blockDim.x) {
    const int Y = i / W, X = i - Y * W;
    const int s = (Y / f) * w + X / f;
    o[i] = __fdiv_rn(pv[s], pw[s]);
  }
}

// Coarse-tile epilogue (world_pipeline.py:948-958), one block per (channel, image):
//   v = x / sigma_data * std[c] + mean[c];  v[1] = v[0] - v[1];  pool by n;  out = cat([v w, w]).
// The block de-normalises its whole plane into shared memory in parallel, then each thread reduces one pooled cell
// (a thread per cell reading the solve output directly serialises n^2 divisions and global loads: 140 us at n = 16 on
// an H100 80GB HBM3 at 700 W).
// Each operation rounds as the reference's separate fp32 CPU ops do: a true division, no FMA contraction.  Pooling is
// torch's CPU arithmetic: avg is the row-major sum from +0 divided once by n*n; max starts at -inf and takes a value
// that is greater or NaN (NaN propagates, the first of equal values -- +-0 included -- is kept); min is -max(-x).
// At n == 1 the reference does not pool at all (an avg would turn -0 into +0), so neither does this kernel.
enum : int { POOL_AVG = 0, POOL_MAX = 1, POOL_MIN = 2 };
constexpr int COARSE_CH = 6, COARSE_EPI_MAX_SIZE = 64, COARSE_EPI_THREADS = 256;

__device__ __forceinline__ float coarse_denorm(float x, float sigma_data, float sd, float mean) {
  return __fadd_rn(__fmul_rn(__fdiv_rn(x, sigma_data), sd), mean);
}

__global__ void __launch_bounds__(COARSE_EPI_THREADS)
coarse_epilogue_kernel(float* out, const float* x, const float* means, const float* stds, const float* w, int size,
                       int pool, int elev_mode, int p5_mode, float sigma_data) {
  __shared__ float v[COARSE_EPI_MAX_SIZE * COARSE_EPI_MAX_SIZE];
  const int c = blockIdx.x, img = blockIdx.y;
  const int in_plane = size * size;
  const float* xi = x + (size_t)img * COARSE_CH * in_plane;
  const float mean = means[c], sd = stds[c];
  for (int s = threadIdx.x; s < in_plane; s += blockDim.x) {
    float vc = coarse_denorm(xi[(size_t)c * in_plane + s], sigma_data, sd, mean);
    if (c == 1) vc = __fsub_rn(coarse_denorm(xi[s], sigma_data, stds[0], means[0]), vc);   // predicted as ch0 - ch1
    v[s] = vc;
  }
  __syncthreads();
  const int mode = c == 0 ? elev_mode : c == 1 ? p5_mode : POOL_AVG;
  const int osz = size / pool, plane = osz * osz;
  float* oi = out + (size_t)img * (COARSE_CH + 1) * plane;
  for (int p = threadIdx.x; p < plane; p += blockDim.x) {
    const int oy = p / osz, ox = p - oy * osz;
    const float* cell = v + oy * pool * size + ox * pool;
    float r;
    if (pool == 1) {
      r = cell[0];
    } else if (mode == POOL_AVG) {
      r = 0.f;
      for (int dy = 0; dy < pool; ++dy)
        for (int dx = 0; dx < pool; ++dx) r = __fadd_rn(r, cell[dy * size + dx]);
      r = __fdiv_rn(r, (float)(pool * pool));
    } else {
      const bool neg = mode == POOL_MIN;
      r = -INFINITY;
      for (int dy = 0; dy < pool; ++dy) {
        for (int dx = 0; dx < pool; ++dx) {
          const float u = neg ? -cell[dy * size + dx] : cell[dy * size + dx];
          if (u > r || isnan(u)) r = u;
        }
      }
      if (neg) r = -r;
    }
    const float ww = w[p];
    oi[(size_t)c * plane + p] = __fmul_rn(r, ww);
    if (c == 0) oi[(size_t)COARSE_CH * plane + p] = ww;
  }
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_trig_mix(float* out, const float* sample, const float* noise, int64_t numel, float a, float b,
                            void* stream) {
  TDX_REQUIRE(out && noise && numel > 0 && numel % 4 == 0, "trig_mix: bad arguments (numel must be a multiple of 4)");
  TDX_REQUIRE(((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(noise) |
                reinterpret_cast<uintptr_t>(sample)) & 15) == 0, "trig_mix: pointers must be 16-byte aligned");
  int blocks = (int)((numel / 4 + 255) / 256);
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  trig_mix_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(out, sample, noise, numel, a, b);
  TDX_CHECK_CUDA(cudaGetLastError());
  return TDX_OK;
}

extern "C" int tdx_pack_weighted(float* out, const float* x, const float* w, int32_t n_img, int32_t channels,
                                 int64_t plane, float scale, void* stream) {
  TDX_REQUIRE(out && x && w && n_img >= 1 && channels >= 1 && plane > 0 && plane % 4 == 0,
              "pack_weighted: bad arguments (plane must be a multiple of 4)");
  TDX_REQUIRE(((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15) == 0,
              "pack_weighted: pointers must be 16-byte aligned");
  int bx = (int)((plane / 4 + 255) / 256);
  if (bx > sm_count() * 4) bx = sm_count() * 4;
  pack_weighted_kernel<<<dim3(bx, n_img), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(out, x, w, channels, plane,
                                                                                            scale);
  TDX_CHECK_CUDA(cudaGetLastError());
  return TDX_OK;
}

extern "C" int tdx_window_to_cond(float* out, const float* packed, int32_t n_img, int32_t packed_channels, int32_t keep,
                                  int32_t h, int32_t w, int32_t factor, void* stream) {
  TDX_REQUIRE(out && packed && n_img >= 1 && packed_channels >= 2 && keep >= 1 && keep < packed_channels && h >= 1 &&
              w >= 1 && factor >= 1, "window_to_cond: bad arguments");
  int bx = (h * factor * w * factor + 255) / 256;
  if (bx > 1024) bx = 1024;
  window_to_cond_kernel<<<dim3(bx, keep, n_img), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      out, packed, packed_channels, keep, h, w, factor);
  TDX_CHECK_CUDA(cudaGetLastError());
  return TDX_OK;
}

extern "C" int tdx_coarse_epilogue(float* out, const float* x, const float* means, const float* stds, const float* w,
                                   int32_t n_img, int32_t size, int32_t pool, int32_t elev_mode, int32_t p5_mode,
                                   float sigma_data, void* stream) {
  TDX_REQUIRE(out && x && means && stds && w, "coarse_epilogue: null pointer");
  TDX_REQUIRE(n_img >= 1 && n_img <= 65535 && size >= 1 && size <= COARSE_EPI_MAX_SIZE && pool >= 1 &&
              size % pool == 0,
              "coarse_epilogue: bad shape (need 1 <= n_img <= 65535, 1 <= size <= 64, pool >= 1 dividing size)");
  TDX_REQUIRE(elev_mode >= POOL_AVG && elev_mode <= POOL_MIN && p5_mode >= POOL_AVG && p5_mode <= POOL_MIN,
              "coarse_epilogue: pool modes must be 0 (avg), 1 (max) or 2 (min)");
  coarse_epilogue_kernel<<<dim3(COARSE_CH, n_img), COARSE_EPI_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      out, x, means, stds, w, size, pool, elev_mode, p5_mode, sigma_data);
  TDX_CHECK_CUDA(cudaGetLastError());
  return TDX_OK;
}
