// The explorer's coarse map (terrain_diffusion/inference/explorer/server.py:58-185) and the random sampler's land search
// (inference/random_sampler.py:61-119).  The reference copies the coarse canvas to the host once per channel it reads
// (`_coarse_channel`, up to six times per request) and runs numpy / matplotlib there; the sampler slides its window over
// the land mask in a Python double loop.  Here:
//   tdx_coarse_readout  (sum v*w, sum w) -> the six real-unit planes and channel 4's display plane, and the NaN-ignoring
//                       min / max of all seven into a small device buffer, in one pass,
//   tdx_coarse_image    Normalize + colormap + the filter dimming + to_rgba(bytes=True) of one channel; it reads the
//                       range from the device buffer, so the image needs no host synchronisation before its copy,
//   tdx_coarse_round    np.round(x, 2) of the six planes,
//   tdx_coarse_land     the land fraction of every (2 half)^2 window, its threshold, and the row-major list of the
//                       windows that pass.
// Every fp32 / fp64 operation is explicitly rounded in the order numpy (NEP 50) or torch's CPU kernels perform it.
#include "tdx_colour.cuh"
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {
namespace {

constexpr int kChannels = 6;         // Elev, p5, Temp, T std, Precip, Precip CV
constexpr int kPlanes = 7;           // the six, then log1p(max(Precip, 0))
constexpr int kPrecip = 4;
constexpr int kCompactThreads = 1024;

// np.sign(x) * np.square(x) in fp32 (torch.sign * torch.square gives the same bits): +0 for either zero, NaN stays NaN.
__device__ __forceinline__ float signed_square(float x) {
  const float s = __fmul_rn(x, x);
  return x > 0.f ? s : (x < 0.f ? -s : (x == 0.f ? 0.f : x));
}

// server.py:113: np.log1p(np.maximum(x, 0)); np.maximum passes NaN and gives +0 for -0.  numpy's fp32 log1p is not
// correctly rounded (2 ulp off on some inputs); log1pf stays within 2 ulp of it and, on the benchmark's canvases, picks
// the same table entry on every cell, where the correctly rounded fp64 log1p does not.
__device__ __forceinline__ float precip_display(float x) { return log1pf(x > 0.f || isnan(x) ? x : 0.f); }

// server.py:60-64 (eps) / world_pipeline.py:269-274 + random_sampler.py:75-77 (no eps), one thread per cell.
// range[2p] = ~key(nanmin), range[2p+1] = key(nanmax) of plane p, atomicMax on a zeroed buffer as tdx_detail_range.
__global__ void coarse_readout_kernel(const float* __restrict__ sums, long n, int eps, float* __restrict__ planes,
                                      unsigned* __restrict__ range) {
  pdl_launch_dependents();
  pdl_wait();
  unsigned nmn[kPlanes], kmx[kPlanes];
#pragma unroll
  for (int p = 0; p < kPlanes; ++p) nmn[p] = kmx[p] = 0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    // torch CPU fp32: coarse[-1:] + 1e-8 adds the scalar rounded to fp32, then one fp32 division per channel
    const float w = eps ? __fadd_rn(sums[(long)kChannels * n + i], 1e-8f) : sums[(long)kChannels * n + i];
    float v[kPlanes];
#pragma unroll
    for (int c = 0; c < kChannels; ++c) {
      const float x = __fdiv_rn(sums[(long)c * n + i], w);
      v[c] = c <= 1 ? signed_square(x) : x;
    }
    v[kChannels] = precip_display(v[kPrecip]);
#pragma unroll
    for (int p = 0; p < kPlanes; ++p) {
      if (planes) planes[(long)p * n + i] = v[p];
      if (!isnan(v[p])) {
        const unsigned k = ordered_key(v[p]);
        nmn[p] = max(nmn[p], ~k);
        kmx[p] = max(kmx[p], k);
      }
    }
  }
#pragma unroll
  for (int p = 0; p < kPlanes; ++p) {
    for (int o = 16; o > 0; o >>= 1) {
      nmn[p] = max(nmn[p], __shfl_xor_sync(0xffffffffu, nmn[p], o));
      kmx[p] = max(kmx[p], __shfl_xor_sync(0xffffffffu, kmx[p], o));
    }
    if ((threadIdx.x & 31) == 0 && kmx[p]) {
      atomicMax(&range[2 * p], nmn[p]);
      atomicMax(&range[2 * p + 1], kmx[p]);
    }
  }
}

// The `ch{c}_min` / `ch{c}_max` bounds, already rounded to fp32 as numpy rounds a Python float compared with an fp32
// array; bit 2c of `active` enables lo[c], bit 2c+1 hi[c].
struct CoarseFilter {
  float lo[kChannels], hi[kChannels];
  unsigned active;
};

// server.py:112-139, one thread per cell.  The display plane's table entry (colour_index), the fp32 RGBA of the table
// (alpha 1; the bad colour (0, 0, 0, 0)), `rgba[~mask, :3] *= 0.3` in fp32 where a bound fails (NaN fails every bound),
// then _png_response's clip and to_rgba(bytes=True).
__global__ void coarse_image_kernel(const float* __restrict__ planes, long n, int channel,
                                    const unsigned* __restrict__ range, const float* __restrict__ lut, CoarseFilter f,
                                    uchar4* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = channel == kPrecip ? kChannels : channel;
  const int idx = colour_index(planes[(long)p * n + i], range + 2 * p);
  float r = 0.f, g = 0.f, b = 0.f, a = 0.f;
  if (idx >= 0) {
    r = lut[idx * 3 + 0];
    g = lut[idx * 3 + 1];
    b = lut[idx * 3 + 2];
    a = 1.f;
  }
  bool keep = true;
#pragma unroll
  for (int c = 0; c < kChannels; ++c) {
    const float x = planes[(long)c * n + i];
    if ((f.active >> (2 * c)) & 1u) keep = keep && x >= f.lo[c];
    if ((f.active >> (2 * c + 1)) & 1u) keep = keep && x <= f.hi[c];
  }
  if (!keep) {
    r = __fmul_rn(r, 0.3f);
    g = __fmul_rn(g, 0.3f);
    b = __fmul_rn(b, 0.3f);
  }
  out[i] = make_uchar4((unsigned char)quantise(clip01(r)), (unsigned char)quantise(clip01(g)),
                       (unsigned char)quantise(clip01(b)), (unsigned char)quantise(a));
}

// server.py:159: np.round(x, 2) on fp32 = multiply by 100 in fp32, rint, divide by 100 in fp32.
__global__ void coarse_round_kernel(const float* __restrict__ x, long n, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = __fdiv_rn(rintf(__fmul_rn(x[i], 100.f)), 100.f);
}

// random_sampler.py:79,90: per row i, the land count (elev_m > 0) of columns [jo, jo + 2 half) for every jo < wo.
__global__ void land_rows_kernel(const float* __restrict__ elev_m, int h, int w, int half, int wo,
                                 int* __restrict__ rows) {
  pdl_launch_dependents();
  pdl_wait();
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long)h * wo) return;
  const int i = (int)(t / wo), jo = (int)(t % wo);
  const float* row = elev_m + (long)i * w + jo;
  int count = 0;
  for (int k = 0; k < 2 * half; ++k) count += row[k] > 0.f;
  rows[t] = count;
}

// random_sampler.py:87-92: the window at (half + io, half + jo) sums rows [io, io + 2 half) of the row counts; its
// mean is torch's CPU fp32 mean of 0 / 1 values, sum / numel correctly rounded (the integer counts are exact), and
// `.item() >= min_land_frac` compares in fp64.  An empty window (half == 0) is 0 / 0 = NaN and never passes.
__global__ void land_mask_kernel(const int* __restrict__ rows, int ho, int wo, int half, double min_land_frac,
                                 uint8_t* __restrict__ mask) {
  pdl_launch_dependents();
  pdl_wait();
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long)ho * wo) return;
  const int io = (int)(t / wo), jo = (int)(t % wo);
  int count = 0;
  for (int k = 0; k < 2 * half; ++k) count += rows[(long)(io + k) * wo + jo];
  const float frac = __fdiv_rn((float)count, (float)(4 * half * half));
  mask[t] = (double)frac >= min_land_frac;
}

// The row-major compaction of mask[n]: list[0] = the number of set entries, list[1..] their indices in order.  One CTA
// walks the mask in chunks of 4 entries per thread, each chunk one block-wide exclusive scan.
__global__ void __launch_bounds__(kCompactThreads) land_compact_kernel(const uint8_t* __restrict__ mask, long n,
                                                                       int* __restrict__ list) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int warp_total[kCompactThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (long c0 = 0; c0 < n; c0 += 4L * kCompactThreads) {
    const long i0 = c0 + 4L * threadIdx.x;
    bool set[4];
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      set[k] = i0 + k < n && mask[i0 + k];
      cnt += set[k];
    }
    int incl = cnt;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) warp_total[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int s = warp_total[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      warp_total[lane] = s;                  // inclusive prefix over warps
    }
    __syncthreads();
    int pos = base + (warp ? warp_total[warp - 1] : 0) + incl - cnt;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (set[k]) list[1 + pos++] = (int)(i0 + k);
    base += warp_total[kCompactThreads / 32 - 1];
    __syncthreads();                         // warp_total is rewritten by the next chunk
  }
  if (threadIdx.x == 0) list[0] = base;
}

template <typename Kernel, typename... Args>
int launch_cells(Kernel kernel, long n, cudaStream_t stream, Args... args) {   // one thread per cell, 256 per block
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream);
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
  return TDX_OK;
}

}  // namespace
}  // namespace tdx

using namespace tdx;

extern "C" int tdx_coarse_readout(const float* sums, int64_t n, int32_t eps, float* planes, uint32_t* range,
                                  void* stream) {
  TDX_REQUIRE(sums && range, "coarse_readout: null pointer");
  TDX_REQUIRE(n >= 1, "coarse_readout: empty input");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TDX_CHECK_CUDA(cudaMemsetAsync(range, 0, 2 * kPlanes * sizeof(uint32_t), st));
  const long blocks = (n + 255) / 256;
  const int grid = (int)(blocks < 4L * sm_count() ? blocks : 4L * sm_count());
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3(grid), dim3(256), 0, st);
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, coarse_readout_kernel, sums, (long)n, (int)(eps != 0), planes,
                                    reinterpret_cast<unsigned*>(range)));
  return TDX_OK;
}

extern "C" int tdx_coarse_image(const float* planes, int64_t n, int32_t channel, const uint32_t* range,
                                const float* lut, const float* bounds, uint32_t active, uint8_t* out, void* stream) {
  TDX_REQUIRE(planes && range && lut && out, "coarse_image: null pointer");
  TDX_REQUIRE(n >= 1, "coarse_image: empty input");
  TDX_REQUIRE(channel >= 0 && channel < kChannels, "coarse_image: channel %d is not in 0..5", (int)channel);
  TDX_REQUIRE((active & ~0xFF3u) == 0, "coarse_image: filter bits 0x%x: channel 1 is never a filter and there are 6 "
              "channels", (unsigned)active);
  TDX_REQUIRE(active == 0 || bounds, "coarse_image: filters without bounds");
  TDX_REQUIRE(reinterpret_cast<uintptr_t>(out) % 4 == 0, "coarse_image: out must be 4-byte aligned");
  CoarseFilter f{};
  for (int c = 0; c < kChannels && active; ++c) {
    f.lo[c] = bounds[2 * c];
    f.hi[c] = bounds[2 * c + 1];
  }
  f.active = active;
  return launch_cells(coarse_image_kernel, (long)n, reinterpret_cast<cudaStream_t>(stream), planes, (long)n,
                      (int)channel, reinterpret_cast<const unsigned*>(range), lut, f, reinterpret_cast<uchar4*>(out));
}

extern "C" int tdx_coarse_round(const float* x, int64_t n, float* out, void* stream) {
  TDX_REQUIRE(x && out, "coarse_round: null pointer");
  TDX_REQUIRE(n >= 1, "coarse_round: empty input");
  return launch_cells(coarse_round_kernel, (long)n, reinterpret_cast<cudaStream_t>(stream), x, (long)n, out);
}

extern "C" int tdx_coarse_land(const float* elev_m, int32_t h, int32_t w, int32_t half, double min_land_frac,
                               int32_t* rows, uint8_t* mask, int32_t* list, void* stream) {
  TDX_REQUIRE(elev_m && list, "coarse_land: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && half >= 0 && half <= 2048, "coarse_land: bad shape %d x %d, half %d", (int)h,
              (int)w, (int)half);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long ho = (long)h - 2L * half, wo = (long)w - 2L * half;
  if (ho <= 0 || wo <= 0) {                    // no window position fits: the list is empty
    TDX_CHECK_CUDA(cudaMemsetAsync(list, 0, sizeof(int32_t), st));
    return TDX_OK;
  }
  TDX_REQUIRE(rows && mask, "coarse_land: null pointer");
  TDX_REQUIRE((long)h * wo < (1L << 31), "coarse_land: %d x %ld positions overflow the int32 list", (int)h, wo);
  int rc = launch_cells(land_rows_kernel, (long)h * wo, st, elev_m, (int)h, (int)w, (int)half, (int)wo,
                        reinterpret_cast<int*>(rows));
  if (rc != TDX_OK) return rc;
  rc = launch_cells(land_mask_kernel, ho * wo, st, reinterpret_cast<const int*>(rows), (int)ho, (int)wo, (int)half,
                    min_land_frac, mask);
  if (rc != TDX_OK) return rc;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3(1), dim3(kCompactThreads), 0, st);
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, land_compact_kernel, (const uint8_t*)mask, ho * wo,
                                    reinterpret_cast<int*>(list)));
  return TDX_OK;
}
