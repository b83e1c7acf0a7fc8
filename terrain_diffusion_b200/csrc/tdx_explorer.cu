// The explorer's detail view (terrain_diffusion/inference/explorer/server.py:188-270): the elevation and temperature
// images of `/api/detail.png`, the 8-bit RGBA of its relief mode, and the `/api/detail_raw` body.  The reference copies
// get()'s elevation and all five climate planes to the host and runs np.nanmin / np.nanmax, matplotlib's Normalize and
// colormap, np.clip and ScalarMappable.to_rgba(bytes=True) there.  Here:
//   tdx_detail_range   NaN-ignoring min and max of a plane into a small device buffer (one pass),
//   tdx_detail_colour  Normalize + colormap + to_rgba(bytes=True), one thread per pixel; it reads the range from the
//                      device buffer, so the image needs no host synchronisation before the final copy,
//   tdx_detail_rgba8   the relief branch's concatenate([clip(rgb), 1]) + to_rgba(bytes=True),
//   tdx_detail_raw     int16 elevation + fp32 temperature, the raw body.
// Every fp32 / fp64 operation is explicitly rounded in the order numpy performs it (NEP 50: the float64 scalars vmin and
// vmax promote the in-place subtraction and division to fp64, rounded once into the fp32 array).
#include "tdx_colour.cuh"
#include "tdx_common.h"
#include "tdx_ptx.cuh"
#include "tdx_upsample.cuh"

namespace tdx {

// range[0] = ~key(nanmin), range[1] = key(nanmax), both atomicMax on a zeroed buffer; 0 means "no non-NaN value".
__global__ void detail_range_kernel(const float* __restrict__ x, long n, unsigned* __restrict__ range) {
  pdl_launch_dependents();
  pdl_wait();
  unsigned nmn = 0, kmx = 0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float v = x[i];
    if (!isnan(v)) {
      const unsigned k = ordered_key(v);
      nmn = max(nmn, ~k);
      kmx = max(kmx, k);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    nmn = max(nmn, __shfl_xor_sync(0xffffffffu, nmn, o));
    kmx = max(kmx, __shfl_xor_sync(0xffffffffu, kmx, o));
  }
  if ((threadIdx.x & 31) == 0 && kmx) {
    atomicMax(&range[0], nmn);
    atomicMax(&range[1], kmx);
  }
}

__global__ void detail_colour_kernel(const float* __restrict__ x, long n, const unsigned* __restrict__ range,
                                     const float* __restrict__ lut, uchar4* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // server.py:207-216 and Colormap.__call__ (colour_index); the fp64 table was rounded to fp32 by
  // `.astype(np.float32)`.  Then _png_response's clip (a no-op on the table) and to_rgba(bytes=True); a NaN channel
  // cannot occur.
  const int idx = colour_index(x[i], range);
  uchar4 px = make_uchar4(0, 0, 0, 0);
  if (idx >= 0) {
    px.x = (unsigned char)quantise(clip01(lut[idx * 3 + 0]));
    px.y = (unsigned char)quantise(clip01(lut[idx * 3 + 1]));
    px.z = (unsigned char)quantise(clip01(lut[idx * 3 + 2]));
    px.w = 255;
  }
  out[i] = px;
}

// server.py:223-228: concatenate([clip(rgb, 0, 1), ones]) -> _png_response's clip -> to_rgba(bytes=True), which sets
// all four channels of a pixel with a NaN channel to 0.
__global__ void detail_rgba8_kernel(const float* __restrict__ rgb, long n, uchar4* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
  uchar4 px = make_uchar4(0, 0, 0, 0);
  if (!(isnan(r) || isnan(g) || isnan(b))) {
    px.x = (unsigned char)quantise(clip01(r));
    px.y = (unsigned char)quantise(clip01(g));
    px.z = (unsigned char)quantise(clip01(b));
    px.w = 255;
  }
  out[i] = px;
}

// server.py:252-260: H*W int16-LE elevation (tdx_post_combine's floor / clip / NaN -> 0 packing), then, with a
// temperature plane, its H*W fp32-LE values copied bit for bit.  The body is written as 16-bit words: the fp32 part
// starts at byte 2*H*W, which is only 2-byte aligned for an odd H*W.
__global__ void detail_raw_kernel(const float* __restrict__ elev, const float* __restrict__ temp, long n,
                                  uint16_t* __restrict__ body) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  body[i] = (uint16_t)elev_to_i16(elev[i]);
  if (temp) {
    const uint32_t bits = __float_as_uint(temp[i]);
    body[n + 2 * i] = (uint16_t)(bits & 0xFFFFu);
    body[n + 2 * i + 1] = (uint16_t)(bits >> 16);
  }
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_detail_range(const float* x, int64_t n, uint32_t* range, void* stream) {
  TDX_REQUIRE(x && range, "detail_range: null pointer");
  TDX_REQUIRE(n >= 1, "detail_range: empty input");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TDX_CHECK_CUDA(cudaMemsetAsync(range, 0, 2 * sizeof(uint32_t), st));
  const long blocks = (n + 255) / 256;
  const int grid = (int)(blocks < 4L * sm_count() ? blocks : 4L * sm_count());
  TDX_CHECK_CUDA(launch(detail_range_kernel, grid, 256, 0, st, x, (long)n, reinterpret_cast<unsigned*>(range)));
  return TDX_OK;
}

extern "C" int tdx_detail_colour(const float* x, int64_t n, const uint32_t* range, const float* lut, uint8_t* out,
                                 void* stream) {
  TDX_REQUIRE(x && range && lut && out, "detail_colour: null pointer");
  TDX_REQUIRE(n >= 1, "detail_colour: empty input");
  TDX_REQUIRE(reinterpret_cast<uintptr_t>(out) % 4 == 0, "detail_colour: out must be 4-byte aligned");
  TDX_CHECK_CUDA(launch(detail_colour_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, x, (long)n,
                        reinterpret_cast<const unsigned*>(range), lut, reinterpret_cast<uchar4*>(out)));
  return TDX_OK;
}

extern "C" int tdx_detail_rgba8(const float* rgb, int64_t n, uint8_t* out, void* stream) {
  TDX_REQUIRE(rgb && out, "detail_rgba8: null pointer");
  TDX_REQUIRE(n >= 1, "detail_rgba8: empty input");
  TDX_REQUIRE(reinterpret_cast<uintptr_t>(out) % 4 == 0, "detail_rgba8: out must be 4-byte aligned");
  TDX_CHECK_CUDA(launch(detail_rgba8_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, rgb, (long)n,
                        reinterpret_cast<uchar4*>(out)));
  return TDX_OK;
}

extern "C" int tdx_detail_raw(const float* elev, const float* temp, int64_t n, void* body, void* stream) {
  TDX_REQUIRE(elev && body, "detail_raw: null pointer");
  TDX_REQUIRE(n >= 1, "detail_raw: empty input");
  TDX_REQUIRE(reinterpret_cast<uintptr_t>(body) % 2 == 0, "detail_raw: body must be 2-byte aligned");
  TDX_CHECK_CUDA(launch(detail_raw_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, elev, temp, (long)n,
                        static_cast<uint16_t*>(body)));
  return TDX_OK;
}
