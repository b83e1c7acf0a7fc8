// Depression filling and river-bed smoothing (inference/postprocessing.py:87-260), the two river functions of the
// reference that run before D8 routing.  The reference fills with a Python heapq Priority-Flood and smooths with a
// numpy Laplacian.  Here:
//   tdx_fill_depressions  classify every pixel (invalid, seed, free), then relax G below to its fixed point in passes
//                         of 32 x 32 shared-memory tiles, each tile iterated to local convergence;
//   tdx_smooth_river_bumps  one launch per iteration, ping-ponging two planes.
//
// Why the relaxation is exact.  With max_raise = None and epsilon >= 0 the heap only ever receives values at or above
// the element just popped, so the pops are non-decreasing and a free cell c takes its value from its first popped
// neighbour, the one with the smallest final value m:
//   out(c) = G(h(c), m) = h(c) if h(c) > m, else max(h(c), fl32(m + fl32(eps))).
// G is monotone in m and never below m, so the reference computes the generalised shortest-path solution from the
// seeds.  Every fixed point of out = G(h, min of the valid neighbours) is at most that solution (chain G along the
// best path from a seed), and relaxing downward from +inf never goes below it (G is monotone), so the relaxation
// ends on it whatever the order of updates and however stale the neighbour values it reads.  Values only decrease;
// a pass that lowers nothing read only final values, so the result is bit-identical under any thread schedule.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

constexpr int kFillTile = 32, kFillRows = 8;            // 32 x 32 cells per CTA; 32 x 8 threads, 4 rows each
constexpr int kFillHalo = kFillTile + 2;                // the tile and a 1-px ring
constexpr uint8_t kFillFree = 0, kFillSeed = 1, kFillInvalid = 2;
constexpr long kFillMaxPixels = 1L << 24;

// NaN, <= 0 (-0.0 and -inf included) or the caller's nodata (NaN when there is none: it equals nothing).
__device__ __forceinline__ bool fill_invalid(float v, float nodata) { return isnan(v) || v <= 0.f || v == nodata; }

// Seeds are the valid border pixels and the valid pixels with an invalid neighbour (the flood's own neighbourhood,
// inside the image); they and the invalid pixels keep h.  Free pixels start at +inf.
__global__ void fill_classify_kernel(const float* __restrict__ h, int H, int W, int eight, float nodata,
                                     uint8_t* __restrict__ kind, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)H * W) return;
  const int y = (int)(i / W), x = (int)(i % W);
  const float v = h[i];
  uint8_t k = kFillFree;
  if (fill_invalid(v, nodata)) {
    k = kFillInvalid;
  } else if (y == 0 || y == H - 1 || x == 0 || x == W - 1) {
    k = kFillSeed;
  } else {
    bool coast = fill_invalid(h[i - W], nodata) || fill_invalid(h[i + W], nodata) ||
                 fill_invalid(h[i - 1], nodata) || fill_invalid(h[i + 1], nodata);
    if (eight)
      coast = coast || fill_invalid(h[i - W - 1], nodata) || fill_invalid(h[i - W + 1], nodata) ||
              fill_invalid(h[i + W - 1], nodata) || fill_invalid(h[i + W + 1], nodata);
    if (coast) k = kFillSeed;
  }
  kind[i] = k;
  out[i] = k == kFillFree ? __int_as_float(0x7f800000) : v;
}

struct FillParams {
  const float* h;
  const uint8_t* kind;
  float* out;         // read and written in place by all CTAs of a pass (each pixel has one writer: its tile's CTA)
  uint32_t* flags;    // flags[p] != 0: pass p of this batch lowered a pixel
  int H, W, tiles_x;
  float eps;
};

// One pass over 32 x 32 tiles.  The tile's values and a 1-px ring (invalid or outside: +inf, never a minimum) are
// staged in shared memory, G is applied to the free pixels in place until an iteration lowers nothing, and the
// lowered pixels are written back.  Pass p runs only when pass p - 1 lowered something.
template <bool kEight>
__global__ void __launch_bounds__(kFillTile* kFillRows) fill_relax_kernel(const FillParams q, int pass) {
  __shared__ float v[kFillHalo][kFillHalo + 1];
  pdl_launch_dependents();
  pdl_wait();
  if (pass > 0 && q.flags[pass - 1] == 0) return;       // converged: the whole grid returns here
  const int tid = threadIdx.x, tx = tid % kFillTile, ty = tid / kFillTile;
  const int y0 = (blockIdx.x / q.tiles_x) * kFillTile, x0 = (blockIdx.x % q.tiles_x) * kFillTile;
  const float inf = __int_as_float(0x7f800000);
  for (int i = tid; i < kFillHalo * kFillHalo; i += blockDim.x) {
    const int r = i / kFillHalo, c = i % kFillHalo, gy = y0 - 1 + r, gx = x0 - 1 + c;
    float val = inf;
    if (gy >= 0 && gy < q.H && gx >= 0 && gx < q.W) {
      const long g = (long)gy * q.W + gx;
      if (q.kind[g] != kFillInvalid) val = q.out[g];
    }
    v[r][c] = val;
  }
  float hv[4], start[4];
  bool free_px[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int y = y0 + ty + j * kFillRows, x = x0 + tx;
    const long g = (long)y * q.W + x;
    free_px[j] = y < q.H && x < q.W && q.kind[g] == kFillFree;
    hv[j] = free_px[j] ? q.h[g] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) start[j] = v[ty + j * kFillRows + 1][tx + 1];

  for (;;) {
    bool lowered = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!free_px[j]) continue;
      const int r = ty + j * kFillRows + 1, c = tx + 1;
      float m = fminf(fminf(v[r - 1][c], v[r + 1][c]), fminf(v[r][c - 1], v[r][c + 1]));
      if (kEight) m = fminf(m, fminf(fminf(v[r - 1][c - 1], v[r - 1][c + 1]), fminf(v[r + 1][c - 1], v[r + 1][c + 1])));
      const float g = hv[j] > m ? hv[j] : fmaxf(hv[j], __fadd_rn(m, q.eps));
      if (g < v[r][c]) {
        v[r][c] = g;
        lowered = true;
      }
    }
    if (!__syncthreads_or(lowered)) break;   // an iteration that lowered nothing read only settled values
  }

  bool wrote = false;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float now = v[ty + j * kFillRows + 1][tx + 1];
    if (free_px[j] && now < start[j]) {
      q.out[(long)(y0 + ty + j * kFillRows) * q.W + x0 + tx] = now;
      wrote = true;
    }
  }
  if (__syncthreads_or(wrote) && tid == 0) q.flags[pass] = 1u;
}

// One iteration of smooth_river_bumps (postprocessing.py:99-133) at every pixel, each operation rounded separately
// in numpy's order.  `mask` is the input's NaN mask, fixed for all iterations; masked pixels read as 0 (h_safe) and
// come out NaN.  np.gradient: central differences / 2 inside, one-sided at the edges; np.roll: the Laplacian's
// neighbours wrap around.  exp is evaluated in fp64 and rounded once.
__global__ void smooth_step_kernel(const float* __restrict__ mask, const float* __restrict__ cur,
                                   float* __restrict__ nxt, int H, int W, float thresh, float strength) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)H * W) return;
  if (isnan(mask[i])) {
    nxt[i] = __int_as_float(0x7fc00000);
    return;
  }
  const int y = (int)(i / W), x = (int)(i % W);
  auto ok = [&](int yy, int xx) { return !isnan(mask[(long)yy * W + xx]); };
  auto hs = [&](int yy, int xx) { return ok(yy, xx) ? cur[(long)yy * W + xx] : 0.f; };
  const float c = cur[i];
  float gy, gx;
  if (y == 0) gy = __fsub_rn(hs(1, x), hs(0, x));
  else if (y == H - 1) gy = __fsub_rn(hs(H - 1, x), hs(H - 2, x));
  else gy = __fdiv_rn(__fsub_rn(hs(y + 1, x), hs(y - 1, x)), 2.f);
  if (x == 0) gx = __fsub_rn(hs(y, 1), hs(y, 0));
  else if (x == W - 1) gx = __fsub_rn(hs(y, W - 1), hs(y, W - 2));
  else gx = __fdiv_rn(__fsub_rn(hs(y, x + 1), hs(y, x - 1)), 2.f);
  const float slope = __fsqrt_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));
  const int yu = y == 0 ? H - 1 : y - 1, yd = y == H - 1 ? 0 : y + 1;
  const int xl = x == 0 ? W - 1 : x - 1, xr = x == W - 1 ? 0 : x + 1;
  const float sum = __fadd_rn(__fadd_rn(__fadd_rn(hs(yu, x), hs(yd, x)), hs(y, xl)), hs(y, xr));
  const float cnt = (float)((int)ok(yu, x) + (int)ok(yd, x) + (int)ok(y, xl) + (int)ok(y, xr));
  const float lap = __fsub_rn(sum, __fmul_rn(cnt, c));
  const float s = __fdiv_rn(slope, thresh);
  const float w = __double2float_rn(exp((double)-__fmul_rn(s, s)));
  nxt[i] = __fadd_rn(c, __fmul_rn(__fmul_rn(strength, w), lap));
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_fill_depressions(const float* height, int32_t h, int32_t w, float epsilon, int32_t connectivity,
                                    float nodata, float* out, uint8_t* kind, uint32_t* flags, int32_t* passes,
                                    void* stream) {
  TDX_REQUIRE(height && out && kind && flags, "fill_depressions: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && (long)h * w <= kFillMaxPixels, "fill_depressions: bad shape %d x %d (at most 2^24 px)",
              h, w);
  TDX_REQUIRE(epsilon >= 0.f && !isinf(epsilon), "fill_depressions: epsilon must be finite and >= 0, got %g",
              (double)epsilon);
  TDX_REQUIRE(out != height, "fill_depressions: out must not alias height");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long n = (long)h * w;
  TDX_CHECK_CUDA(launch(fill_classify_kernel, (unsigned)((n + 255) / 256), 256, 0, st, height, (int)h, (int)w,
                        (int)(connectivity != 4), nodata, kind, out));
  FillParams q;
  q.h = height; q.kind = kind; q.out = out; q.flags = flags; q.H = h; q.W = w; q.eps = epsilon;
  q.tiles_x = (w + kFillTile - 1) / kFillTile;
  const long tiles = (long)q.tiles_x * ((h + kFillTile - 1) / kFillTile);
  auto relax = connectivity != 4 ? fill_relax_kernel<true> : fill_relax_kernel<false>;
  // Batches of passes, each pass returning at once after a pass that lowered nothing; one flag read-back per batch.
  // Every pass that continues lowers a pixel, and after k passes every pixel whose best path from a seed has k cells
  // is final, so at most n + 1 passes run.
  uint32_t seen[TDX_FILL_BATCH];
  long total = 0;
  for (int batch = 4;; batch = batch * 2 > TDX_FILL_BATCH ? TDX_FILL_BATCH : batch * 2) {
    TDX_CHECK_CUDA(cudaMemsetAsync(flags, 0, batch * sizeof(uint32_t), st));
    for (int p = 0; p < batch; ++p)
      TDX_CHECK_CUDA(launch(relax, (unsigned)tiles, kFillTile * kFillRows, 0, st, q, p));
    TDX_CHECK_CUDA(cudaMemcpyAsync(seen, flags, batch * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    TDX_CHECK_CUDA(cudaStreamSynchronize(st));
    int p = 0;
    while (p < batch && seen[p]) ++p;
    if (p < batch) {
      total += p + 1;
      break;
    }
    total += batch;
    TDX_REQUIRE(total <= n + 1, "fill_depressions: no fixed point after %ld passes", total);
  }
  if (passes) *passes = (int32_t)total;
  return TDX_OK;
}

extern "C" int tdx_smooth_river_bumps(const float* height, int32_t h, int32_t w, float slope_thresh,
                                      float smooth_strength, int32_t iterations, float* out, float* scratch,
                                      void* stream) {
  TDX_REQUIRE(height && out, "smooth_river_bumps: null pointer");
  TDX_REQUIRE(h >= 2 && w >= 2 && (long)h * w <= kFillMaxPixels,
              "smooth_river_bumps: bad shape %d x %d (H, W >= 2, at most 2^24 px)", h, w);
  TDX_REQUIRE(out != height && scratch != height && scratch != out, "smooth_river_bumps: planes must not alias");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long n = (long)h * w;
  if (iterations <= 0) {
    TDX_CHECK_CUDA(cudaMemcpyAsync(out, height, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return TDX_OK;
  }
  TDX_REQUIRE(iterations == 1 || scratch, "smooth_river_bumps: %d iterations need a scratch plane", iterations);
  const float* src = height;
  for (int k = 0; k < iterations; ++k) {
    float* dst = (iterations - 1 - k) % 2 == 0 ? out : scratch;   // the last iteration lands in out
    TDX_CHECK_CUDA(launch(smooth_step_kernel, (unsigned)((n + 255) / 256), 256, 0, st, height, src, dst, (int)h,
                          (int)w, slope_thresh, smooth_strength));
    src = dst;
  }
  return TDX_OK;
}
