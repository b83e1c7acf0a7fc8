// River routing (inference/postprocessing.py:6-85): D8 steepest-descent receivers, upstream cell counts and the
// log1p flow indicator that the relief map draws rivers from.  The reference runs them on the CPU, the accumulation as
// a Python loop over every land pixel in descending elevation order.  Here:
//   tdx_flow_d8          one stencil pass: kmax, is_sink, rr / cc, the receiver of every pixel that pushes its count
//                        downstream, and each pixel's in-degree, gathered from the neighbours' receivers (no atomics);
//   tdx_flow_link        the same receiver / in-degree arrays from receivers given by the caller, with the checks that
//                        make the accumulation exact (indices in range, every followed edge strictly downhill);
//   tdx_flow_accumulate  exact integer subtree sums over that forest: leaves walk downstream, and at each node only
//                        the last child to arrive carries on, so no thread ever waits for another;
//   tdx_flow_indicator   non-overlapping k x k max-pool and log1p.
// A pixel is ocean (invalid) when it is NaN or <= 0 (-inf included).  A pixel "pushes" when it is valid, not a sink,
// and its receiver is valid: exactly the edges flow_accumulation follows.  Only +inf is flagged: a +inf pixel next to
// another makes the reference's slope NaN (inf - inf), and its argmax then depends on where the NaN sits.  -inf is
// ocean, so the ocean rules overwrite every slope it takes part in.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

constexpr int kFlowTileW = 32, kFlowTileH = 8;                  // output pixels per CTA of the D8 pass
constexpr int kFlowCodeW = kFlowTileW + 2, kFlowCodeH = kFlowTileH + 2;   // receivers of the tile and its 1-px ring
constexpr int kFlowZW = kFlowTileW + 4, kFlowZH = kFlowTileH + 4;         // elevations: a 2-px ring
constexpr unsigned char kNoPush = 0xff;

__device__ __forceinline__ bool is_ocean(float v) { return isnan(v) || v <= 0.f; }
__device__ __forceinline__ bool is_pos_inf(float v) { return v == __int_as_float(0x7f800000); }
__device__ __forceinline__ int clampi(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

struct D8Cell {
  int k;        // first argmax of the `prefer` column
  bool sink;
  bool push;
  int ry, rx;   // receiver, clamped into the image
};

// d8_flow at image pixel (y, x), whose elevation is zs[sy][sx]; zs holds the edge-clamped elevations around it.
// Neighbour order N, S, W, E, NW, NE, SW, SE.  slope = (z - n) / dist in fp32 (dist = fp32(sqrt 2) on the diagonals),
// -inf below tol (compared in fp32, as NumPy 2 compares a float32 array with a Python float).  `prefer`: -inf for an
// ocean centre, +inf for an ocean neighbour of a land centre, else the slope; `ignore`: -inf for both.  No slope is
// NaN once those rules apply: a NaN operand is ocean.
__device__ __forceinline__ D8Cell d8_cell(const float (*zs)[kFlowZW], int sy, int sx, int y, int x, int h, int w,
                                          float tol) {
  constexpr int dy[8] = {-1, 1, 0, 0, -1, -1, 1, 1};
  constexpr int dx[8] = {0, 0, -1, 1, -1, 1, -1, 1};
  const float c = zs[sy][sx];
  const bool c_ocean = is_ocean(c);
  const float inf = __int_as_float(0x7f800000);
  float best = -inf;
  int kmax = 0, best_dy = dy[0], best_dx = dx[0];
  bool best_ocean = false, any_ocean = false, any_slope = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float n = zs[sy + dy[k]][sx + dx[k]];
    const bool n_ocean = is_ocean(n);
    float s = __fdiv_rn(__fsub_rn(c, n), k < 4 ? 1.0f : 1.41421354f);
    if (s < tol) s = -inf;
    any_ocean |= n_ocean;
    any_slope |= !c_ocean && !n_ocean && s != -inf;   // a finite entry of `ignore`
    const float p = c_ocean ? -inf : (n_ocean ? inf : s);
    if (p > best) {
      best = p;
      kmax = k;
      best_dy = dy[k];
      best_dx = dx[k];
      best_ocean = n_ocean;
    }
  }
  D8Cell r;
  r.k = kmax;
  r.sink = c_ocean || (!any_ocean && !any_slope);
  r.push = !r.sink && !best_ocean;   // the chosen neighbour is the receiver's own (clamped) value
  r.ry = clampi(y + best_dy, h - 1);
  r.rx = clampi(x + best_dx, w - 1);
  return r;
}

__device__ __forceinline__ unsigned char push_code(const D8Cell& r, int y, int x) {
  return r.push ? (unsigned char)((r.ry - y + 1) * 3 + (r.rx - x + 1)) : kNoPush;
}

struct FlowD8Params {
  const float* z;
  int h, w, tiles_x;
  float tol;
  int8_t* kmax;
  uint8_t* is_sink;
  int64_t* rr;
  int64_t* cc;
  int32_t* recv;
  uint32_t* indeg;
  uint32_t* flags;
};

// One CTA = a 32 x 8 tile.  The elevations of the tile and a 2-px ring are staged edge-clamped in shared memory; D8 is
// evaluated on the tile and its 1-px ring (the ring's receivers are recomputed by both neighbouring CTAs), and each
// pixel counts the neighbours whose receiver it is.
__global__ void __launch_bounds__(kFlowTileW* kFlowTileH) flow_d8_kernel(const FlowD8Params q) {
  __shared__ float zs[kFlowZH][kFlowZW];
  __shared__ unsigned char code[kFlowCodeH][kFlowCodeW];
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x;
  const int y0 = (blockIdx.x / q.tiles_x) * kFlowTileH, x0 = (blockIdx.x % q.tiles_x) * kFlowTileW;
  for (int i = tid; i < kFlowZH * kFlowZW; i += blockDim.x) {
    const int r = i / kFlowZW, c = i % kFlowZW;
    zs[r][c] = q.z[(long)clampi(y0 - 2 + r, q.h - 1) * q.w + clampi(x0 - 2 + c, q.w - 1)];
  }
  __syncthreads();

  // this thread's own pixel
  const int ly = tid / kFlowTileW, lx = tid % kFlowTileW, y = y0 + ly, x = x0 + lx;
  const bool inside = y < q.h && x < q.w;
  D8Cell own = {};
  if (inside) own = d8_cell(zs, ly + 2, lx + 2, y, x, q.h, q.w, q.tol);
  code[ly + 1][lx + 1] = inside ? push_code(own, y, x) : kNoPush;
  // the 84 cells of the 1-px ring: top row, bottom row, left column, right column
  constexpr int kRing = 2 * kFlowCodeW + 2 * kFlowTileH;
  if (tid < kRing) {
    int cy, cx;
    if (tid < kFlowCodeW) cy = 0, cx = tid;
    else if (tid < 2 * kFlowCodeW) cy = kFlowCodeH - 1, cx = tid - kFlowCodeW;
    else if (tid < 2 * kFlowCodeW + kFlowTileH) cy = tid - 2 * kFlowCodeW + 1, cx = 0;
    else cy = tid - 2 * kFlowCodeW - kFlowTileH + 1, cx = kFlowCodeW - 1;
    const int gy = y0 - 1 + cy, gx = x0 - 1 + cx;
    unsigned char cd = kNoPush;
    if (gy >= 0 && gy < q.h && gx >= 0 && gx < q.w)
      cd = push_code(d8_cell(zs, cy + 1, cx + 1, gy, gx, q.h, q.w, q.tol), gy, gx);
    code[cy][cx] = cd;
  }
  __syncthreads();
  if (!inside) return;

  const long o = (long)y * q.w + x;
  if (is_pos_inf(zs[ly + 2][lx + 2])) atomicOr(q.flags, (unsigned)TDX_FLOW_INF);
  if (q.kmax) q.kmax[o] = (int8_t)own.k;
  if (q.is_sink) q.is_sink[o] = own.sink;
  if (q.rr) q.rr[o] = own.ry;
  if (q.cc) q.cc[o] = own.rx;
  if (q.recv) q.recv[o] = own.push ? (int32_t)((long)own.ry * q.w + own.rx) : -1;
  if (q.indeg) {
    // neighbour (y+a, x+b) drains here when its receiver offset is (-a, -b)
    unsigned deg = 0;
#pragma unroll
    for (int a = -1; a <= 1; ++a)
#pragma unroll
      for (int b = -1; b <= 1; ++b)
        if ((a || b) && code[ly + 1 + a][lx + 1 + b] == (unsigned char)((1 - a) * 3 + (1 - b))) ++deg;
    q.indeg[o] = deg;
  }
}

// Receivers given by the caller (flow_accumulation's rr, cc, is_sink): the edges the reference follows, their
// in-degrees by atomic scatter, and flags for the inputs on which its result would depend on the visiting order.
__global__ void flow_link_kernel(const float* __restrict__ z, const int64_t* __restrict__ rr,
                                 const int64_t* __restrict__ cc, const uint8_t* __restrict__ is_sink, int h, int w,
                                 int32_t* __restrict__ recv, uint32_t* __restrict__ indeg,
                                 uint32_t* __restrict__ flags) {
  pdl_launch_dependents();
  pdl_wait();
  const long v = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (long)h * w) return;
  const float c = z[v];
  unsigned bad = is_pos_inf(c) ? (unsigned)TDX_FLOW_INF : 0u;
  const int64_t r = rr[v], s = cc[v];
  int32_t t = -1;
  if (r < 0 || r >= h || s < 0 || s >= w) {
    bad |= (unsigned)TDX_FLOW_RANGE;
  } else if (!is_ocean(c) && !is_sink[v]) {
    const int32_t u = (int32_t)(r * w + s);
    const float e = z[u];
    if (!is_ocean(e)) {
      if (e < c) t = u;
      else bad |= (unsigned)TDX_FLOW_NOT_DOWNHILL;
    }
  }
  recv[v] = t;
  if (t >= 0) atomicAdd(&indeg[t], 1u);
  if (bad) atomicOr(flags, bad);
}

// A[v] = 1 + sum of A over v's children, exactly, for valid v; 0 for invalid v.  state[t] packs (children arrived,
// sum of their A) as hi:lo 32 bits, so one 64-bit atomicAdd both adds a child's total and counts its arrival, and the
// child that sees the count reach in-degree - 1 holds the complete sum: it writes A[t] and carries it on.  Each edge is
// added once: O(n) atomics.  No thread waits for another; the latency is the longest flow path.  Counts are at most
// n <= 2^24, so the fp32 store is exact.
__global__ void flow_accumulate_kernel(const float* __restrict__ z, const int32_t* __restrict__ recv,
                                       const uint32_t* __restrict__ indeg, unsigned long long* __restrict__ state,
                                       float* __restrict__ A, int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  if (is_ocean(z[v])) {
    A[v] = 0.f;
    return;
  }
  if (indeg[v] != 0) return;   // finished by the last of its children to arrive
  unsigned total = 1;
  A[v] = 1.f;
  for (int t = recv[v]; t >= 0; t = recv[t]) {
    const unsigned long long old = atomicAdd(&state[t], (1ull << 32) | total);
    if ((unsigned)(old >> 32) + 1u != indeg[t]) break;
    total = (unsigned)old + total + 1u;
    A[t] = (float)total;
  }
}

// np.log1p of the k x k max-pool of A (remainder rows / columns dropped), in fp32 rounded once from fp64.
__global__ void flow_indicator_kernel(const float* __restrict__ A, int w, int k, int oh, int ow,
                                      float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)oh * ow) return;
  const int oy = (int)(i / ow), ox = (int)(i % ow);
  const float* p = A + (long)oy * k * w + (long)ox * k;
  float m = p[0];
  for (int a = 0; a < k; ++a)
    for (int b = 0; b < k; ++b) m = fmaxf(m, p[(long)a * w + b]);
  out[i] = __double2float_rn(log1p((double)m));
}

constexpr long kFlowMaxPixels = 1L << 24;

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_flow_d8(const float* z, int32_t h, int32_t w, float tol, int8_t* kmax, uint8_t* is_sink,
                           int64_t* rr, int64_t* cc, int32_t* recv, uint32_t* indeg, uint32_t* flags, void* stream) {
  TDX_REQUIRE(z && flags, "flow_d8: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && (long)h * w <= kFlowMaxPixels, "flow_d8: bad shape %d x %d (at most 2^24 px)", h, w);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TDX_CHECK_CUDA(cudaMemsetAsync(flags, 0, sizeof(uint32_t), st));
  FlowD8Params q;
  q.z = z; q.h = h; q.w = w; q.tol = tol;
  q.tiles_x = (w + kFlowTileW - 1) / kFlowTileW;
  q.kmax = kmax; q.is_sink = is_sink; q.rr = rr; q.cc = cc; q.recv = recv; q.indeg = indeg; q.flags = flags;
  const long tiles = (long)q.tiles_x * ((h + kFlowTileH - 1) / kFlowTileH);
  TDX_CHECK_CUDA(launch(flow_d8_kernel, (unsigned)tiles, kFlowTileW * kFlowTileH, 0, st, q));
  return TDX_OK;
}

extern "C" int tdx_flow_link(const float* z, const int64_t* rr, const int64_t* cc, const uint8_t* is_sink, int32_t h,
                             int32_t w, int32_t* recv, uint32_t* indeg, uint32_t* flags, void* stream) {
  TDX_REQUIRE(z && rr && cc && is_sink && recv && indeg && flags, "flow_link: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && (long)h * w <= kFlowMaxPixels, "flow_link: bad shape %d x %d (at most 2^24 px)", h,
              w);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long n = (long)h * w;
  TDX_CHECK_CUDA(cudaMemsetAsync(flags, 0, sizeof(uint32_t), st));
  TDX_CHECK_CUDA(cudaMemsetAsync(indeg, 0, n * sizeof(uint32_t), st));
  TDX_CHECK_CUDA(launch(flow_link_kernel, (unsigned)((n + 255) / 256), 256, 0, st, z, rr, cc, is_sink, (int)h, (int)w,
                        recv, indeg, flags));
  return TDX_OK;
}

extern "C" int tdx_flow_accumulate(const float* z, int64_t n, const int32_t* recv, const uint32_t* indeg,
                                   uint64_t* state, float* A, void* stream) {
  TDX_REQUIRE(z && recv && indeg && state && A, "flow_accumulate: null pointer");
  TDX_REQUIRE(n >= 1 && n <= kFlowMaxPixels, "flow_accumulate: %lld px (1 .. 2^24)", (long long)n);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TDX_CHECK_CUDA(cudaMemsetAsync(state, 0, n * sizeof(uint64_t), st));
  TDX_CHECK_CUDA(launch(flow_accumulate_kernel, (unsigned)((n + 255) / 256), 256, 0, st, z, recv, indeg,
                        reinterpret_cast<unsigned long long*>(state), A, (int)n));
  return TDX_OK;
}

extern "C" int tdx_flow_indicator(const float* A, int32_t h, int32_t w, int32_t k, float* out, void* stream) {
  TDX_REQUIRE(h >= 1 && w >= 1 && (long)h * w <= kFlowMaxPixels, "flow_indicator: bad shape %d x %d", h, w);
  if (k < 1) k = 1;
  const int oh = h / k, ow = w / k;
  if (oh == 0 || ow == 0) return TDX_OK;   // k exceeds the image: an empty result
  TDX_REQUIRE(A && out, "flow_indicator: null pointer");
  const long m = (long)oh * ow;
  TDX_CHECK_CUDA(launch(flow_indicator_kernel, (unsigned)((m + 255) / 256), 256, 0, stream, A, (int)w, (int)k, oh, ow,
                        out));
  return TDX_OK;
}
