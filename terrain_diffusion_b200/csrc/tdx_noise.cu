// Tile-seeded Gaussian noise field on the GPU, bit-compatible with the reference's sequential generator.
//
// Reference: terrain_diffusion/inference/portable_rng.py:24-82 (PCG-XSH-RR 64/32 + Marsaglia polar, fp64 math, numba)
//            terrain_diffusion/inference/world_pipeline.py:58-115 (_tile_seed, gaussian_noise_patch)
//
// The reference stream is sequential: candidate pair p consumes LCG outputs 2p and 2p+1, and the output position of an
// accepted pair is twice the number of pairs accepted before it.  Both are parallelisable exactly:
//   * the LCG state after k steps is an affine function of the seed (jump-ahead in O(log k) 64-bit multiplies);
//   * the output position is an exclusive prefix sum of the acceptance flags.
// So each thread jumps to a chunk of kChunk candidate pairs, (pass 1) counts its acceptances, (pass 2) a single block
// scans the counts, (pass 3) each thread regenerates its chunk and writes its normals -- only those that fall inside
// the requested patch -- at their exact stream positions.  Acceptance uses the reference's fp64 arithmetic with
// separately rounded multiplies and adds (no FMA contraction), so the integer stream positions are bit-exact.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

constexpr unsigned long long kMult = 6364136223846793005ULL;
constexpr unsigned long long kInc = 1442695040888963407ULL;
constexpr int kChunk = 8;  // candidate pairs per thread

__host__ __device__ inline unsigned long long lcg_jump(unsigned long long state, unsigned long long steps) {
  unsigned long long acc_mult = 1ULL, acc_plus = 0ULL, cur_mult = kMult, cur_plus = kInc;
  while (steps > 0) {
    if (steps & 1ULL) {
      acc_mult *= cur_mult;
      acc_plus = acc_plus * cur_mult + cur_plus;
    }
    cur_plus = (cur_mult + 1ULL) * cur_plus;
    cur_mult *= cur_mult;
    steps >>= 1;
  }
  return acc_mult * state + acc_plus;
}

__device__ __forceinline__ unsigned int pcg_next(unsigned long long& state) {
  state = state * kMult + kInc;
  const unsigned long long s = state;
  const unsigned int x = (unsigned int)(((s >> 18) ^ s) >> 27);
  const unsigned int rot = (unsigned int)(s >> 59);
  return (x >> rot) | (x << ((32 - rot) & 31));
}

__device__ __forceinline__ bool polar_pair(unsigned long long& state, double& v1, double& v2, double& s) {
  const unsigned int u1 = pcg_next(state);
  const unsigned int u2 = pcg_next(state);
  const double inv = 1.0 / 4294967296.0;
  v1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, __dadd_rn((double)u1, 1.0)), inv), -1.0);
  v2 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, __dadd_rn((double)u2, 1.0)), inv), -1.0);
  s = __dadd_rn(__dmul_rn(v1, v1), __dmul_rn(v2, v2));
  return s > 0.0 && s < 1.0;
}

// Pass 1: how many of the candidate pairs of `chunk` the polar method accepts.
__device__ __forceinline__ void count_chunk(unsigned long long seed, long long n_pairs, long long chunk, int* counts) {
  const long long p0 = chunk * kChunk;
  if (p0 >= n_pairs) return;
  unsigned long long state = lcg_jump(seed, 2ULL * (unsigned long long)p0);
  int c = 0;
  for (int i = 0; i < kChunk && p0 + i < n_pairs; ++i) {
    double v1, v2, s;
    c += polar_pair(state, v1, v2, s) ? 1 : 0;
  }
  counts[chunk] = c;
}

// Pass 2: exclusive scan of `n` ints in place by one block (n is a few tens of thousands at most).
__device__ __forceinline__ void scan_counts(int* counts, long long n) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long base = 0; base < n; base += blockDim.x) {
    const long long i = base + threadIdx.x;
    const int v = i < n ? counts[i] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffff, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffff, w, o);
        if (lane >= o) w += t;
      }
      warp_tot[lane] = w;  // inclusive scan of warp totals
    }
    __syncthreads();
    const int warp_off = warp == 0 ? 0 : warp_tot[warp - 1];
    const int block_total = warp_tot[(blockDim.x >> 5) - 1];
    if (i < n) counts[i] = carry + warp_off + incl - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += block_total;
    __syncthreads();
  }
}

struct NoiseEmit {
  unsigned long long seed;
  long long n_pairs, n_out;        // candidate pairs generated; normals in one tile stream (C*th*tw)
  int tile_h, tile_w;
  long long tile_y0, tile_x0;      // world coordinate of the tile origin
  long long y0, x0;                // patch origin
  int h, w, channels;
  float* out;                      // [C][h][w]
  int* status;                     // set to 1 if the candidate budget was too small
};

__device__ __forceinline__ void noise_store(const NoiseEmit& p, long long idx, double val) {
  if (idx >= p.n_out) return;
  const long long plane = (long long)p.tile_h * p.tile_w;
  const int c = (int)(idx / plane);
  const long long rem = idx - c * plane;
  const long long Y = p.tile_y0 + rem / p.tile_w, X = p.tile_x0 + rem % p.tile_w;
  if (Y < p.y0 || Y >= p.y0 + p.h || X < p.x0 || X >= p.x0 + p.w) return;
  p.out[((long long)c * p.h + (Y - p.y0)) * p.w + (X - p.x0)] = (float)val;
}

// Pass 3: regenerate the pairs of `chunk` and store the normals that fall inside the patch at their stream positions.
// The last chunk flags a budget that ran out before the stream was complete.
__device__ __forceinline__ void emit_chunk(const NoiseEmit& p, const int* offsets, long long chunk,
                                           long long n_chunks) {
  if (chunk >= n_chunks) return;
  const long long p0 = chunk * kChunk;
  long long pos = 2LL * offsets[chunk];
  if (pos >= p.n_out) return;
  unsigned long long state = lcg_jump(p.seed, 2ULL * (unsigned long long)p0);
  for (int i = 0; i < kChunk && p0 + i < p.n_pairs; ++i) {
    double v1, v2, s;
    if (polar_pair(state, v1, v2, s)) {
      const double f = sqrt(__ddiv_rn(__dmul_rn(-2.0, log(s)), s));
      noise_store(p, pos, __dmul_rn(v1, f));
      noise_store(p, pos + 1, __dmul_rn(v2, f));
      pos += 2;
      if (pos >= p.n_out) return;
    }
  }
  if (chunk == n_chunks - 1 && pos < p.n_out) *p.status = 1;
}

// ---- single form: one (patch, tile) job per launch
__global__ void noise_count_kernel(unsigned long long seed, long long n_pairs, int* counts) {
  pdl_launch_dependents();
  pdl_wait();
  count_chunk(seed, n_pairs, (long long)blockIdx.x * blockDim.x + threadIdx.x, counts);
}

__global__ void noise_scan_kernel(int* counts, long long n_chunks) {
  pdl_launch_dependents();
  pdl_wait();
  scan_counts(counts, n_chunks);
}

__global__ void noise_emit_kernel(const NoiseEmit p, const int* offsets, long long n_chunks) {
  pdl_launch_dependents();
  pdl_wait();
  emit_chunk(p, offsets, (long long)blockIdx.x * blockDim.x + threadIdx.x, n_chunks);
}

// ---- batched form: up to kBatchJobs (patch, tile) jobs per launch, job = blockIdx.y, one counts slice per job
constexpr int kBatchJobs = 32;
struct NoiseBatch {
  int n_jobs;
  long long n_chunks;
  NoiseEmit job[kBatchJobs];
};

__global__ void noise_count_batch_kernel(const __grid_constant__ NoiseBatch b, int* counts) {
  pdl_launch_dependents();
  pdl_wait();
  const NoiseEmit& p = b.job[blockIdx.y];
  count_chunk(p.seed, p.n_pairs, (long long)blockIdx.x * blockDim.x + threadIdx.x,
              counts + (long long)blockIdx.y * b.n_chunks);
}

__global__ void noise_scan_batch_kernel(int* counts, long long n_chunks) {
  pdl_launch_dependents();
  pdl_wait();
  scan_counts(counts + (long long)blockIdx.x * n_chunks, n_chunks);
}

__global__ void noise_emit_batch_kernel(const __grid_constant__ NoiseBatch b, const int* counts) {
  pdl_launch_dependents();
  pdl_wait();
  emit_chunk(b.job[blockIdx.y], counts + (long long)blockIdx.y * b.n_chunks,
             (long long)blockIdx.x * blockDim.x + threadIdx.x, b.n_chunks);
}

static long long floordiv(long long a, long long b) {
  long long q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}

static long long pair_budget(long long n_out) {
  // acceptance probability pi/4; 2 % + 1024 pairs of head-room is > 20 sigma for every stream length
  const double need = (double)((n_out + 1) / 2) / 0.7853981633974483;
  return (long long)(need * 1.02) + 1024;
}

unsigned long long tile_seed(unsigned long long base, long long ty, long long tx) {
  unsigned long long h = base * 0x9E3779B9ULL;
  h = h + ((unsigned long long)ty & 0xFFFFFFFFULL);
  h = h * 0x9E3779B9ULL + ((unsigned long long)tx & 0xFFFFFFFFULL);
  return h;
}

constexpr int kNoiseThreads = 128;   // threads of the count and emit passes; the scan runs on one 1024-thread block

// The three passes of one single-form job, counts[n_chunks] as their scratch.
static int run_noise_job(const NoiseEmit& p, int* counts, long long n_chunks, cudaStream_t stream) {
  const int blocks = (int)((n_chunks + kNoiseThreads - 1) / kNoiseThreads);
  TDX_CHECK_CUDA(launch(noise_count_kernel, blocks, kNoiseThreads, 0, stream, p.seed, p.n_pairs, counts));
  TDX_CHECK_CUDA(launch(noise_scan_kernel, 1, 1024, 0, stream, counts, n_chunks));
  TDX_CHECK_CUDA(launch(noise_emit_kernel, blocks, kNoiseThreads, 0, stream, p, counts, n_chunks));
  return TDX_OK;
}

}  // namespace tdx

using namespace tdx;

extern "C" int64_t tdx_noise_patch_workspace_bytes(int32_t channels, int32_t tile_h, int32_t tile_w) {
  const long long n_out = (long long)channels * tile_h * tile_w;
  const long long chunks = (pair_budget(n_out) + kChunk - 1) / kChunk;
  return (int64_t)(chunks * sizeof(int) + 256);
}

extern "C" uint64_t tdx_tile_seed(uint64_t base_seed, int64_t ty, int64_t tx) { return tile_seed(base_seed, ty, tx); }

extern "C" int tdx_noise_patch(uint64_t base_seed, int64_t y0, int64_t x0, int32_t h, int32_t w, int32_t channels,
                               int32_t tile_h, int32_t tile_w, float* out, void* workspace, int64_t workspace_bytes,
                               void* stream_) {
  TDX_REQUIRE(out && workspace, "noise_patch: null pointer");
  TDX_REQUIRE(h >= 1 && w >= 1 && channels >= 1 && tile_h >= 1 && tile_w >= 1, "noise_patch: bad shape");
  TDX_REQUIRE(workspace_bytes >= tdx_noise_patch_workspace_bytes(channels, tile_h, tile_w),
              "noise_patch: workspace too small (%lld bytes)", (long long)workspace_bytes);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long n_out = (long long)channels * tile_h * tile_w;
  TDX_REQUIRE(n_out < (1LL << 30), "noise_patch: tile stream too long");
  const long long n_pairs = pair_budget(n_out);
  const long long n_chunks = (n_pairs + kChunk - 1) / kChunk;
  int* status = reinterpret_cast<int*>(workspace);
  int* counts = status + 64;
  TDX_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  const long long ty0 = floordiv(y0, tile_h), ty1 = floordiv(y0 + h - 1, tile_h);
  const long long tx0 = floordiv(x0, tile_w), tx1 = floordiv(x0 + w - 1, tile_w);
  for (long long ty = ty0; ty <= ty1; ++ty) {
    for (long long tx = tx0; tx <= tx1; ++tx) {
      const NoiseEmit p = {tile_seed(base_seed, ty, tx), n_pairs, n_out, tile_h, tile_w, ty * tile_h, tx * tile_w, y0,
                           x0, h, w, channels, out, status};
      int rc = run_noise_job(p, counts, n_chunks, stream);
      if (rc != TDX_OK) return rc;
    }
  }
  return TDX_OK;
}

/* Batched tdx_noise_patch: n_patches patches of one shape, origins in HOST arrays y0s / x0s, out = [n][C][h][w].
 * Every (patch, covering tile) pair is one job; 32 jobs share a launch (three launches per 32 jobs instead of three per
 * job).  workspace >= tdx_noise_patches_workspace_bytes(channels, tile_h, tile_w).  Bit-identical to the single form. */
extern "C" int64_t tdx_noise_patches_workspace_bytes(int32_t channels, int32_t tile_h, int32_t tile_w) {
  const long long n_out = (long long)channels * tile_h * tile_w;
  const long long chunks = (pair_budget(n_out) + kChunk - 1) / kChunk;
  return (int64_t)(chunks * sizeof(int) * kBatchJobs + 256);
}

extern "C" int tdx_noise_patches(uint64_t base_seed, int32_t n_patches, const int64_t* y0s, const int64_t* x0s, int32_t h,
                                 int32_t w, int32_t channels, int32_t tile_h, int32_t tile_w, float* out,
                                 void* workspace, int64_t workspace_bytes, void* stream_) {
  TDX_REQUIRE(out && workspace && y0s && x0s, "noise_patches: null pointer");
  TDX_REQUIRE(n_patches >= 1 && h >= 1 && w >= 1 && channels >= 1 && tile_h >= 1 && tile_w >= 1,
              "noise_patches: bad shape");
  TDX_REQUIRE(workspace_bytes >= tdx_noise_patches_workspace_bytes(channels, tile_h, tile_w),
              "noise_patches: workspace too small (%lld bytes)", (long long)workspace_bytes);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long n_out = (long long)channels * tile_h * tile_w;
  TDX_REQUIRE(n_out < (1LL << 30), "noise_patches: tile stream too long");
  const long long n_pairs = pair_budget(n_out);
  const long long n_chunks = (n_pairs + kChunk - 1) / kChunk;
  int* status = reinterpret_cast<int*>(workspace);
  int* counts = status + 64;
  TDX_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  const int blocks = (int)((n_chunks + kNoiseThreads - 1) / kNoiseThreads);
  NoiseBatch b;
  b.n_jobs = 0;
  b.n_chunks = n_chunks;
  auto flush = [&]() -> int {
    if (b.n_jobs == 0) return TDX_OK;
    TDX_CHECK_CUDA(launch(noise_count_batch_kernel, dim3(blocks, b.n_jobs), kNoiseThreads, 0, stream, b, counts));
    TDX_CHECK_CUDA(launch(noise_scan_batch_kernel, b.n_jobs, 1024, 0, stream, counts, n_chunks));
    TDX_CHECK_CUDA(launch(noise_emit_batch_kernel, dim3(blocks, b.n_jobs), kNoiseThreads, 0, stream, b, counts));
    b.n_jobs = 0;
    return TDX_OK;
  };
  for (int i = 0; i < n_patches; ++i) {
    const long long y0 = y0s[i], x0 = x0s[i];
    const long long ty0 = floordiv(y0, tile_h), ty1 = floordiv(y0 + h - 1, tile_h);
    const long long tx0 = floordiv(x0, tile_w), tx1 = floordiv(x0 + w - 1, tile_w);
    for (long long ty = ty0; ty <= ty1; ++ty) {
      for (long long tx = tx0; tx <= tx1; ++tx) {
        b.job[b.n_jobs++] = {tile_seed(base_seed, ty, tx), n_pairs, n_out, tile_h, tile_w, ty * tile_h, tx * tile_w,
                             y0, x0, h, w, channels, out + (long long)i * channels * h * w, status};
        if (b.n_jobs == kBatchJobs) {
          int rc = flush();
          if (rc != TDX_OK) return rc;
        }
      }
    }
  }
  return flush();
}

/* portable_rng.standard_normal(seed, n): ONE stream of n fp32 normals seeded directly with `seed` (no tile hash);
 * workspace: tdx_noise_patch_workspace_bytes(1, 1, n) bytes. */
extern "C" int tdx_standard_normal(uint64_t seed, int64_t n, float* out, void* workspace, int64_t workspace_bytes,
                                   void* stream_) {
  TDX_REQUIRE(out && workspace && n >= 1 && n < (1LL << 30), "standard_normal: bad arguments");
  TDX_REQUIRE(workspace_bytes >= tdx_noise_patch_workspace_bytes(1, 1, (int32_t)n),
              "standard_normal: workspace too small (%lld bytes)", (long long)workspace_bytes);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long n_pairs = pair_budget(n);
  const long long n_chunks = (n_pairs + kChunk - 1) / kChunk;
  int* status = reinterpret_cast<int*>(workspace);
  int* counts = status + 64;
  TDX_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  const NoiseEmit p = {seed, n_pairs, n, 1, (int)n, 0, 0, 0, 0, 1, (int)n, 1, out, status};
  return run_noise_job(p, counts, n_chunks, stream);
}

/* Reads back the overflow flag written by the last tdx_noise_patch on this workspace (synchronises the stream). */
extern "C" int tdx_noise_patch_status(void* workspace, void* stream_) {
  int st = 0;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  TDX_CHECK_CUDA(cudaMemcpyAsync(&st, workspace, sizeof(int), cudaMemcpyDeviceToHost, stream));
  TDX_CHECK_CUDA(cudaStreamSynchronize(stream));
  if (st != 0) {
    set_error("noise_patch: candidate budget exhausted before the stream was complete");
    return TDX_E_INVALID;
  }
  return TDX_OK;
}
