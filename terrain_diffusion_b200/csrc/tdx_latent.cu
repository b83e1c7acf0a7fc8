// The base model's embedding rows for the latent stage, computed on the device one CTA per row
// (world_pipeline.py:1018-1050 + edm_unet.py:145-159).  Every row is a function of its own coarse window only: the
// conditioning vector and both embedding dot products run in a fixed order that does not depend on how many rows the
// launch holds, so a batch-invariant latent solve gives every tile the bits of its one-tile solve.
#include <float.h>

#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

constexpr int kLatentCh = 7, kLatentCells = 16;           // packed coarse window [7][4][4]: 6 channels x w, then w
constexpr int kLatentHead = 52;                           // means(16) p5(16) climate(4) mask(16); tail = hist + level
constexpr int kLatentMaxCond = 128, kLatentMaxNoise = 512, kLatentMaxEmb = 1024, kLatentThreads = 256;

struct LatentEmbedParams {
  float* emb;                 // [n][E]
  float* cond_vec;            // [n][D] or null
  const float* coarse;        // [n][7][4][4]
  const float* means;         // [7]
  const float* stds;          // [7]
  const float* tail;          // [D - 52]: histogram, then noise level
  const float* scale;         // [D]: mp_concat's per-column scale
  const float* freqs;         // [noise_dims / 2]
  const float* noise_weight;  // [noise_dims][E]
  const float* cond_weight;   // [D][E]
  int D, noise_dims, E;
  float label, w_noise, w_cond, w_norm;
};

// silu(x) / 0.596 as torch computes silu in fp32: x / (1 + exp(-x)), each op rounded on its own
__device__ __forceinline__ float latent_mp_silu(float x) {
  return __fdiv_rn(__fdiv_rn(x, __fadd_rn(1.0f, expf(-x))), 0.596f);
}

// x = nan_to_num((cimg - mean) / std, nan=means[0]) of channel c at cell s, cimg = coarse[c] / coarse[6] (c < 6) or 1
__device__ __forceinline__ float latent_x(const float* win, const float* means, const float* stds, int c, int s) {
  const float ci = c < 6 ? __fdiv_rn(win[c * kLatentCells + s], win[6 * kLatentCells + s]) : 1.0f;
  const float x = __fdiv_rn(__fsub_rn(ci, means[c]), stds[c]);
  if (isnan(x)) return means[0];
  if (isinf(x)) return x > 0.f ? FLT_MAX : -FLT_MAX;
  return x;
}

__global__ void __launch_bounds__(kLatentThreads) latent_embed_kernel(const __grid_constant__ LatentEmbedParams p) {
  __shared__ float cv[kLatentMaxCond];
  __shared__ float pe[kLatentMaxNoise];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const float* win = p.coarse + (size_t)row * kLatentCh * kLatentCells;
  for (int k = threadIdx.x; k < p.D; k += blockDim.x) {
    float v;
    if (k < 32) {
      v = latent_x(win, p.means, p.stds, k >> 4, k & 15);                       // means, p5
    } else if (k < 36) {
      const int c = 2 + (k - 32);                                               // climate: mean of x[c, 1:3, 1:3]
      float s = latent_x(win, p.means, p.stds, c, 5);
      s = __fadd_rn(s, latent_x(win, p.means, p.stds, c, 6));
      s = __fadd_rn(s, latent_x(win, p.means, p.stds, c, 9));
      s = __fadd_rn(s, latent_x(win, p.means, p.stds, c, 10));
      v = __fmul_rn(s, 0.25f);
    } else if (k < kLatentHead) {
      v = latent_x(win, p.means, p.stds, 6, k - 36);                            // mask
    } else {
      v = p.tail[k - kLatentHead];                                              // histogram, noise level
    }
    v = __fmul_rn(v, p.scale[k]);
    cv[k] = v;
    if (p.cond_vec) p.cond_vec[(size_t)row * p.D + k] = v;
  }
  // MPPositionalEmbedding of the noise label (mp_layers.py:88-107), fp32, as embed_kernel computes it
  const int half = p.noise_dims >> 1;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float yv = __fmul_rn(p.label, p.freqs[i]);
    pe[i] = __fmul_rn(sinf(yv), 1.41421356237309515f);
    pe[half + i] = __fmul_rn(cosf(yv), 1.41421356237309515f);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < p.E; j += blockDim.x) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    for (int i = 0; i < p.noise_dims; i += 4) {
      s0 = fmaf(__ldg(p.noise_weight + (size_t)(i + 0) * p.E + j), pe[i + 0], s0);
      s1 = fmaf(__ldg(p.noise_weight + (size_t)(i + 1) * p.E + j), pe[i + 1], s1);
      s2 = fmaf(__ldg(p.noise_weight + (size_t)(i + 2) * p.E + j), pe[i + 2], s2);
      s3 = fmaf(__ldg(p.noise_weight + (size_t)(i + 3) * p.E + j), pe[i + 3], s3);
    }
    const float noise = __fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3));
    float c = 0.f;
    for (int k = 0; k < p.D; ++k) c = fmaf(__ldg(p.cond_weight + (size_t)k * p.E + j), cv[k], c);
    // mp_sum of the two embeddings with weights (w_noise, w_cond), then mp_silu
    const float sum = __fadd_rn(__fmul_rn(noise, p.w_noise), __fmul_rn(latent_mp_silu(c), p.w_cond));
    p.emb[(size_t)row * p.E + j] = latent_mp_silu(__fdiv_rn(sum, p.w_norm));
  }
}

}  // namespace tdx

using namespace tdx;

extern "C" int tdx_latent_embed(float* emb, float* cond_vec, const float* coarse, const float* cond_means,
                                const float* cond_stds, const float* tail, int32_t n_tail, const float* concat_scale,
                                const float* noise_freqs, const float* noise_weight, const float* cond_weight,
                                int32_t noise_dims, int32_t emb_channels, float label, float w_noise, float w_cond,
                                float w_norm, int32_t n_rows, void* stream) {
  TDX_REQUIRE(emb && coarse && cond_means && cond_stds && tail && concat_scale && noise_freqs && noise_weight &&
              cond_weight, "latent_embed: null pointer");
  TDX_REQUIRE(n_rows >= 1 && n_rows <= 65535, "latent_embed: n_rows=%d not in 1..65535", n_rows);
  TDX_REQUIRE(n_tail >= 1 && kLatentHead + n_tail <= kLatentMaxCond,
              "latent_embed: n_tail=%d not in 1..%d (the conditioning vector holds 52 + n_tail values)", n_tail,
              kLatentMaxCond - kLatentHead);
  TDX_REQUIRE(noise_dims >= 4 && noise_dims <= kLatentMaxNoise && noise_dims % 4 == 0,
              "latent_embed: noise_dims=%d must be a multiple of 4 in 4..%d", noise_dims, kLatentMaxNoise);
  TDX_REQUIRE(emb_channels >= 1 && emb_channels <= kLatentMaxEmb, "latent_embed: emb_channels=%d not in 1..%d",
              emb_channels, kLatentMaxEmb);
  TDX_REQUIRE(w_norm > 0.f, "latent_embed: the weight norm must be positive");
  LatentEmbedParams p;
  p.emb = emb;
  p.cond_vec = cond_vec;
  p.coarse = coarse;
  p.means = cond_means;
  p.stds = cond_stds;
  p.tail = tail;
  p.scale = concat_scale;
  p.freqs = noise_freqs;
  p.noise_weight = noise_weight;
  p.cond_weight = cond_weight;
  p.D = kLatentHead + n_tail;
  p.noise_dims = noise_dims;
  p.E = emb_channels;
  p.label = label;
  p.w_noise = w_noise;
  p.w_cond = w_cond;
  p.w_norm = w_norm;
  TDX_CHECK_CUDA(launch(latent_embed_kernel, dim3(n_rows), kLatentThreads, 0, stream, p));
  return TDX_OK;
}
