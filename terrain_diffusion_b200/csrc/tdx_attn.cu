// Cosine self-attention of the EDM2 block (reference: UNetBlock.attn, models/unet_block.py:102-108):
//   q, k, v = per-head pixel-norm over the 64 head channels of the 1x1 qkv projection
//   w = softmax_k(q^T k / sqrt(d)) ;  y = w v
// Only the latent (base) model has such a block, at 8x8 = 64 tokens x 12 heads x 64 channels (< 0.2 % of its FLOPs,
// SURVEY.md section 0 item 2), so this is a small CUDA-core kernel: one block per (head, image), one thread per
// query token, q/k/v of the head staged in shared memory as fp32.  The 1x1 projections around it run on the
// tensor-core implicit-GEMM kernel.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

struct AttnParams {
  const uint4* q;
  const uint4* k;
  const uint4* v;
  uint4* out;
  int heads, tokens, C8;   // C8 = heads * 8 channel groups
};

// layout: NC8HW8 -> element (channel c, token t) of image n at uint4 index ((n*C8 + c/8) * tokens + t), lane c%8
__global__ void __launch_bounds__(256) attn_kernel(const AttnParams p) {
  extern __shared__ float sm[];  // q[T][65], k[T][65], v[T][65]
  const int T = p.tokens;
  float* sq = sm;
  float* sk = sm + (size_t)T * 65;
  float* sv = sk + (size_t)T * 65;
  const int h = blockIdx.x, n = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  // stage + normalise: thread t owns token t
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const uint4* srcs[3] = {p.q, p.k, p.v};
    float* dsts[3] = {sq, sk, sv};
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      float vals[64];
      float ss = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const uint4 u = __ldg(srcs[w] + ((size_t)n * p.C8 + h * 8 + g) * T + t);
        unpack_bf16x2(u.x, vals[g * 8 + 0], vals[g * 8 + 1]);
        unpack_bf16x2(u.y, vals[g * 8 + 2], vals[g * 8 + 3]);
        unpack_bf16x2(u.z, vals[g * 8 + 4], vals[g * 8 + 5]);
        unpack_bf16x2(u.w, vals[g * 8 + 6], vals[g * 8 + 7]);
      }
#pragma unroll
      for (int d = 0; d < 64; ++d) ss = fmaf(vals[d], vals[d], ss);
      const float inv = 1.0f / (1e-4f + sqrtf(ss * (1.0f / 64.0f)));   // normalize(y, dim=2): x / (eps + rms)
#pragma unroll
      for (int d = 0; d < 64; ++d) dsts[w][(size_t)t * 65 + d] = vals[d] * inv;
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    float qv[64];
#pragma unroll
    for (int d = 0; d < 64; ++d) qv[d] = sq[(size_t)t * 65 + d] * 0.125f;   // 1/sqrt(64)
    // two passes over the keys: max, then exp-sum and weighted values (T is tiny)
    float mx = -1e30f;
    for (int kk = 0; kk < T; ++kk) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) s = fmaf(qv[d], sk[(size_t)kk * 65 + d], s);
      mx = fmaxf(mx, s);
    }
    float acc[64];
#pragma unroll
    for (int d = 0; d < 64; ++d) acc[d] = 0.f;
    float den = 0.f;
    for (int kk = 0; kk < T; ++kk) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) s = fmaf(qv[d], sk[(size_t)kk * 65 + d], s);
      const float e = expf(s - mx);
      den += e;
#pragma unroll
      for (int d = 0; d < 64; ++d) acc[d] = fmaf(e, sv[(size_t)kk * 65 + d], acc[d]);
    }
    const float r = 1.0f / den;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      uint4 u;
      u.x = pack_bf16x2(acc[g * 8 + 0] * r, acc[g * 8 + 1] * r);
      u.y = pack_bf16x2(acc[g * 8 + 2] * r, acc[g * 8 + 3] * r);
      u.z = pack_bf16x2(acc[g * 8 + 4] * r, acc[g * 8 + 5] * r);
      u.w = pack_bf16x2(acc[g * 8 + 6] * r, acc[g * 8 + 7] * r);
      p.out[((size_t)n * p.C8 + h * 8 + g) * T + t] = u;
    }
  }
}

int attn_validate(const TdxAttnDesc& d) {
  TDX_REQUIRE(d.q && d.k && d.v && d.out, "attn: null pointer");
  TDX_REQUIRE(d.head_dim == 64, "attn: head_dim=%d (only 64, the reference's channels_per_head)", d.head_dim);
  TDX_REQUIRE(d.heads >= 1 && d.n_img >= 1 && d.tokens >= 1, "attn: bad shape");
  TDX_REQUIRE((size_t)d.tokens * 65 * 3 * 4 <= 200 * 1024, "attn: %d tokens exceed the shared-memory plan (<= 262)",
              d.tokens);
  return TDX_OK;
}

int attn_prepare() {
  static bool seen[16] = {false};
  if (first_use_on_device(seen)) {
    TDX_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  return TDX_OK;
}

int attn_launch(const TdxAttnDesc& d, cudaStream_t stream) {
  int rc = attn_prepare();
  if (rc != TDX_OK) return rc;
  AttnParams p;
  p.q = reinterpret_cast<const uint4*>(d.q);
  p.k = reinterpret_cast<const uint4*>(d.k);
  p.v = reinterpret_cast<const uint4*>(d.v);
  p.out = reinterpret_cast<uint4*>(d.out);
  p.heads = d.heads;
  p.tokens = d.tokens;
  p.C8 = d.heads * 8;
  const int threads = d.tokens < 256 ? ((d.tokens + 31) / 32) * 32 : 256;
  TDX_CHECK_CUDA(launch(attn_kernel, dim3(d.heads, d.n_img), threads, (size_t)d.tokens * 65 * 3 * 4, stream, p));
  return TDX_OK;
}

}  // namespace tdx

extern "C" int tdx_attn_run(const TdxAttnDesc* d, void* stream) {
  if (!d) { tdx::set_error("attn: null descriptor"); return TDX_E_INVALID; }
  int rc = tdx::attn_validate(*d);
  if (rc != TDX_OK) return rc;
  return tdx::attn_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
