// Terrain read-out of the generative evaluations (evaluation/base_consistency.py:34-72 `_decode_latents_to_terrain`
// and its copies in base_diffusion.py and the infinite_consistency*.py drivers): after the consistency decode, every
// image's residual and low-frequency planes are de-normalised, optionally Laplacian-denoised (laplacian_denoise,
// sigma 5) and recombined (laplacian_decode with extrapolation).  The reference runs this through torchvision on
// [B, 1, H, W]; the single-plane chain of inference/postproc.py takes one plane per call.  Here every step is one
// launch over the whole batch (the plane is the grid's z axis), with the per-element arithmetic of tdx_post.cu
// (tdx_post.cuh), so each plane is bit-identical to that chain.  HBM-bound and small next to the decoder U-Net.
#include "tdx_common.h"
#include "tdx_post.cuh"
#include "tdx_ptx.cuh"

namespace tdx {

// pad_linear_extrapolation of x [n][h][w] (plane stride x_plane; de-normalised on read as x * scale + offset when
// `affine`) into out, plane stride out_plane.
__global__ void eval_pad_kernel(const float* __restrict__ x, long x_plane, int h, int w, int affine, float scale,
                                float offset, float* __restrict__ out, long out_plane) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= w + 2 || oy >= h + 2) return;
  const float* xp = x + (long)blockIdx.z * x_plane;
  const auto ld = [&](int r, int c) {
    const float v = xp[(long)r * w + c];
    return affine ? __fadd_rn(__fmul_rn(v, scale), offset) : v;
  };
  out[(long)blockIdx.z * out_plane + (long)oy * (w + 2) + ox] = pad_extrapolate_at(ld, h, w, oy, ox);
}

// One anti-aliased bilinear axis of x [n][h][w] (plane stride x_plane) into out (plane stride out_plane).
__global__ void eval_resize_kernel(const float* __restrict__ x, long x_plane, int h, int w, float* __restrict__ out,
                                   long out_plane, int out_size, int axis) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  const int oh = axis == 0 ? out_size : h, ow = axis == 1 ? out_size : w;
  if (ox >= ow || oy >= oh) return;
  out[(long)blockIdx.z * out_plane + (long)oy * ow + ox] =
      resize_aa_at(x + (long)blockIdx.z * x_plane, h, w, out_size, axis, oy, ox);
}

__global__ void eval_blur_kernel(const float* __restrict__ x, long x_plane, int h, int w, float* __restrict__ out,
                                 long out_plane, const BlurParams bp) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= w || oy >= h) return;
  out[(long)blockIdx.z * out_plane + (long)oy * w + ox] =
      gaussian_blur_at(x + (long)blockIdx.z * x_plane, h, w, bp, oy, ox);
}

// out = f(residual * scale + offset + up[oi + y][oj + x]) over [n][H][W]; up has plane stride up_plane and row pitch
// up_pitch.  f = sign(v) v^2 with signed_sq, else the identity.
__global__ void eval_combine_kernel(const float* __restrict__ residual, float scale, float offset,
                                    const float* __restrict__ up, long up_plane, int up_pitch, int oi, int oj,
                                    float* __restrict__ out, long out_plane, int H, int W, int signed_sq) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W || y >= H) return;
  const long p = blockIdx.z;
  out[p * out_plane + (long)y * W + x] = denorm_combine(residual[p * H * W + (long)y * W + x], scale, offset,
                                                        up[p * up_plane + (long)(y + oi) * up_pitch + x + oj], signed_sq);
}

// The decoder evaluations' read-out of pre-padded low-frequency planes: out[p][y][x] over the [ch][cw] crop at (cy, cx)
// = f(residual[p][cy + y][cx + x] * scale + offset + up[cy + y + 8][cx + x + 8]), where up is the height pass of the
// (H + 16) x (W + 16) resize, evaluated here from the width pass tmp [lh][W + 16] (plane stride tmp_plane) only where
// the crop reads it.
__global__ void eval_padded_combine_kernel(const float* __restrict__ residual, float scale, float offset,
                                           const float* __restrict__ tmp, long tmp_plane, int lh, int H, int W,
                                           int cy, int cx, float* __restrict__ out, int ch, int cw, int signed_sq) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= cw || y >= ch) return;
  const long p = blockIdx.z;
  const float up = resize_aa_at(tmp + p * tmp_plane, lh, W + 16, H + 16, 0, cy + y + 8, cx + x + 8);
  out[p * ch * cw + (long)y * cw + x] =
      denorm_combine(residual[p * H * W + (long)(cy + y) * W + cx + x], scale, offset, up, signed_sq);
}

namespace {

// resize_extrapolated's geometry (laplacian_encoder.py:42-60) for an lh x lw plane and a th x tw target: the resized
// padded size (rh, rw) and the crop origin (ph, pw).  Python's round() is round-half-even, as nearbyint is here.
struct ExtrapGeom {
  int rh, rw, ph, pw;
};
ExtrapGeom extrap_geom(int lh, int lw, int th, int tw) {
  const double sh = (double)th / lh, sw = (double)tw / lw;
  return {(int)nearbyint(th + 2 * sh), (int)nearbyint(tw + 2 * sw), (int)nearbyint(sh), (int)nearbyint(sw)};
}

// torchvision's resize to an int size: the shorter edge becomes `size`, the longer one int(size * long / short).
void short_edge_size(int h, int w, int size, int* nh, int* nw) {
  if (w <= h) {
    *nw = size;
    *nh = (int)((double)size * h / w);
  } else {
    *nh = size;
    *nw = (int)((double)size * w / h);
  }
}

bool overlaps(const float* a, int64_t na, const float* b, int64_t nb) { return a < b + nb && b < a + na; }

// The batch's launches.  Two scratch plane sets of `plane` floats per image; `cur` holds the latest intermediate.
struct Readout {
  int n, H, W;
  float residual_mean, residual_std;
  float* buf[2];
  long plane;
  int cur;
  void* stream;

  dim3 grid(int ow, int oh) const { return dim3((ow + 127) / 128, oh, n); }

  // resize_bilinear of buf[cur] (ch x cw planes) to th x tw: width pass, then height pass, each skipped when the size
  // does not change.  Updates ch, cw and cur.
  cudaError_t resize(int* ch, int* cw, int th, int tw) {
    if (tw != *cw) {
      cudaError_t e = launch(eval_resize_kernel, grid(tw, *ch), 128, 0, stream, (const float*)buf[cur], plane, *ch,
                             *cw, buf[cur ^ 1], plane, tw, 1);
      if (e != cudaSuccess) return e;
      *cw = tw;
      cur ^= 1;
    }
    if (th != *ch) {
      cudaError_t e = launch(eval_resize_kernel, grid(*cw, th), 128, 0, stream, (const float*)buf[cur], plane, *ch,
                             *cw, buf[cur ^ 1], plane, th, 0);
      if (e != cudaSuccess) return e;
      *ch = th;
      cur ^= 1;
    }
    return cudaSuccess;
  }

  // laplacian_decode(residual * std + mean, lo, extrapolate=True) into dst (plane stride dst_plane), or, for a NULL
  // dst, into the free plane set, which then becomes buf[cur]: pad lo [n][lh][lw] (plane stride lo_plane,
  // de-normalised on read when lo_affine; not in buf[cur ^ 1]) into buf[cur ^ 1], resize to the padded target, add
  // the crop to the residual.
  cudaError_t decode(const float* residual, const float* lo, long lo_plane, int lh, int lw, int lo_affine,
                     float lo_scale, float lo_offset, float* dst, long dst_plane, int signed_sq) {
    cudaError_t e = launch(eval_pad_kernel, grid(lw + 2, lh + 2), 128, 0, stream, lo, lo_plane, lh, lw, lo_affine,
                           lo_scale, lo_offset, buf[cur ^ 1], plane);
    if (e != cudaSuccess) return e;
    cur ^= 1;
    const ExtrapGeom g = extrap_geom(lh, lw, H, W);
    int ch = lh + 2, cw = lw + 2;
    if ((e = resize(&ch, &cw, g.rh, g.rw)) != cudaSuccess) return e;
    float* to = dst ? dst : buf[cur ^ 1];
    e = launch(eval_combine_kernel, grid(W, H), 128, 0, stream, residual, residual_std, residual_mean,
               (const float*)buf[cur], plane, cw, g.ph, g.pw, to, dst ? dst_plane : plane, H, W, signed_sq);
    if (!dst) cur ^= 1;
    return e;
  }
};

}  // namespace
}  // namespace tdx

using namespace tdx;

extern "C" int tdx_eval_terrain(const float* residual, const float* lowfreq, int32_t n, int32_t h, int32_t w,
                                float residual_mean, float residual_std, float lowfreq_mean, float lowfreq_std,
                                int32_t denoise, int32_t signed_square, float* out, float* scratch,
                                int64_t scratch_elems, void* stream) {
  TDX_REQUIRE(residual && lowfreq && out && scratch, "eval_terrain: null pointer");
  TDX_REQUIRE(n >= 1 && n <= 65535, "eval_terrain: batch of %d images (1..65535)", n);
  TDX_REQUIRE(h >= 1 && w >= 1 && 8 * (int64_t)h + 16 <= 65535 && w <= (1 << 24),
              "eval_terrain: bad low-frequency shape %d x %d", h, w);
  const int H = 8 * h, W = 8 * w;
  const long plane = (long)(H + 16) * (W + 16);
  const int64_t need = 2 * (int64_t)n * plane;
  TDX_REQUIRE(scratch_elems >= need, "eval_terrain: scratch holds %lld floats, %d images of %d x %d need %lld",
              (long long)scratch_elems, n, h, w, (long long)need);
  const int64_t n_res = (int64_t)n * H * W, n_low = (int64_t)n * h * w;
  TDX_REQUIRE(!overlaps(out, n_res, residual, n_res) && !overlaps(out, n_res, lowfreq, n_low) &&
                  !overlaps(out, n_res, scratch, need) && !overlaps(scratch, need, residual, n_res) &&
                  !overlaps(scratch, need, lowfreq, n_low),
              "eval_terrain: out and scratch must not overlap each other or the inputs");
  int nh = h, nw = w;
  if (denoise) {
    // laplacian_encode resizes the decoded [H][W] plane to the INT size w: the shorter edge becomes w
    short_edge_size(H, W, w, &nh, &nw);
    TDX_REQUIRE(nh <= H && nw <= W, "eval_terrain: denoising would resize the %d x %d plane up to %d x %d (the image "
                "is more than 8 times wider than high)", H, W, nh, nw);
    TDX_REQUIRE(nh > 5 && nw > 5,
                "eval_terrain: denoising blurs a %d x %d plane; reflect padding of 5 needs both sides larger", nh, nw);
  }

  Readout r;
  r.n = n; r.H = H; r.W = W;
  r.residual_mean = residual_mean; r.residual_std = residual_std;
  r.plane = plane;
  r.buf[0] = scratch;
  r.buf[1] = scratch + (int64_t)n * plane;
  r.cur = 1;
  r.stream = stream;
  if (!denoise) {
    TDX_CHECK_CUDA(r.decode(residual, lowfreq, (long)h * w, h, w, 1, lowfreq_std, lowfreq_mean, out, (long)H * W,
                            signed_square));
    return TDX_OK;
  }
  // laplacian_denoise(sigma=5): decoded = laplacian_decode(residual, lowfreq, extrapolate=True) ...
  TDX_CHECK_CUDA(r.decode(residual, lowfreq, (long)h * w, h, w, 1, lowfreq_std, lowfreq_mean, nullptr, 0, 0));
  // ... resized to nh x nw and blurred with kernel_size_for(5) = 11, sigma 5 ...
  int ch = H, cw = W;
  TDX_CHECK_CUDA(r.resize(&ch, &cw, nh, nw));
  TDX_CHECK_CUDA(launch(eval_blur_kernel, r.grid(nw, nh), 128, 0, stream, (const float*)r.buf[r.cur], plane, nh, nw,
                        r.buf[r.cur ^ 1], plane, gaussian_blur_params(11, 5.0f)));
  r.cur ^= 1;
  // ... then laplacian_decode(residual, denoised lowfreq, extrapolate=True)
  TDX_CHECK_CUDA(r.decode(residual, r.buf[r.cur], plane, nh, nw, 0, 1.f, 0.f, out, (long)H * W, signed_square));
  return TDX_OK;
}

// The decoder evaluations' read-out (evaluation/decoder_consistency.py:183-196, tiled_decoder_consistency.py:185-196):
// laplacian_decode(residual * std + mean, lowfreq_padded, pre_padded=True) (laplacian_encoder.py:93-132), whose low-
// frequency plane arrives with its one-pixel border: resized to (H + 16) x (W + 16), cropped by pad_pixels = W / w = 8
// on every side.  Then the optional signed square and centre crop.  Two launches over the whole batch: the width pass
// into scratch, then the height pass fused with the combine and the crop.
extern "C" int tdx_eval_padded_terrain(const float* residual, const float* lowfreq_padded, int32_t n, int32_t h,
                                       int32_t w, float residual_mean, float residual_std, int32_t signed_square,
                                       int32_t crop, float* out, float* scratch, int64_t scratch_elems, void* stream) {
  TDX_REQUIRE(residual && lowfreq_padded && out && scratch, "eval_padded_terrain: null pointer");
  TDX_REQUIRE(n >= 1 && n <= 65535, "eval_padded_terrain: batch of %d planes (1..65535)", n);
  TDX_REQUIRE(h >= 1 && w >= 1 && 8 * (int64_t)h + 16 <= 65535 && w <= (1 << 24),
              "eval_padded_terrain: bad low-frequency shape %d x %d (before its padding)", h, w);
  const int H = 8 * h, W = 8 * w;
  TDX_REQUIRE(crop >= 0 && crop <= H && crop <= W, "eval_padded_terrain: crop %d of a %d x %d plane", crop, H, W);
  const int ch = crop ? crop : H, cw = crop ? crop : W;
  const long tmp_plane = (long)(h + 2) * (W + 16);
  const int64_t need = (int64_t)n * tmp_plane;
  TDX_REQUIRE(scratch_elems >= need, "eval_padded_terrain: scratch holds %lld floats, %d planes of %d x %d need %lld",
              (long long)scratch_elems, n, h, w, (long long)need);
  const int64_t n_res = (int64_t)n * H * W, n_low = (int64_t)n * (h + 2) * (w + 2), n_out = (int64_t)n * ch * cw;
  TDX_REQUIRE(!overlaps(out, n_out, residual, n_res) && !overlaps(out, n_out, lowfreq_padded, n_low) &&
                  !overlaps(out, n_out, scratch, need) && !overlaps(scratch, need, residual, n_res) &&
                  !overlaps(scratch, need, lowfreq_padded, n_low),
              "eval_padded_terrain: out and scratch must not overlap each other or the inputs");
  TDX_CHECK_CUDA(launch(eval_resize_kernel, dim3((W + 16 + 127) / 128, h + 2, n), 128, 0, stream, lowfreq_padded,
                        (long)(h + 2) * (w + 2), h + 2, w + 2, scratch, tmp_plane, W + 16, 1));
  TDX_CHECK_CUDA(launch(eval_padded_combine_kernel, dim3((cw + 127) / 128, ch, n), 128, 0, stream, residual,
                        residual_std, residual_mean, (const float*)scratch, tmp_plane, h + 2, H, W, (H - ch) / 2,
                        (W - cw) / 2, out, ch, cw, (int)signed_square));
  return TDX_OK;
}
