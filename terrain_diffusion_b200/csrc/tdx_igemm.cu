// Persistent, warp-specialised implicit-GEMM convolution for sm_90a.
//
//   D[128 pixels x N channels] (fp32) += A[128 x 16] (bf16, smem halo patch) * B[N x 16] (bf16, smem weights)
//
// * Work item = (M tile of 16 rows x 8 columns of output pixels) x (N-channel slice of Cout, N = 64 .. 256).  The
//   slices of one M tile are adjacent work items, so they run concurrently on neighbouring CTAs and share the A patch
//   in L2; small layers (32x32, 64x64 resolution) get Cout/N times more CTAs this way.
// * The A operand of every filter tap is the SAME (18 x 10)-pixel halo patch in shared memory: activations are stored
//   NC8HW8, so TMA drops the patch as [kc][18][10][8ch] and the wgmma K-major/no-swizzle descriptor (8-row core
//   matrices 128 B contiguous, SBO = 10 px * 16 B between pixel rows, LBO = one 8-channel plane) addresses tap (r,c)
//   by just adding (r*10+c)*16 B to the start address.  The patch is fetched once per 64-channel chunk and used by all
//   9 taps (1.4x halo overhead instead of 9x re-fetch); conv zero padding is TMA out-of-bounds fill.
// * B (weights) are pre-packed on the host in exactly the shared-memory image order, one stage per (chunk, tap), and
//   streamed with 1-D bulk copies through their own ring.
// * Warp roles: w0 A-producer (TMA tiled), w1 B-producer (bulk copy), w2 barrier set-up, w4..w11 two consumer
//   warpgroups.  Warpgroup g issues m64nNk16 wgmmas for pixels 64g .. 64g+63 (tile rows 8g .. 8g+7) with the
//   accumulator in registers, then writes it to a shared-memory staging tile (fp32, [channel][pixel]) from which all
//   eight warps run the epilogue with one thread per pixel.  The producers keep filling the rings for the next item
//   while the epilogue runs.
// * Epilogue: each thread owns one pixel; it applies emb-scale+mp_silu / residual mp_sum + clip / pixel-norm and
//   writes up to three bf16 NC8HW8 outputs (raw, activated, activated+resampled) for the consumers.  Pixel-norm needs
//   the sum of squares over ALL Cout channels: the Cout/N CTAs of one M tile are then launched as a thread-block
//   cluster and exchange their per-pixel partial sums through distributed shared memory + a cluster-scope mbarrier.
// * Programmatic dependent launch: barrier init, descriptor prefetch and the weight stream of kernel N+1 overlap the
//   tail of kernel N; griddepcontrol.wait guards everything that depends on earlier kernels.
//
// Reference math being replaced: models/mp_layers.py:201-221 (MPConv), models/unet_block.py:116-156 (UNetBlock).
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

constexpr int kTileH = 16, kTileW = 8;
constexpr int kPatchH = kTileH + 2, kPatchW = kTileW + 2;
constexpr int kKcBytes = kPatchH * kPatchW * 16;  // one 8-channel plane of the halo patch: 2880 B
constexpr int kAStageBytes = 8 * kKcBytes;        // 64 channels: 23040 B
constexpr int kSA = 3;                            // A ring depth (max; 2 when the staging tile leaves no room)
constexpr int kMaxSB = 18;                        // B ring depth (max; also the largest resident weight set)
constexpr int kWQ = 2;                            // epilogue warps per 32-pixel quadrant
constexpr int kEpiWarps = 4 * kWQ;                // = the two consumer warpgroups
constexpr int kChunk = 32;                        // accumulator columns an epilogue warp handles at a time
constexpr int kGroups = kChunk / 8;               // 8-channel groups (one uint4 of bf16) per chunk
constexpr int kThreads = 128 + 32 * kEpiWarps;
constexpr int kMaxSplit = 8;                      // max CTAs (cluster size) sharing one M tile's pixel-norm statistics
constexpr int kSmemMisc = 14336;                  // barriers, pixel-norm statistics
constexpr int kSmemBudget = 227 * 1024;
// Staging tile row pitch in floats: the 4 lanes of a wgmma fragment quad write channels 2 apart, 264 words = 8 banks
// apart, so a warp's fragment store and the epilogue's per-pixel loads are both free of bank conflicts.
constexpr int kStgLd = 132;

// Division by a launch constant with a host-made reciprocal: exact while n * d < 2^32 (all uses divide blockIdx.x-sized
// numbers); keeps runtime integer divisions (~150 cycles each) off the launch's critical path.
struct FastDiv {
  uint32_t d, magic;
};
static FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = (uint32_t)d;
  f.magic = d <= 1 ? 0u : (uint32_t)(0xFFFFFFFFull / (uint32_t)d + 1ull);
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t n, const FastDiv& f) { return f.d == 1 ? n : __umulhi(n, f.magic); }

struct IgemmParams {
  int nseg;
  int seg_chunks[3];
  int seg_taps[3];
  const __nv_bfloat16* B;
  int cout, nsplit;
  float inv_cout;
  int ncta;                   // output channels per work item = MMA N (64, 128, 192 or 256); cout = ncta * nsplit
  int SA;                     // A ring depth
  int SB;                     // B ring depth
  int b_stage_bytes;          // ncta * 128
  int resident;               // the whole weight set of an item fits the ring: loaded once per CTA, reused by every item
  int bgroup;                 // taps per weight hand-over group (9, 3 or 1): one full-barrier per group
  int ksplit;                 // split-K: the (chunk, tap) stages of a work item are shared by the ksplit CTAs of a cluster
  float* ws;                  // split-K fp32 partial sums [group][dst part][ksplit-1 sources][ncta/ksplit cols][128 pixels]
  int H, W, nimg, tiles_x, tiles_y, num_items;
  FastDiv fd_ks, fd_nsplit, fd_per, fd_tx, fd_ty;   // ksplit, nsplit, nsplit*ksplit, tiles_x, tiles_y
  int dtx, dty, dimg;                               // the per-iteration tile step gridDim.x / (nsplit*ksplit), decomposed
  int stages_per_item;
  int epi;
  int cluster_stats;          // pixel-norm statistics are exchanged across the xsplit CTAs of a cluster
  int xsplit;                 // CTAs that together hold all Cout channels of an M tile (= cluster size when cluster_stats)
  const float* cvec;
  const uint4* resid;
  int resid_spatial, resid_pnorm;
  float resid_scale, clip;
  TdxOutSpec out[3];
  float* rms_out;             // optional fp32 [nimg][H][W]: 1 / (eps + rms) of this launch's result
  const float* resid_inv;     // optional fp32 plane at the residual's resolution: r' = r * resid_inv[pixel]
  unsigned long long* timeline;  // debug: [2] = {first CTA start, last CTA end} in globaltimer ns, normally null
  unsigned long long* trace;  // debug: per-item phase timestamps of CTA 0 (tools/trace_igemm.py), normally null
};

// K is walked in "stages" (one tap of one 64-channel chunk, in packed-weight order).
// flat stage index -> (segment, chunk in segment, tap, taps of that segment)
__device__ __forceinline__ void stage_locate(const IgemmParams& p, int s, int& seg, int& ch, int& tap, int& taps) {
  int base = 0;
  for (seg = 0;; ++seg) {
    taps = p.seg_taps[seg];
    const int n = p.seg_chunks[seg] * taps;
    if (s < base + n || seg == p.nseg - 1) break;
    base += n;
  }
  ch = taps == 9 ? (s - base) / 9 : (s - base);
  tap = (s - base) - ch * taps;
}

// Debug hooks (per-item phase clocks, in-graph launch timeline: tools/trace_igemm.py, tools/timeline_forward.py) are
// compiled in only with -DTDX_DEBUG_HOOKS=1 (TDX_DEBUG_HOOKS=1 python -m terrain_diffusion_b200.build): in the
// production kernel they would cost ~40 instructions per item and epilogue warp.
#ifndef TDX_DEBUG_HOOKS
#define TDX_DEBUG_HOOKS 0
#endif
#if TDX_DEBUG_HOOKS
#define TDX_TRACE(slot, it)                                                                  \
  do {                                                                                       \
    if (p.trace && blockIdx.x == 0 && (it) < 16) p.trace[(it) * 8 + (slot)] = clock64();     \
  } while (0)
#else
#define TDX_TRACE(slot, it) do { } while (0)
#endif

// item = ((tile * nsplit) + split) * ksplit + kpart.  A CTA's items are blockIdx.x, blockIdx.x + gridDim.x, ...;
// gridDim.x is a multiple of nsplit * ksplit, so the channel slice and the K part are fixed per CTA and only the M tile
// advances -- by a constant step, which is tracked here without per-item divisions.
struct TileWalk {
  int tx, ty, img;      // current M tile
  int dtx, dty, dimg;   // the tile step, decomposed (dtx < tiles_x, dty < tiles_y)
  int split, kpart;
  __device__ __forceinline__ void init(const IgemmParams& p) {
    const uint32_t b = blockIdx.x;
    const uint32_t bk = fdiv(b, p.fd_ks);
    kpart = (int)(b - bk * p.fd_ks.d);
    split = (int)(bk - fdiv(bk, p.fd_nsplit) * p.fd_nsplit.d);
    const uint32_t t = fdiv(b, p.fd_per);
    const uint32_t t1 = fdiv(t, p.fd_tx);
    tx = (int)(t - t1 * p.fd_tx.d);
    const uint32_t t2 = fdiv(t1, p.fd_ty);
    ty = (int)(t1 - t2 * p.fd_ty.d);
    img = (int)t2;
    dtx = p.dtx;
    dty = p.dty;
    dimg = p.dimg;
  }
  __device__ __forceinline__ void next(const IgemmParams& p) {
    tx += dtx;
    int c = tx >= p.tiles_x ? 1 : 0;
    tx -= c ? p.tiles_x : 0;
    ty += dty + c;
    c = ty >= p.tiles_y ? 1 : 0;
    ty -= c ? p.tiles_y : 0;
    img += dimg + c;
  }
};
// this CTA's share [s0, s1) of an item's K stages (constant per CTA)
__device__ __forceinline__ void stage_range(const IgemmParams& p, int kpart, int& s0, int& s1) {
  s0 = (int)fdiv((uint32_t)(p.stages_per_item * kpart), p.fd_ks);
  s1 = (int)fdiv((uint32_t)(p.stages_per_item * (kpart + 1)), p.fd_ks);
}

// ---------------------------------------------------------------------------------------------- cluster helpers
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t remote_bar_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote_bar_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------- epilogue helpers
// kChunk accumulator columns from `col` of pixel m, out of the staging tile
__device__ __forceinline__ void load_acc(const float* stg, int m, int col, float (&v)[kChunk]) {
#pragma unroll
  for (int i = 0; i < kChunk; ++i) v[i] = stg[(col + i) * kStgLd + m];
}

// 1 / (eps + sqrt(mean square)) with the two MUFU approximations (relative error ~2^-22: invisible after bf16 rounding)
__device__ __forceinline__ float inv_rms(float sumsq, float inv_n) {
  float s;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(s) : "f"(sumsq * inv_n));
  return __fdividef(1.0f, 1e-4f + s);
}

// One output of one chunk: kChunk channels of this thread's pixel -> bf16, optionally through mp_silu, one uint4 per
// 8-channel group (plane stride `plane`), replicated 2x2 for nearest-neighbour upsampling outputs.
__device__ __forceinline__ void store_chunk(uint4* dst, uint32_t plane, int Wo, int kind, int spatial, bool active,
                                            const float (&v)[kChunk], float hs, float hsk) {
  uint4 u[kGroups];
  if (kind == TDX_OUT_RAW) {
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      u[g].x = pack_bf16x2(v[g * 8 + 0], v[g * 8 + 1]);
      u[g].y = pack_bf16x2(v[g * 8 + 2], v[g * 8 + 3]);
      u[g].z = pack_bf16x2(v[g * 8 + 4], v[g * 8 + 5]);
      u[g].w = pack_bf16x2(v[g * 8 + 6], v[g * 8 + 7]);
    }
  } else {
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      float w[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) w[i] = mp_silu_scaled(v[g * 8 + i], hs, hsk);
      u[g].x = pack_bf16x2(w[0], w[1]);
      u[g].y = pack_bf16x2(w[2], w[3]);
      u[g].z = pack_bf16x2(w[4], w[5]);
      u[g].w = pack_bf16x2(w[6], w[7]);
    }
  }
  if (!active) return;
  if (spatial == TDX_SP_UP2) {
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      uint4* d = dst + (size_t)g * plane;
      d[0] = u[g];
      d[1] = u[g];
      d[Wo] = u[g];
      d[Wo + 1] = u[g];
    }
  } else {
#pragma unroll
    for (int g = 0; g < kGroups; ++g) dst[(size_t)g * plane] = u[g];
  }
}

// Ring positions of the consumer warpgroups (every consumer thread keeps the same copy).
struct ConsumerRing {
  int sa, sb;
  uint32_t pha;     // a_full parity
  uint32_t fmask;   // expected parity of every b_full barrier (a hand-over group's barrier = its first slot's)
};

// One work item's K stages [s0, s1) on the tensor cores.  Consumer warpgroup wg computes pixels 64 wg .. 64 wg + 63
// against all kN channels of the item, then stores its accumulator into the staging tile stg[channel * kStgLd + pixel].
template <int kN>
__device__ __forceinline__ void mma_item(const IgemmParams& p, const uint8_t* a_ring, const uint8_t* b_ring,
                                         uint64_t* a_full, uint64_t* a_empty, uint64_t* b_full, uint64_t* b_empty,
                                         ConsumerRing& r, int s0, int s1, bool steady, float* stg) {
  const int lane = threadIdx.x & 31, wl = (threadIdx.x >> 5) & 3, wg = (int)(threadIdx.x >> 7) - 1;
  float acc[kN / 2];
#pragma unroll
  for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
  constexpr uint32_t b_lbo = kN * 16;
  const uint32_t a_base = smem_u32(a_ring) + wg * 8 * kPatchW * 16;
  const uint32_t b_base = smem_u32(b_ring);
  // A stage's ring slots are released one stage late, so one stage is in flight while the next is issued.  A one-slot
  // weight ring cannot wait like that: its only slot is the one the next stage needs.
  const bool deep = p.SB > 1 || p.resident;
  int pend_a = -1, pend_b = -1;
  auto release = [&](int a, int b) {
    __syncwarp();
    if (lane == 0) {
      if (b >= 0) mbar_arrive(&b_empty[b]);
      if (a >= 0) mbar_arrive(&a_empty[a]);
    }
  };
  for (int s = s0; s < s1;) {
    int seg, ch, tap0, taps;
    stage_locate(p, s, seg, ch, tap0, taps);
    const int tap1 = (taps - tap0 < s1 - s) ? taps : tap0 + (s1 - s);
    const int nt = tap1 - tap0;
    s += nt;
    mbar_wait(&a_full[r.sa], r.pha);
    const uint32_t a_stage = a_base + r.sa * kAStageBytes;
    // tap offsets (r * 10 + c pixels) come from a packed table, 5 bits per tap; a 1x1 segment reads the patch centre
    unsigned long long tt = taps == 9 ? (0x16ad18b50820ull >> (5 * tap0)) : (unsigned long long)(kPatchW + 1);
    // hand-over groups of up to `bgroup` taps (one group = everything when the weights are already resident)
    const int gsz = steady ? nt : p.bgroup;
    int t = 0;
    for (int g0 = 0; g0 < nt; g0 += gsz) {
      const int gn = nt - g0 < gsz ? nt - g0 : gsz;
      if (!steady) {
        mbar_wait(&b_full[r.sb], (r.fmask >> r.sb) & 1u);
        r.fmask ^= 1u << r.sb;
      }
      for (int k = 0; k < gn; ++k, ++t, tt >>= 5) {
        const uint32_t al = a_stage + (uint32_t)(tt & 31ull) * 16;
        const uint32_t bl = b_base + r.sb * p.b_stage_bytes;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j)
          wgmma_bf16<kN>(acc, make_smem_desc(al + j * 2 * kKcBytes, kKcBytes, kPatchW * 16),
                         make_smem_desc(bl + j * 2 * b_lbo, b_lbo, 128), 1u);
        wgmma_commit();
        const int rel_b = p.resident ? -1 : r.sb;
        const int rel_a = t == nt - 1 ? r.sa : -1;   // the chunk's last tap frees its halo patch
        if (deep) {
          wgmma_wait<1>();
          release(pend_a, pend_b);
          pend_a = rel_a;
          pend_b = rel_b;
        } else {
          wgmma_wait<0>();
          release(rel_a, rel_b);
        }
        if (++r.sb == p.SB) r.sb = 0;
      }
    }
    if (++r.sa == p.SA) { r.sa = 0; r.pha ^= 1; }
  }
  wgmma_wait<0>();
  release(pend_a, pend_b);
  named_bar_sync(13, 32 * kEpiWarps);   // the previous item's epilogue has read the staging tile
  float* dst = stg + 64 * wg + 16 * wl + (lane >> 2);
#pragma unroll
  for (int j = 0; j < kN / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) dst[(8 * j + 2 * (lane & 3) + c) * kStgLd + 8 * i] = acc[4 * j + 2 * i + c];
  named_bar_sync(13, 32 * kEpiWarps);
}

// kCL = the launch uses clusters (split-K and / or pixel-norm statistics across CTAs).  The many-item launches do not:
// their instantiation carries none of that code (a shorter epilogue loop, fewer instruction-cache misses).
// kN = output channels per work item (the wgmma N).
template <bool kCL, int kN>
__global__ void __launch_bounds__(kThreads, 1)
igemm_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
             const __grid_constant__ CUtensorMap tm2, const __grid_constant__ IgemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int ksplit_ = kCL ? p.ksplit : 1;
  const bool cstats_ = kCL && p.cluster_stats;
  uint8_t* a_ring = smem;
  uint8_t* b_ring = smem + p.SA * kAStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_ring + p.SB * p.b_stage_bytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kSA;
  uint64_t* b_full = a_empty + kSA;
  uint64_t* b_empty = b_full + kMaxSB;
  uint64_t* x_full = b_empty + kMaxSB;                                // [2] cluster statistics barriers
  float* ssq = reinterpret_cast<float*>(bars) + 256;                  // [4 epilogue warps of a pixel][128 pixels]
  float* rss = ssq + 512;                                             // same, for the residual's pixel-norm
  float* stot = rss + 512;                                            // [128] per-pixel totals over the cluster
  float* xstat = stot + 128;                                          // [2 parity][kMaxSplit][128] from peer CTAs
  float* stg = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + kSmemMisc);   // [kN][kStgLd] accumulator

  // The role id goes through a shuffle so that ptxas KNOWS it is warp-uniform: with a plain threadIdx.x >> 5 the role
  // branches count as divergent regions, and inside a divergent region nothing is kept in uniform registers.
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
#if TDX_DEBUG_HOOKS
  if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) p.trace[126] = clock64();
  if (p.timeline && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    atomicMin(p.timeline, t);
  }
#endif

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tm0);
    if (p.nseg > 1) tma_prefetch_desc(&tm1);
    if (p.nseg > 2) tma_prefetch_desc(&tm2);
  }
  if (warp == 2) {
    // all 44 barriers at once, two per lane (one thread initialising them in turn costs ~800 cycles of every launch):
    // [a_full 3][a_empty 3][b_full 18][b_empty 18][x_full 2], contiguous from `bars`.  Every consumer warp frees a slot.
    constexpr int kBars = 2 * kSA + 2 * kMaxSB + 2;
    static_assert(kBars <= 64, "two barriers per lane");
    const int x_full0 = 2 * kSA + 2 * kMaxSB;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int i = lane + 32 * k;
      if (i < kBars) {
        uint32_t count = 1;
        if ((i >= kSA && i < 2 * kSA) || (i >= 2 * kSA + kMaxSB && i < x_full0)) count = kEpiWarps;
        if (i >= x_full0) count = p.xsplit > 1 ? (uint32_t)(p.xsplit - 1) * 128u : 1u;
        mbar_init(&bars[i], count);
      }
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (cstats_) cluster_sync_all();   // peers' barriers are initialised before anyone arrives on them
#if TDX_DEBUG_HOOKS
  if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) p.trace[127] = clock64();
#endif
  // Let the next kernel in the stream start its own prologue as soon as SMs free up (it still waits for our memory).
  pdl_launch_dependents();

  if (warp == 0) {
    // ------------------------------------------------------------------ A producer (halo patches via tiled TMA)
    pdl_wait();  // activations are produced by the previous kernel
    int sa = 0;
    uint32_t ph = 0;
    int it = 0;
    TileWalk tw;
    tw.init(p);
    int s0, s1;
    stage_range(p, tw.kpart, s0, s1);
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x, ++it, tw.next(p)) {
      const int img = tw.img, Y0 = tw.ty * kTileH, X0 = tw.tx * kTileW;
      if (lane == 0) TDX_TRACE(0, it);
      for (int s = s0; s < s1;) {
        int seg, ch, tap, taps;
        stage_locate(p, s, seg, ch, tap, taps);
        const CUtensorMap* tm = seg == 0 ? &tm0 : (seg == 1 ? &tm1 : &tm2);
        mbar_wait(&a_empty[sa], ph ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&a_full[sa], kAStageBytes);
          tma_load_4d(tm, &a_full[sa], a_ring + sa * kAStageBytes, (X0 - 1) * 8, Y0 - 1, ch * 8, img);
        }
        __syncwarp();
        if (++sa == p.SA) { sa = 0; ph ^= 1; }
        s += taps - tap;   // the rest of this chunk's taps use the same patch
      }
    }
    if (ksplit_ > 1) cluster_sync_all();   // split-K hand-over barrier (see the epilogue)
  } else if (warp == 1) {
    // ------------------------------------------------------------------ B producer (pre-packed weight stages)
    // Weights are constants: no dependency on the previous kernel, so this starts streaming during its tail.
    int sb = 0;
    uint32_t ph = 0;
    TileWalk tw;
    tw.init(p);
    const int split = tw.split;
    int st0, st1;
    stage_range(p, tw.kpart, st0, st1);
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
      const uint8_t* bsrc = reinterpret_cast<const uint8_t*>(p.B) +
                            ((size_t)split * p.stages_per_item + st0) * p.b_stage_bytes;
      // The stages are handed over in GROUPS of up to `bgroup` consecutive taps of one 64-channel chunk: a group
      // completes ONE barrier, the one of its first slot, so the issuer waits once per group instead of once per 4
      // MMAs (an mbarrier try_wait costs ~90 cycles even when the phase is already complete).  bgroup = 9 when the
      // ring holds two chunks or the whole weight slice, 1 (stage by stage) for shorter, streaming rings.
      if (p.bgroup == 1) {
        // stage-by-stage hand-over (streaming rings): the tightest loop possible -- at N >= 128 this warp has to issue a
        // stage every ~256 cycles, and an mbarrier try_wait alone costs ~90
        for (int ks = 0; ks < st1 - st0; ++ks) {
          mbar_wait(&b_empty[sb], ph ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&b_full[sb], p.b_stage_bytes);
            bulk_load_1d(bsrc + (size_t)ks * p.b_stage_bytes, &b_full[sb], b_ring + sb * p.b_stage_bytes,
                         p.b_stage_bytes);
          }
          __syncwarp();
          if (++sb == p.SB) { sb = 0; ph ^= 1; }
        }
        continue;
      }
      int ks = 0;
      for (int s = st0; s < st1;) {
        int seg, ch, tap0, taps;
        stage_locate(p, s, seg, ch, tap0, taps);
        const int nt = (taps - tap0 < st1 - s) ? taps - tap0 : st1 - s;
        int head = sb, gi = 0;
        for (int t = 0; t < nt; ++t) {
          if (!p.resident) mbar_wait(&b_empty[sb], ph ^ 1);
          const bool first = gi == 0;                        // first stage of a hand-over group: its barrier carries the group
          if (++gi == p.bgroup) gi = 0;                      // (no integer division in this loop: ~150 cycles each)
          if (first) head = sb;
          if (elect_one()) {
            uint64_t* full = &b_full[head];
            if (first) mbar_expect_tx(full, (uint32_t)(nt - t < p.bgroup ? nt - t : p.bgroup) * p.b_stage_bytes);
            bulk_load_1d(bsrc + (size_t)(ks + t) * p.b_stage_bytes, full, b_ring + sb * p.b_stage_bytes,
                         p.b_stage_bytes);
          }
          __syncwarp();
          if (++sb == p.SB) { sb = 0; ph ^= 1; }
        }
        ks += nt;
        s += nt;
      }
      if (p.resident) break;   // the ring now holds this CTA's whole weight slice for every later item
    }
    if (ksplit_ > 1) cluster_sync_all();
  } else if (warp < 4) {
    if (ksplit_ > 1) cluster_sync_all();
  } else {
    // ------------------------------------------------------------------ consumers: MMA, then the epilogue
    // In the epilogue warp w handles quadrant q = w & 3 of the staging tile (pixels q*32 .. q*32+31, one per lane); the
    // kWQ warps of a quadrant (wq = 0 .. kWQ-1) take the item's kChunk-column chunks round-robin.
    pdl_wait();  // residual / cvec come from earlier kernels; our stores must not race their readers
    const int q = warp & 3;
    const int wq = (warp - 4) >> 2;
    const int m = q * 32 + lane;
    const int y = m >> 3, x = m & 7;
    const int C8 = p.cout >> 3;
    const bool need_norm = (p.epi & TDX_EPI_PNORM) || p.out[0].kind == TDX_OUT_PNORM_SILU ||
                           p.out[1].kind == TDX_OUT_PNORM_SILU || p.out[2].kind == TDX_OUT_PNORM_SILU ||
                           p.rms_out != nullptr;
    const uint32_t my_rank = cstats_ ? cluster_ctarank() : 0;
    TileWalk tw;
    tw.init(p);
    ConsumerRing ring = {0, 0, 0u, 0u};
    int s0, s1;
    stage_range(p, tw.kpart, s0, s1);
    // Per-CTA constants: with split-K (one item per CTA) this part finalises `slice` of the item's columns.
    const int ks = ksplit_, kpart = tw.kpart;
    const int slice = p.ncta / ks, sch = slice / kChunk;
    const int nchunks_all = p.ncta / kChunk;              // chunks of the whole accumulator tile
    const int nchunks = sch;                              // chunks this CTA finalises
    const int col0 = kpart * slice;                       // first accumulator column this CTA finalises
    const int chbase = tw.split * p.ncta + col0;          // first output channel this CTA writes
    const uint32_t plane = (uint32_t)(p.H * p.W);         // (all tensor offsets fit 32 bits: igemm_validate)
    // Element offset of this thread's pixel in a tensor of this launch's (scaled) geometry.  A tile origin (16 ty, 8 tx) is
    // even, so the offset is SEPARABLE: off = [img * istride + ty * rowstep + tx * colstep] + tpart, where the bracket
    // is warp-uniform and per item (three multiply-adds from launch constants) and `tpart` is a per-thread constant.
    // (The former per-item evaluation of (Y >> 1) * (W >> 1) + ..., with its branches on the spatial mode, was most of
    // the ~500 non-arithmetic instructions an epilogue warp spent per item.)
    struct OffSpec {
      uint32_t istride, rowstep, colstep, tpart;
    };
    auto make_spec = [&](int spatial, uint32_t planes_per_img) -> OffSpec {
      OffSpec o;
      if (spatial == TDX_SP_DOWN2) {
        o.istride = planes_per_img * (plane >> 2);
        o.rowstep = (uint32_t)(kTileH / 2) * (uint32_t)(p.W >> 1);
        o.colstep = kTileW / 2;
        o.tpart = (uint32_t)((y >> 1) * (p.W >> 1) + (x >> 1));
      } else if (spatial == TDX_SP_UP2) {
        o.istride = planes_per_img * (plane << 2);
        o.rowstep = (uint32_t)(kTileH * 2) * (uint32_t)(p.W << 1);
        o.colstep = kTileW * 2;
        o.tpart = (uint32_t)((y << 1) * (p.W << 1) + (x << 1));
      } else {
        o.istride = planes_per_img * plane;
        o.rowstep = (uint32_t)kTileH * (uint32_t)p.W;
        o.colstep = kTileW;
        o.tpart = (uint32_t)(y * p.W + x);
      }
      return o;
    };
    auto item_off = [&](const OffSpec& o, const TileWalk& t) -> uint32_t {
      return (uint32_t)t.img * o.istride + (uint32_t)t.ty * o.rowstep + (uint32_t)t.tx * o.colstep + o.tpart;
    };
    // Residual reads.  "UP2" = the residual is at half resolution, "DOWN2" = at double resolution (the inverse of an
    // output's meaning).
    const bool has_resid = (p.epi & TDX_EPI_RESID) != 0;
    const uint32_t rplane = p.resid_spatial == TDX_SP_UP2 ? (plane >> 2) : (p.resid_spatial == TDX_SP_DOWN2 ? (plane << 2) : plane);
    const int rsp = p.resid_spatial == TDX_SP_UP2 ? TDX_SP_DOWN2 : (p.resid_spatial == TDX_SP_DOWN2 ? TDX_SP_UP2 : TDX_SP_SAME);
    const OffSpec rspec = make_spec(rsp, (uint32_t)C8), rinv_spec = make_spec(rsp, 1u);
    // outputs: the channel-slice offset of this CTA is folded into the thread part; bit o of `omask` = output o exists
    // and this thread's pixel is stored (an odd pixel of a 2x-downsampled output is not: (Y | X) & 1 == (y | x) & 1)
    OffSpec ospec[3];
    uint32_t omask = 0;
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const int sp = p.out[o].spatial;
      ospec[o] = make_spec(sp, (uint32_t)C8);
      const uint32_t oplane = sp == TDX_SP_DOWN2 ? (plane >> 2) : (sp == TDX_SP_UP2 ? (plane << 2) : plane);
      ospec[o].tpart += (uint32_t)(chbase >> 3) * oplane;
      omask |= (uint32_t)(p.out[o].kind != TDX_OUT_NONE && !(sp == TDX_SP_DOWN2 && ((y | x) & 1))) << o;
    }
    // The values an item needs from global memory before it can touch its accumulator are requested ONE ITEM AHEAD
    // (`fetch_ahead`, called where the current item has consumed them): the residual's first-chunk channels or the
    // modulation vector's first chunk (`pre`) and the residual's pixel-norm factor (`rinv_pre`), so that their first use
    // does not wait on a global load.
    constexpr int kPreN = (kChunk / 4 > kGroups) ? kChunk / 4 : kGroups;
    uint4 pre[kPreN];
    const uint4* rbase_pre = nullptr;
    float rinv_pre = 1.f;
    const bool cv_ahead = (p.epi & TDX_EPI_EMB_SILU) && !has_resid;   // `pre` holds cvec (else: the residual)
    const bool ahead = has_resid || cv_ahead;
    const bool own_rnorm = has_resid && p.resid_pnorm && !p.resid_inv;
    auto fetch_ahead = [&](const TileWalk& t) {
      if (cv_ahead) {
        const uint4* cp = reinterpret_cast<const uint4*>(p.cvec + (size_t)t.img * p.cout + chbase + wq * kChunk);
#pragma unroll
        for (int j = 0; j < kChunk / 4; ++j) pre[j] = (wq < nchunks) ? __ldg(cp + j) : make_uint4(0, 0, 0, 0);
        return;
      }
      if (!has_resid) return;
      const int Y_ = t.ty * kTileH + y, X_ = t.tx * kTileW + x;
      const bool vld = (Y_ < p.H) && (X_ < p.W);
      rbase_pre = p.resid + item_off(rspec, t);
      // the producer of the residual left 1 / (eps + rms) per pixel: one float instead of all Cout channels
      if (p.resid_inv) rinv_pre = vld ? __ldg(p.resid_inv + item_off(rinv_spec, t)) : 0.f;
      const uint4* rptr = rbase_pre + (size_t)((chbase >> 3) + wq * kGroups) * rplane;
#pragma unroll
      for (int g = 0; g < kGroups; ++g)
        pre[g] = (vld && wq < nchunks) ? __ldg(rptr + (size_t)g * rplane) : make_uint4(0, 0, 0, 0);
    };
    if (ahead) fetch_ahead(tw);
    int it = 0;
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x, ++it, tw.next(p)) {
      const int img = tw.img;
      const int Y = tw.ty * kTileH + y, X = tw.tx * kTileW + x;
      const bool valid = (Y < p.H) && (X < p.W);
      if (warp == 4 && lane == 0) TDX_TRACE(1, it);
      mma_item<kN>(p, a_ring, b_ring, a_full, a_empty, b_full, b_empty, ring, s0, s1, p.resident && it > 0, stg);
      if (warp == 4 && lane == 0) TDX_TRACE(2, it);

      // ---------------- split-K: the ksplit CTAs of a cluster each hold a partial sum of the same 128 x ncta tile.
      // Reduce-scatter through an L2-resident fp32 workspace: every part publishes the column slices the other parts
      // own, the cluster barrier (release/acquire, all warps of all parts take it once) hands them over, and each part
      // finishes the epilogue of its own ncta/ksplit columns.  (Launches with ksplit > 1 have one item per CTA.)
      const float* red_src = nullptr;
      if (ks > 1) {
        float* wsg = p.ws + (size_t)fdiv((uint32_t)item, p.fd_ks) * (ks - 1) * p.ncta * 128;   // [dst part][source slot][slice cols][128]
        if (warp == 4 && lane == 0) TDX_TRACE(3, it);
        for (int ck = wq; ck < nchunks_all; ck += kWQ) {
          const int dst = ck / sch;
          if (dst == kpart) continue;
          const int slot = kpart - (kpart > dst ? 1 : 0);
          float* d = wsg + ((size_t)(dst * (ks - 1) + slot) * slice + (size_t)(ck - dst * sch) * kChunk) * 128 + m;
          float v[kChunk];
          __syncwarp();
          load_acc(stg, m, ck * kChunk, v);
#pragma unroll
          for (int j = 0; j < kChunk; ++j) __stcg(d + (size_t)j * 128, v[j]);
        }
        cluster_sync_all();
        red_src = wsg + (size_t)kpart * (ks - 1) * slice * 128 + m;
      }
      const float* cvb = p.cvec ? p.cvec + (size_t)img * p.cout + chbase : nullptr;
      // adds the other parts' partial sums to this CTA's chunk ck (no-op without split-K)
      auto add_partials = [&](int ck, float (&v)[kChunk]) {
        for (int kp = 0; kp < ks - 1; ++kp) {
          const float* src = red_src + ((size_t)kp * slice + (size_t)(ck * kChunk)) * 128;
#pragma unroll
          for (int j = 0; j < kChunk; ++j) v[j] += __ldcg(src + (size_t)j * 128);
        }
      };

      {
        // ---------------- general: residual mp_sum (+pixel-norm of the residual), clip, pixel-norm, up to 3 outputs
        float rscale = p.resid_scale;
        const uint4* rbase = rbase_pre;
        const bool more = ahead && item + (int)gridDim.x < p.num_items;
        TileWalk tn = tw;
        tn.next(p);
        if (has_resid && p.resid_inv) {
          rscale = p.resid_scale * rinv_pre;
        } else if (own_rnorm) {
          // the residual's pixel-norm runs over ALL Cout channels: the kWQ warps of a pixel quadrant each read their
          // share of the 8-channel planes (C8 is a multiple of 8) and combine through shared memory
          float ss = 0.f;
          auto sq8 = [&](const uint4& u) {
            float a, b;
            unpack_bf16x2(u.x, a, b); ss = fmaf(a, a, fmaf(b, b, ss));
            unpack_bf16x2(u.y, a, b); ss = fmaf(a, a, fmaf(b, b, ss));
            unpack_bf16x2(u.z, a, b); ss = fmaf(a, a, fmaf(b, b, ss));
            unpack_bf16x2(u.w, a, b); ss = fmaf(a, a, fmaf(b, b, ss));
          };
          if (valid) {
            for (int g0 = wq * 2; g0 < C8; g0 += 2 * kWQ) {
              const uint4 u0 = __ldg(rbase + (size_t)g0 * rplane), u1 = __ldg(rbase + (size_t)(g0 + 1) * rplane);
              sq8(u0);
              sq8(u1);
            }
          }
          rss[wq * 128 + m] = ss;
          named_bar_sync(9 + q, 32 * kWQ);
          ss = 0.f;
#pragma unroll
          for (int w = 0; w < kWQ; ++w) ss += rss[w * 128 + m];
          rscale = p.resid_scale * inv_rms(ss, p.inv_cout);
        }
        // this thread's pixel in each output (inactive: out of the image, or an odd pixel of a 2x-downsampled output)
        uint4* optr[3];
        bool oact[3];
#pragma unroll
        for (int o = 0; o < 3; ++o) {
          oact[o] = valid && ((omask >> o) & 1u);
          optr[o] = reinterpret_cast<uint4*>(p.out[o].ptr) + item_off(ospec[o], tw);
        }


        // v = accumulator chunk `ck` after emb-silu / residual / clip (everything that precedes the pixel-norm)
        auto compute_v = [&](int ck, float (&v)[kChunk]) {
          __syncwarp();
          load_acc(stg, m, col0 + ck * kChunk, v);
          add_partials(ck, v);
          if (p.epi & TDX_EPI_EMB_SILU) {
#pragma unroll
            for (int i = 0; i < kChunk; i += 4) {
              const uint4 cu = (cv_ahead && ck == wq) ? pre[i >> 2] : __ldg(reinterpret_cast<const uint4*>(cvb + ck * kChunk + i));
              const float4 c4 = make_float4(__uint_as_float(cu.x), __uint_as_float(cu.y), __uint_as_float(cu.z), __uint_as_float(cu.w));
              v[i + 0] = mp_silu_f(v[i + 0] * c4.x);
              v[i + 1] = mp_silu_f(v[i + 1] * c4.y);
              v[i + 2] = mp_silu_f(v[i + 2] * c4.z);
              v[i + 3] = mp_silu_f(v[i + 3] * c4.w);
            }
          }
          if (p.epi & TDX_EPI_RESID) {
            const uint4* rptr = rbase + (size_t)((chbase >> 3) + ck * kGroups) * rplane;
#pragma unroll
            for (int g = 0; g < kGroups; ++g) {
              uint4 u = (ck == wq) ? pre[g] : (valid ? __ldg(rptr + (size_t)g * rplane) : make_uint4(0, 0, 0, 0));
              float rr[8];
              unpack_bf16x2(u.x, rr[0], rr[1]);
              unpack_bf16x2(u.y, rr[2], rr[3]);
              unpack_bf16x2(u.z, rr[4], rr[5]);
              unpack_bf16x2(u.w, rr[6], rr[7]);
#pragma unroll
              for (int i = 0; i < 8; ++i) v[g * 8 + i] = fmaf(rscale, rr[i], v[g * 8 + i]);
            }
          }
          if (p.clip > 0.f) {
#pragma unroll
            for (int i = 0; i < kChunk; ++i) v[i] = fminf(fmaxf(v[i], -p.clip), p.clip);
          }
        };
        auto emit_v = [&](int ck, float (&v)[kChunk], float inv) {
          if (p.epi & TDX_EPI_PNORM) {
#pragma unroll
            for (int i = 0; i < kChunk; ++i) v[i] *= inv;
          }
#pragma unroll
          for (int o = 0; o < 3; ++o) {
            const int kind = p.out[o].kind, sp = p.out[o].spatial;
            if (kind == TDX_OUT_NONE) continue;
            float hs = 0.5f * p.out[o].scale;
            if (kind == TDX_OUT_PNORM_SILU) hs = (p.epi & TDX_EPI_PNORM) ? 0.5f : 0.5f * inv;
            const uint32_t oplane = sp == TDX_SP_DOWN2 ? (plane >> 2) : (sp == TDX_SP_UP2 ? (plane << 2) : plane);
            const int Wo = sp == TDX_SP_DOWN2 ? (p.W >> 1) : (sp == TDX_SP_UP2 ? (p.W << 1) : p.W);
            store_chunk(optr[o] + (size_t)(ck * kGroups) * oplane, oplane, Wo, kind, sp, oact[o], v, hs,
                        hs * (1.0f / 0.596f));
          }
        };
        // per-pixel sum of squares over ALL Cout channels -> 1 / (eps + rms)
        auto finish_norm = [&](float sumsq) -> float {
          // (1) combine the warps that own the same pixels (named barrier per lane quadrant)
          ssq[wq * 128 + m] = sumsq;
          named_bar_sync(1 + q, 32 * kWQ);
          float tot = 0.f;
#pragma unroll
          for (int w = 0; w < kWQ; ++w) tot += ssq[w * 128 + m];
          if (cstats_) {
            // (2) combine the CTAs that hold the other channels of this M tile through distributed shared memory
            const int par = it & 1;
            if (wq == 0) {
              for (uint32_t r = 0; r < (uint32_t)p.xsplit; ++r) {
                if (r == my_rank) continue;
                st_cluster_f32(map_to_cta(smem_u32(&xstat[(par * kMaxSplit + my_rank) * 128 + m]), r), tot);
                mbar_arrive_cluster(map_to_cta(smem_u32(&x_full[par]), r));
              }
              const uint32_t xph = (it >> 1) & 1;
              if (!mbar_try_wait_cluster(&x_full[par], xph)) {
                const long long t0 = clock64();
                while (!mbar_try_wait_cluster(&x_full[par], xph)) {
                  if (clock64() - t0 > TDX_WAIT_LIMIT) asm volatile("trap;");
                }
              }
              for (uint32_t r = 0; r < (uint32_t)p.xsplit; ++r)
                if (r != my_rank) tot += xstat[(par * kMaxSplit + r) * 128 + m];
              stot[m] = tot;
            }
            named_bar_sync(5 + q, 32 * kWQ);
            tot = stot[m];
          }
          return inv_rms(tot, p.inv_cout);
        };

        // One code path for all cases (keeps the kernel small enough for the instruction cache): an optional
        // statistics pass, then the emitting pass.  When every warp has at most one chunk, it stays in registers
        // across the statistics exchange instead of being recomputed.
        float v[kChunk];
        float sumsq = 0.f, inv = 1.f;
        const bool reuse = need_norm && nchunks <= kWQ;
#pragma unroll 1
        for (int pass = need_norm ? 0 : 1; pass < 2; ++pass) {
#pragma unroll 1
          for (int ck = wq; ck < nchunks; ck += kWQ) {
            if (pass == 0 || !reuse) {
              compute_v(ck, v);
              // `pre` (chunk wq of this item) has just been used for the last time: request the next item's
              if (ck == wq && (reuse || pass == 1) && more) fetch_ahead(tn);
            }
            if (pass == 0) {
#pragma unroll
              for (int i = 0; i < kChunk; ++i) sumsq = fmaf(v[i], v[i], sumsq);
            } else {
              emit_v(ck, v, inv);
            }
          }
          if (pass == 0) {
            inv = finish_norm(sumsq);
            if (p.rms_out && wq == 0 && kpart == 0 && tw.split == 0 && valid)
              p.rms_out[(uint32_t)img * plane + (uint32_t)(Y * p.W + X)] = inv;
          }
        }
      }
      if (warp == 4 && lane == 0) TDX_TRACE(4, it);
    }
  }

  __syncthreads();
  if (cstats_) cluster_sync_all();   // nobody leaves while a peer may still write into its shared memory
#if TDX_DEBUG_HOOKS
  if (p.trace && blockIdx.x == 0 && threadIdx.x == 96) p.trace[125] = clock64();
  if (p.timeline && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    atomicMax(p.timeline + 1, t);
  }
#endif
}

// ---------------------------------------------------------------------------------------------------- host side
static unsigned long long* g_trace_ptr = nullptr;
static unsigned long long* g_timeline_ptr = nullptr;   // debug: consecutive launches fill consecutive [start,end] pairs
static int g_timeline_idx = 0, g_timeline_cap = 0;

static int ensure_scratch(float** ws);

typedef decltype(&igemm_kernel<false, 64>) IgemmKernel;

static IgemmKernel igemm_kernel_for(bool cluster, int n) {
  switch (n) {
    case 64: return cluster ? igemm_kernel<true, 64> : igemm_kernel<false, 64>;
    case 128: return cluster ? igemm_kernel<true, 128> : igemm_kernel<false, 128>;
    case 192: return cluster ? igemm_kernel<true, 192> : igemm_kernel<false, 192>;
    default: return cluster ? igemm_kernel<true, 256> : igemm_kernel<false, 256>;
  }
}

int igemm_prepare() {
  static bool seen[16] = {false};
  if (first_use_on_device(seen)) {
    for (int n = 64; n <= 256; n += 64)
      for (int cl = 0; cl < 2; ++cl)
        TDX_CHECK_CUDA(
            cudaFuncSetAttribute(igemm_kernel_for(cl, n), cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget));
  }
  float* ws;
  return ensure_scratch(&ws);
}

static bool needs_norm(const TdxIgemmDesc& d) {
  if (d.epi_flags & TDX_EPI_PNORM) return true;
  if (d.rms_out) return true;
  for (int o = 0; o < 3; ++o)
    if (d.out[o].kind == TDX_OUT_PNORM_SILU) return true;
  return false;
}

// Split-K scratch (fp32 partial accumulators), one per device, allocated outside stream capture.
constexpr size_t kWsBytes = 24u << 20;
static float* g_ws[16] = {nullptr};

static int ensure_scratch(float** ws) {
  int dev = 0;
  TDX_CHECK_CUDA(cudaGetDevice(&dev));
  TDX_REQUIRE(dev >= 0 && dev < 16, "igemm: device index %d out of range", dev);
  if (!g_ws[dev]) TDX_CHECK_CUDA(cudaMalloc(&g_ws[dev], kWsBytes));
  *ws = g_ws[dev];
  return TDX_OK;
}

// How many clusters of `csize` one-CTA-per-SM igemm CTAs the device can hold at once (cached per size).
static int max_active_clusters(int csize) {
  static int cache[9] = {0};
  if (csize <= 1) return sm_count();
  if (csize > 8) return 0;
  if (cache[csize]) return cache[csize];
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cudaLaunchAttribute attr[1];
  cfg.gridDim = dim3((sm_count() / csize) * csize);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kSmemBudget;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = csize;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  cudaFuncSetAttribute(igemm_kernel<true, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget);
  if (cudaOccupancyMaxActiveClusters(&n, igemm_kernel<true, 64>, &cfg) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    n = (sm_count() * 3 / 4) / csize;   // no GPU to ask (or the query failed): assume some GPCs cannot be filled
  }
  cache[csize] = n;
  return n;
}

// Choose the output-channel width of a work item (MMA N) and the split-K factor.  A rough cost model (cycles):
//   * the 128 x N x 16 product of one K step takes N cycles of the SM's tensor cores (dense bf16 peak of the H100
//     data sheet: ~2048 multiply-adds per SM per cycle);
//   * L2 -> SM delivers ~5 KB/clk chip-wide and ~56 B/clk into one SM; per item the A patches (23 KB per 64 input
//     channels) and, unless the item's whole weight slice fits the B ring ("resident": loaded once per CTA), the
//     weights (N*128 B per stage);
//   * the fp32 staging tile (N * kStgLd * 4 B) shares shared memory with the rings: wide items get shallower rings,
//     and a one-slot weight ring cannot overlap weight loads with the MMAs;
//   * layers with fewer work items than SMs are a serial MMA chain per CTA: split their (chunk, tap) stages over the
//     `ks` CTAs of a cluster, which reduce-scatter fp32 partial sums through L2 (each part then finalises N/ks columns,
//     so N/ks must be a multiple of the epilogue's 32-column chunk);
//   * pixel-norm layers exchange statistics inside a cluster, so all nsplit*ks CTAs of an M tile share one (<= 8).
struct ItemShape { int ncta, resident, sa, sb, ksplit; };

static ItemShape choose_item_shape(int cout, int tiles, int stages, int chunks, int forced_n, bool norm) {
  if (forced_n && (forced_n > cout || cout % forced_n)) forced_n = 0;
  double best = 1e30;
  ItemShape bs = {64, 0, kSA, 2, 1};
  for (int n = 64; n <= 256 && n <= cout; n += 64) {
    if (cout % n) continue;
    if (forced_n && n != forced_n) continue;
    const int nsplit = cout / n;
    if (norm && nsplit > kMaxSplit) continue;   // pixel-norm statistics travel inside one cluster
    const int stage_bytes = n * 128;
    const int free_bytes = kSmemBudget - kSmemMisc - n * kStgLd * 4;
    const int sa = free_bytes - kSA * kAStageBytes >= 2 * stage_bytes ? kSA : 2;
    const int ring_budget = free_bytes - sa * kAStageBytes;
    const long items = (long)tiles * nsplit;
    for (int ks = 1; ks <= 8; ++ks) {
      const int csize = ks * ((norm && nsplit > 1) ? nsplit : 1);
      if (ks > 1) {
        if (n % (kChunk * ks) || ks > stages || csize > kMaxSplit) continue;
        if (items * ks > (long)max_active_clusters(csize) * csize) continue;   // one item per CTA, all resident
        if ((size_t)items * (ks - 1) * n * 512 > kWsBytes) continue;
      }
      const int my_stages = (stages + ks - 1) / ks;
      const int my_chunks = (chunks + ks - 1) / ks + (ks > 1 ? 1 : 0);
      const int resident = (ks == 1 && stages * stage_bytes <= ring_budget && stages <= kMaxSB) ? 1 : 0;
      int sb = resident ? stages : ring_budget / stage_bytes;
      if (sb > kMaxSB) sb = kMaxSB;
      if (sb < 1) continue;
      int grid = items * ks < sm_count() ? (int)(items * ks) : sm_count();
      grid -= grid % (nsplit * ks);
      if (grid <= 0) continue;
      const double rounds = (double)((items * ks + grid - 1) / grid);
      const double mma = rounds * my_stages * 4.0 * n * (sb < 2 && !resident ? 2.0 : 1.0) + 800.0;
      const double a_bytes = (double)items * ks * my_chunks * kAStageBytes;
      const double b_bytes = resident ? (double)grid * stages * stage_bytes : (double)items * stages * stage_bytes;
      const double red_bytes = ks > 1 ? (double)(ks - 1) / ks * n * 512.0 : 0.0;   // written and read per CTA
      const double l2 = (a_bytes + b_bytes + 2.0 * red_bytes * items * ks) / 5000.0;
      const double per_sm = (double)(my_chunks * kAStageBytes + my_stages * stage_bytes) / 56.0;  // one SM's L2 port
      const int epi_chunks = ((n / ks) / kChunk + 3) / 4;
      const double epi = rounds * epi_chunks * 100.0;
      const double red = ks > 1 ? 2.0 * red_bytes / 56.0 + 2000.0 : 0.0;
      double t = mma;
      if (l2 > t) t = l2;
      if (per_sm > t) t = per_sm;
      t += epi + red;
      if (t < best) { best = t; bs = {n, resident, sa, sb, ks}; }
    }
  }
  return bs;
}

int igemm_launch(const TdxIgemmDesc& d, const CUtensorMap* tms, cudaStream_t stream) {
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.nseg = d.n_seg;
  p.stages_per_item = 0;
  int chunks = 0;
  for (int s = 0; s < d.n_seg; ++s) {
    p.seg_chunks[s] = d.a_channels[s] / 64;
    p.seg_taps[s] = d.a_taps[s];
    p.stages_per_item += p.seg_chunks[s] * p.seg_taps[s];
    chunks += p.seg_chunks[s];
  }
  p.B = reinterpret_cast<const __nv_bfloat16*>(d.b_packed);
  p.cout = d.c_out;
  p.inv_cout = 1.0f / (float)d.c_out;
  p.H = d.height;
  p.W = d.width;
  p.nimg = d.n_img;
  p.tiles_x = (d.width + kTileW - 1) / kTileW;
  p.tiles_y = (d.height + kTileH - 1) / kTileH;
  const int tiles = p.tiles_x * p.tiles_y * d.n_img;
  const bool norm = needs_norm(d);
  const ItemShape shp = choose_item_shape(d.c_out, tiles, p.stages_per_item, chunks, d.n_per_item, norm);
  p.ncta = shp.ncta;
  p.resident = shp.resident;
  p.SA = shp.sa;
  p.SB = shp.sb;
  // streaming rings stay stage by stage: a grouped hand-over makes the issuer wait for a group's LAST stage, which
  // costs latency slack exactly where the weight stream is L2-bound (measured: N=128 layers 5-25 % slower)
  p.bgroup = (shp.resident || shp.sb >= 18) ? 9 : 1;
  p.ksplit = shp.ksplit;
  p.nsplit = d.c_out / p.ncta;
  p.b_stage_bytes = p.ncta * 128;
  p.num_items = tiles * p.nsplit * p.ksplit;
  if (p.ksplit > 1) {
    int rc_ws = ensure_scratch(&p.ws);
    if (rc_ws != TDX_OK) return rc_ws;
  }
  p.epi = d.epi_flags;
  p.cluster_stats = (norm && p.nsplit * p.ksplit > 1) ? 1 : 0;
  p.xsplit = p.cluster_stats ? p.nsplit * p.ksplit : 1;
  const int cluster = p.cluster_stats ? p.xsplit : p.ksplit;
  p.cvec = d.cvec;
  p.resid = reinterpret_cast<const uint4*>(d.resid);
  p.resid_spatial = d.resid_spatial;
  p.resid_pnorm = d.resid_pnorm;
  p.resid_scale = d.resid_scale;
  p.clip = d.clip;
  for (int o = 0; o < 3; ++o) p.out[o] = d.out[o];
  p.rms_out = d.rms_out;
  p.resid_inv = d.resid_inv;
  p.trace = g_trace_ptr;
  p.timeline = (g_timeline_ptr && g_timeline_idx < g_timeline_cap) ? g_timeline_ptr + 2 * (g_timeline_idx++) : nullptr;

  int rc_prep = igemm_prepare();
  if (rc_prep != TDX_OK) return rc_prep;
  // grid: one CTA per SM at most, a multiple of nsplit so the slices of an M tile always run side by side
  int grid = p.num_items < sm_count() ? p.num_items : sm_count();
  grid -= grid % (p.nsplit * p.ksplit);
  {
    const int per = p.nsplit * p.ksplit;
    p.fd_ks = make_fastdiv(p.ksplit);
    p.fd_nsplit = make_fastdiv(p.nsplit);
    p.fd_per = make_fastdiv(per);
    p.fd_tx = make_fastdiv(p.tiles_x);
    p.fd_ty = make_fastdiv(p.tiles_y);
    int dstep = grid / per;
    p.dtx = dstep % p.tiles_x;
    dstep /= p.tiles_x;
    p.dty = dstep % p.tiles_y;
    p.dimg = dstep / p.tiles_y;
  }
  const int smem = p.SA * kAStageBytes + p.SB * p.b_stage_bytes + kSmemMisc + p.ncta * kStgLd * 4;
  const CUtensorMap& t0 = tms[0];
  const CUtensorMap& t1 = tms[d.n_seg > 1 ? 1 : 0];
  const CUtensorMap& t2 = tms[d.n_seg > 2 ? 2 : 0];
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  fill_launch_config(&cfg, attr, dim3(grid), dim3(kThreads), smem < 120 * 1024 ? 120 * 1024 : smem, stream);
  if (cluster > 1) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
    attr[cfg.numAttrs].val.clusterDim.x = cluster;
    attr[cfg.numAttrs].val.clusterDim.y = 1;
    attr[cfg.numAttrs].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs += 1;
  }
  TDX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, igemm_kernel_for(cluster > 1, p.ncta), t0, t1, t2, p));
  return TDX_OK;
}

int igemm_validate(const TdxIgemmDesc& d) {
  TDX_REQUIRE(d.n_seg >= 1 && d.n_seg <= 3, "igemm: n_seg=%d not in 1..3", d.n_seg);
  for (int s = 0; s < d.n_seg; ++s) {
    TDX_REQUIRE(d.a_ptr[s] != nullptr, "igemm: a_ptr[%d] is null", s);
    TDX_REQUIRE(d.a_channels[s] > 0 && d.a_channels[s] % 64 == 0, "igemm: a_channels[%d]=%d not a multiple of 64", s,
                d.a_channels[s]);
    TDX_REQUIRE(d.a_taps[s] == 9 || d.a_taps[s] == 1, "igemm: a_taps[%d]=%d not 9 or 1", s, d.a_taps[s]);
  }
  TDX_REQUIRE(d.b_packed != nullptr, "igemm: b_packed is null");
  TDX_REQUIRE(d.c_out >= 64 && d.c_out <= 2048 && d.c_out % 64 == 0, "igemm: c_out=%d must be a multiple of 64 <= 2048",
              d.c_out);
  if (needs_norm(d))
    TDX_REQUIRE(d.c_out / d.n_per_item <= kMaxSplit, "igemm: pixel-norm over %d channels needs n_per_item >= %d",
                d.c_out, d.c_out / kMaxSplit);
  TDX_REQUIRE(d.n_per_item >= 64 && d.n_per_item <= 256 && d.n_per_item % 64 == 0 && d.c_out % d.n_per_item == 0,
              "igemm: n_per_item=%d must be 64/128/192/256 and divide c_out=%d (use tdx_igemm_choose_n)", d.n_per_item,
              d.c_out);
  TDX_REQUIRE((unsigned long long)d.n_img * (d.c_out / 8) * d.height * d.width * 4ull < (1ull << 32),
              "igemm: tensor of %d x %d x %d x %d exceeds the 32-bit element offsets of the epilogue", d.n_img, d.c_out,
              d.height, d.width);
  TDX_REQUIRE(d.n_img >= 1 && d.height >= 8 && d.width >= 8 && d.height % 8 == 0 && d.width % 8 == 0,
              "igemm: bad shape n=%d h=%d w=%d (h, w multiples of 8)", d.n_img, d.height, d.width);
  if (d.epi_flags & TDX_EPI_EMB_SILU) TDX_REQUIRE(d.cvec != nullptr, "igemm: EMB_SILU needs cvec");
  if (d.resid_inv)
    TDX_REQUIRE((d.epi_flags & TDX_EPI_RESID) && !d.resid_pnorm,
                "igemm: resid_inv needs TDX_EPI_RESID and resid_pnorm == 0 (it replaces the recomputed pixel-norm)");
  if (d.epi_flags & TDX_EPI_RESID) {
    TDX_REQUIRE(d.resid != nullptr, "igemm: RESID needs resid");
    if (d.resid_spatial == TDX_SP_UP2)
      TDX_REQUIRE(d.height % 2 == 0 && d.width % 2 == 0, "igemm: UP2 residual needs even h, w");
  }
  for (int o = 0; o < 3; ++o) {
    if (d.out[o].kind == TDX_OUT_NONE) continue;
    TDX_REQUIRE(d.out[o].ptr != nullptr, "igemm: out[%d].ptr is null", o);
    TDX_REQUIRE(d.out[o].kind >= 1 && d.out[o].kind <= 3, "igemm: out[%d].kind=%d", o, d.out[o].kind);
    if (d.out[o].spatial == TDX_SP_DOWN2)
      TDX_REQUIRE(d.height % 2 == 0 && d.width % 2 == 0, "igemm: DOWN2 output needs even h, w");
  }
  return TDX_OK;
}

}  // namespace tdx

// Debug hooks (tools/trace_igemm.py): device buffer of 128 u64 that CTA 0 fills with per-item phase clocks.
extern "C" void tdx_debug_set_igemm_trace(void* device_u64x128) {
  tdx::g_trace_ptr = reinterpret_cast<unsigned long long*>(device_u64x128);
}
// Debug: every igemm launch recorded from now on writes {first CTA start, last CTA end} (globaltimer ns) into the next
// slot of `device_u64_pairs` (pre-filled with {~0, 0}); pass null to stop.
extern "C" void tdx_debug_set_igemm_timeline(void* device_u64_pairs, int capacity) {
  tdx::g_timeline_ptr = reinterpret_cast<unsigned long long*>(device_u64_pairs);
  tdx::g_timeline_idx = 0;
  tdx::g_timeline_cap = capacity;
}

extern "C" int tdx_igemm_choose_n(int32_t c_out, int32_t n_img, int32_t height, int32_t width,
                                  const int32_t* a_channels, const int32_t* a_taps, int32_t n_seg) {
  if (c_out < 64 || c_out % 64 || n_seg < 1 || n_seg > 3) return 64;
  int stages = 0, chunks = 0;
  for (int s = 0; s < n_seg; ++s) {
    stages += (a_channels[s] / 64) * a_taps[s];
    chunks += a_channels[s] / 64;
  }
  const int tiles = ((width + tdx::kTileW - 1) / tdx::kTileW) * ((height + tdx::kTileH - 1) / tdx::kTileH) * n_img;
  // conservative: assume the launch may need cluster-wide pixel-norm statistics (slices per tile <= cluster limit)
  return tdx::choose_item_shape(c_out, tiles, stages, chunks, 0, true).ncta;
}

// Debug: the (n_per_item, ksplit, resident, ring depth) the launch heuristics pick for a shape.
extern "C" void tdx_debug_igemm_plan(int32_t c_out, int32_t n_img, int32_t height, int32_t width,
                                     const int32_t* a_channels, const int32_t* a_taps, int32_t n_seg,
                                     int32_t n_per_item, int32_t needs_norm, int32_t* out4) {
  int stages = 0, chunks = 0;
  for (int s = 0; s < n_seg; ++s) {
    stages += (a_channels[s] / 64) * a_taps[s];
    chunks += a_channels[s] / 64;
  }
  const int tiles = ((width + tdx::kTileW - 1) / tdx::kTileW) * ((height + tdx::kTileH - 1) / tdx::kTileH) * n_img;
  tdx::ItemShape shp = tdx::choose_item_shape(c_out, tiles, stages, chunks, n_per_item, needs_norm != 0);
  out4[0] = shp.ncta; out4[1] = shp.ksplit; out4[2] = shp.resident; out4[3] = shp.sb;
}

extern "C" int64_t tdx_igemm_packed_weight_elems(const int32_t* a_channels, const int32_t* a_taps, int32_t n_seg,
                                                 int32_t c_out) {
  int64_t n = 0;
  for (int s = 0; s < n_seg; ++s) n += (int64_t)a_channels[s] * a_taps[s] * c_out;
  return n;
}

extern "C" int tdx_igemm_run(const TdxIgemmDesc* desc, void* stream) {
  if (!desc) {
    tdx::set_error("igemm: null descriptor");
    return TDX_E_INVALID;
  }
  int rc = tdx::igemm_validate(*desc);
  if (rc != TDX_OK) return rc;
  CUtensorMap tms[3];
  for (int s = 0; s < desc->n_seg; ++s) {
    rc = tdx::make_act_tensor_map(&tms[s], desc->a_ptr[s], desc->n_img, desc->a_channels[s], desc->height,
                                  desc->width);
    if (rc != TDX_OK) return rc;
  }
  return tdx::igemm_launch(*desc, tms, reinterpret_cast<cudaStream_t>(stream));
}
