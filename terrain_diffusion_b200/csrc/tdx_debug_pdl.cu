// Debug hook that tests the PDL ordering of every libtdx kernel (tests/test_pdl_order_gpu.py).  Compiled into every
// build; nothing on the sampling path calls it.
//
// tdx_debug_pdl_interpose enqueues one small kernel that, between its own griddepcontrol.wait and its exit, holds a set
// of device regions poisoned while the NEXT launch on the stream is allowed to start (it triggers the dependent launch
// right after poisoning, then spins for `delay_ns`).  A successor that waits (pdl_wait) before it touches a region sees
// the restored contents and computes what it computes without the hook; one that reads a region early reads the poison,
// and one that writes a region early shows up in the region's snapshot, taken at the end of the delay.
#include "tdx_common.h"
#include "tdx_ptx.cuh"

namespace tdx {

// One region, as the caller lays it out in DEVICE memory (six 64-bit words).  word: bytes of the poison word (1, 2, 4
// or 8), or 0 to leave the region as it is (only saved and snapshotted).  save: `bytes` of scratch that holds the
// contents while the region is poisoned; snapshot: `bytes` that receive the region at the end of the delay, or 0.
struct PdlRegion {
  unsigned long long ptr;
  long long bytes;
  unsigned long long poison;   // the word, little-endian in the low `word` bytes
  long long word;
  unsigned long long save;
  unsigned long long snapshot;
};

constexpr int kPdlThreads = 256;
constexpr int kPdlGrid = 8;                       // CTAs: most SMs stay free for the successor
constexpr long long kPdlMaxDelayNs = 100000000;   // 0.1 s: the spin is bounded whatever the caller passes

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ bool vec_ok(const PdlRegion& r) {
  return ((r.ptr | r.save | r.snapshot | (unsigned long long)r.bytes) & 15ull) == 0;
}

// The poison word repeated over 16 bytes (the region's start is 16-byte aligned on this path).
__device__ __forceinline__ uint4 poison16(const PdlRegion& r) {
  unsigned long long v = r.poison;
  if (r.word == 1) v = (v & 0xffull) * 0x0101010101010101ull;
  else if (r.word == 2) v = (v & 0xffffull) * 0x0001000100010001ull;
  else if (r.word == 4) v = (v & 0xffffffffull) * 0x0000000100000001ull;
  return make_uint4((unsigned)v, (unsigned)(v >> 32), (unsigned)v, (unsigned)(v >> 32));
}

template <typename T>
__device__ __forceinline__ void copy_units(unsigned long long dst, unsigned long long src, T poison, long long n) {
  const long long step = (long long)gridDim.x * kPdlThreads;
  for (long long i = (long long)blockIdx.x * kPdlThreads + threadIdx.x; i < n; i += step)
    reinterpret_cast<T*>(dst)[i] = src ? reinterpret_cast<const T*>(src)[i] : poison;
}

// dst = src (or the poison when src is 0) over this CTA's share of one region: in 16-byte units when every pointer and
// the size allow it, else in units of the poison word (bytes when the region is not poisoned).
__device__ void copy_share(const PdlRegion& r, unsigned long long dst, unsigned long long src) {
  if (vec_ok(r)) return copy_units(dst, src, poison16(r), r.bytes / 16);
  if (r.word == 8) return copy_units(dst, src, (unsigned long long)r.poison, r.bytes / 8);
  if (r.word == 4) return copy_units(dst, src, (unsigned)r.poison, r.bytes / 4);
  if (r.word == 2) return copy_units(dst, src, (unsigned short)r.poison, r.bytes / 2);
  copy_units(dst, src, (unsigned char)r.poison, r.bytes);
}

__global__ void __launch_bounds__(kPdlThreads) pdl_interpose_kernel(const PdlRegion* regions, int n, long long delay_ns) {
  pdl_wait();
  for (int k = 0; k < n; ++k) {
    const PdlRegion r = regions[k];
    copy_share(r, r.save, r.ptr);
    if (r.word) copy_share(r, r.ptr, 0);
  }
  __threadfence();
  __syncthreads();
  pdl_launch_dependents();
  const unsigned long long t0 = global_ns();
  while (global_ns() - t0 < (unsigned long long)delay_ns) {
  }
  __threadfence();
  for (int k = 0; k < n; ++k) {
    const PdlRegion r = regions[k];
    if (r.snapshot) copy_share(r, r.snapshot, r.ptr);
    if (r.word) copy_share(r, r.ptr, r.save);
  }
}

}  // namespace tdx

using namespace tdx;

// regions: DEVICE array of n_regions PdlRegion records (above); regions must not overlap.
extern "C" int tdx_debug_pdl_interpose(const void* regions, int32_t n_regions, int64_t delay_ns, void* stream) {
  TDX_REQUIRE(n_regions >= 0 && (regions || n_regions == 0), "pdl_interpose: bad region list");
  TDX_REQUIRE(delay_ns >= 0 && delay_ns <= kPdlMaxDelayNs, "pdl_interpose: delay %lld ns outside 0..%lld",
              (long long)delay_ns, kPdlMaxDelayNs);
  TDX_CHECK_CUDA(launch(pdl_interpose_kernel, kPdlGrid, kPdlThreads, 0, stream,
                        reinterpret_cast<const PdlRegion*>(regions), (int)n_regions, (long long)delay_ns));
  return TDX_OK;
}
