// Internal helpers shared by the libtdx translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <utility>

#include "../../include/tdx.h"

namespace tdx {

void set_error(const char* fmt, ...);
int sm_count();

#define TDX_CHECK_CUDA(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::tdx::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return TDX_E_CUDA;                                                                       \
    }                                                                                          \
  } while (0)

#define TDX_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      ::tdx::set_error(__VA_ARGS__);      \
      return TDX_E_INVALID;               \
    }                                     \
  } while (0)

bool first_use_on_device(bool (&seen)[16]);

// The one way libtdx launches a kernel: with programmatic dependent launch (PDL) allowed and, when cluster > 1, in
// thread-block clusters of `cluster` CTAs along x.  Returns the launch's error; call sites wrap it in TDX_CHECK_CUDA so
// that a failure names them.
//
// Under PDL a kernel may start while its predecessor in the stream is still running; only griddepcontrol.wait orders
// it after that predecessor's completion.  So every libtdx kernel calls pdl_wait() (tdx_ptx.cuh) before it touches data
// an earlier kernel produced and before any of its threads returns, even a kernel that reads nothing earlier kernels
// wrote: one that did not wait could finish before its predecessor, and a later kernel waiting on it would then not be
// ordered after that predecessor.  Kernels open with pdl_launch_dependents(); pdl_wait(); (the igemm kernel first runs
// its prologue) so that the next launch overlaps its own prologue with this kernel's tail.
// tests/test_launch_policy_cpu.py checks the rule on the sources.
template <typename... Params, typename... Args>
cudaError_t launch_clustered(unsigned cluster, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem,
                             void* stream, Args&&... args) {
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = reinterpret_cast<cudaStream_t>(stream);
  cfg.attrs = attr;
  cfg.numAttrs = cluster > 1 ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

template <typename... Params, typename... Args>
cudaError_t launch(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, void* stream, Args&&... args) {
  return launch_clustered(1, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}

// bf16 NC8HW8 activation -> 4-D tiled tensor map (dims: W*8 elems, H, C/8, N; box: 80 x 18 x 8 x 1).
int make_act_tensor_map(CUtensorMap* out, const void* base, int n_img, int channels, int height, int width);

}  // namespace tdx
