// Internal helpers shared by the libtdx translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

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
// Launch configuration with programmatic dependent launch (PDL) enabled: every libtdx kernel calls
// griddepcontrol.wait before touching data produced by earlier kernels, so consecutive launches may overlap their
// prologue (barrier init, weight prefetch) with the previous kernel's tail.
void fill_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, dim3 grid, dim3 block, size_t smem,
                        cudaStream_t stream);

// bf16 NC8HW8 activation -> 4-D tiled tensor map (dims: W*8 elems, H, C/8, N; box: 80 x 18 x 8 x 1).
int make_act_tensor_map(CUtensorMap* out, const void* base, int n_img, int channels, int height, int width);

}  // namespace tdx
