"""libtdx's one launch policy, read from the sources under csrc/ (no GPU and no build needed).

Every kernel is launched through `launch` / `launch_clustered` of tdx_common.h, which allows programmatic dependent
launch (PDL): a kernel may then start while its predecessor in the stream is still running.  That is only correct if
every kernel runs griddepcontrol.wait (`pdl_wait()`) before it touches earlier results and before any of its threads
returns -- a kernel that exits without waiting can finish before its predecessor, and a later kernel that waits on it
would no longer be ordered after that predecessor.

The code a kernel runs before its first pdl_wait() overlaps its predecessor, so it must not touch global memory: no
__ldg, TMA or bulk copy, atomic, subscript outside a __shared__ declaration, or call to a helper that could hide one.
The kernels in EARLY_READS are the exceptions, each reading only what no launch writes.  This text check is what
covers the second and later kernels of a multi-kernel entry point; tests/test_pdl_order_gpu.py checks the first one
(and every launch of the shipped programs) on the device, behind a kernel still writing their inputs."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parent.parent / "terrain_diffusion_b200" / "csrc"
HELPER = "tdx_common.h"

# kernels that read global memory before pdl_wait(), and why that is safe
EARLY_READS = {
    "conv_out_kernel": "stages the weights in shared memory; tdx.h requires them not to be written by an in-flight "
                       "launch",
    "fbm_kernel": "load_gradients reads the __device__ gradient table, a constant no launch writes",
    "synth_kernel": "load_gradients reads the __device__ gradient table, a constant no launch writes",
    "igemm_kernel": "its prologue prefetches the tensor-map descriptors (kernel parameters) before any warp waits, and "
                    "the B producer streams the packed weights (constants by tdx.h) without waiting; the per-warp waits "
                    "are beyond a text check, so tests/test_pdl_order_gpu.py covers them",
}
# what code before the first pdl_wait() may call
PRE_WAIT_CALLS = {"pdl_launch_dependents", "static_assert", "__align__", "if", "for", "while", "sizeof"}
GLOBAL_ACCESS = re.compile(r"__ldg|\bld\.global|\btma_\w*|\bbulk_\w*|cp\.async|\batomic\w*")


def _sources() -> dict:
    return {p.name: p.read_text() for p in sorted(CSRC.iterdir()) if p.suffix in (".cu", ".cuh", ".h")}


def _code(text: str) -> str:
    """The source with comments blanked out (string literals kept, so a "//" inside one is not a comment)."""
    return re.sub(r'"(?:\\.|[^"\\\n])*"|//[^\n]*|/\*.*?\*/',
                  lambda m: m.group(0) if m.group(0).startswith('"') else " ", text, flags=re.S)


def _kernels(code: str):
    """(name, body) of every __global__ function defined in `code`."""
    for m in re.finditer(r"\b__global__\b", code):
        i, depth = m.end(), 0
        while depth or code[i] not in "{;":            # skip __launch_bounds__(...) and the parameter list
            depth += {"(": 1, ")": -1}.get(code[i], 0)
            i += 1
        assert code[i] == "{", f"__global__ declaration without a body: {code[m.start():i + 1]!r}"
        names = re.findall(r"(\w+)\s*\(", code[m.end():i])
        start, depth = i, 0
        while True:
            depth += {"{": 1, "}": -1}.get(code[i], 0)
            i += 1
            if depth == 0:
                break
        yield names[-1], code[start:i]


def test_sources_are_found():
    src = _sources()
    assert HELPER in src and "tdx_noise.cu" in src and "tdx_igemm.cu" in src
    assert sum(1 for text in src.values() for _ in _kernels(_code(text))) > 40


def test_no_triple_chevron_launches():
    found = [name for name, text in _sources().items() if "<<<" in text]
    assert not found, f"<<<>>> launches bypass the PDL launch helper: {found}"


def test_fill_launch_config_is_gone():
    found = [name for name, text in _sources().items() if "fill_launch_config" in text]
    assert not found, found


def test_kernel_launch_api_is_called_only_by_the_helper():
    calls = [(name, m.group(0)) for name, text in _sources().items()
             for m in re.finditer(r"\bcu(?:da)?Launch(?:Cooperative)?Kernel\w*(?=\s*\()", _code(text))]
    assert calls == [(HELPER, "cudaLaunchKernelEx")], calls


def test_every_kernel_waits_before_it_returns():
    late = []
    for name, text in _sources().items():
        for kernel, body in _kernels(_code(text)):
            wait = body.find("pdl_wait()")
            ret = re.search(r"\breturn\b", body)
            if wait < 0 or (ret and ret.start() < wait):
                late.append(f"{name}: {kernel}")
    assert not late, f"kernels that can return (or finish) without pdl_wait(): {late}"


def _early_access(body: str) -> list:
    """What the code before the first pdl_wait() of a kernel body does that may touch global memory."""
    pre = body[1:body.find("pdl_wait()")]
    found = [m.group(0) for m in GLOBAL_ACCESS.finditer(pre)]
    for stmt in re.split(r"[;{}]", pre):
        if "__shared__" not in stmt:
            found += [f"subscript {m.group(0)}" for m in re.finditer(r"\w+\s*\[", stmt)]
    found += [f"call {m.group(1)}()" for m in re.finditer(r"\b(\w+)\s*\(", pre) if m.group(1) not in PRE_WAIT_CALLS]
    return found


def test_no_kernel_touches_global_memory_before_it_waits():
    early, seen = {}, set()
    for name, text in _sources().items():
        for kernel, body in _kernels(_code(text)):
            found = _early_access(body)
            if found:
                seen.add(kernel)
                if kernel not in EARLY_READS:
                    early[f"{name}: {kernel}"] = found
    assert not early, f"kernels that may touch global memory before pdl_wait(): {early}"
    stale = sorted(set(EARLY_READS) - seen)
    assert not stale, f"EARLY_READS entries whose kernels no longer read before waiting: {stale}"


def test_early_access_check_sees_loads_subscripts_and_helpers():
    def body(pre):
        return "{" + pre + " pdl_wait(); out[0] = 1; }"
    assert _early_access(body("__shared__ float s[64]; pdl_launch_dependents();")) == []
    assert _early_access(body("float v = __ldg(x);"))
    assert _early_access(body("float v = x[threadIdx.x];"))
    assert _early_access(body("atomicAdd(c, 1);"))
    assert _early_access(body("tma_load_4d(&tm, bar, dst, 0, 0, 0, 0);"))
    assert _early_access(body("load_gradients(g);"))
