"""libtdx's one launch policy, read from the sources under csrc/ (no GPU and no build needed).

Every kernel is launched through `launch` / `launch_clustered` of tdx_common.h, which allows programmatic dependent
launch (PDL): a kernel may then start while its predecessor in the stream is still running.  That is only correct if
every kernel runs griddepcontrol.wait (`pdl_wait()`) before it touches earlier results and before any of its threads
returns -- a kernel that exits without waiting can finish before its predecessor, and a later kernel that waits on it
would no longer be ordered after that predecessor."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parent.parent / "terrain_diffusion_b200" / "csrc"
HELPER = "tdx_common.h"


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
