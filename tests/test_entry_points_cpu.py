"""Every C entry point of libtdx is named by some test, so none is reached only through a Python wrapper that always
passes the same well-formed arguments.  Needs no GPU and no build: it reads include/tdx.h, the `extern "C"` definitions
under csrc/ and the test sources."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "tdx.h"
CSRC = ROOT / "terrain_diffusion_b200" / "csrc"

# entry points no test names directly, each with the reason
ALLOWLIST = {
    "tdx_debug_set_igemm_trace": "debug hook compiled only into debug builds; tools/trace_igemm.py drives it",
    "tdx_debug_set_igemm_timeline": "debug hook compiled only into debug builds; tools/timeline_forward.py drives it",
    "tdx_igemm_packed_weight_elems": "sizes the packed weights in models/plan.py, which every model test runs",
    "tdx_program_create": "models/plan.py builds every model forward as a program; every model test runs it",
    "tdx_program_add_im2col": "models/plan.py records the first convolution; every model test runs it",
    "tdx_program_add_igemm": "models/plan.py records every convolution; every model test runs it",
    "tdx_program_add_conv_out": "models/plan.py records the last convolution; every model test runs it",
    "tdx_program_add_embed": "models/plan.py records the embedding; every model test runs it",
    "tdx_program_add_attn": "models/plan.py records the attention blocks; every model test runs it",
    "tdx_program_num_launches": "models/plan.py sizes its profile buffers with it; every model test runs it",
    "tdx_program_run": "models/plan.py replays every forward through it; every model test runs it",
    "tdx_program_instantiate": "models/plan.py instantiates the graph before timing; every model test runs it",
    "tdx_program_profile": "models/plan.py's per-launch profile; the planner tests run it",
    "tdx_program_destroy": "models/plan.py frees every program; every model test runs it",
}


def header_entry_points() -> set:
    src = re.sub(r"/\*.*?\*/", " ", HEADER.read_text(), flags=re.S)
    return set(re.findall(r"\b(tdx_\w+)\s*\(", src))


def exported_entry_points() -> set:
    names = set()
    for f in CSRC.glob("*.cu"):
        names |= set(re.findall(r'extern\s+"C"\s+[\w\s\*]*?\b(tdx_\w+)\s*\(', f.read_text()))
    return names


def _test_code() -> str:
    """The tests and their helpers (tests/_*.py), without this file."""
    return "\n".join(p.read_text() for p in sorted((ROOT / "tests").glob("*.py")) if p.name != Path(__file__).name)


def test_header_parses():
    names = header_entry_points()
    assert len(names) > 50
    for n in ("tdx_flow_d8", "tdx_fill_depressions", "tdx_noise_patch", "tdx_tile_seed", "tdx_canvas_add",
              "tdx_program_run", "tdx_last_error"):
        assert n in names, n


def test_every_exported_function_is_declared_or_a_debug_hook():
    undeclared = exported_entry_points() - header_entry_points()
    assert undeclared == {n for n in undeclared if n.startswith("tdx_debug_")}, sorted(undeclared)
    missing = sorted(header_entry_points() - exported_entry_points())
    assert not missing, f"declared in tdx.h but not defined as extern \"C\" under csrc/: {missing}"


def test_every_entry_point_is_named_by_a_test():
    tests = _test_code()
    names = header_entry_points() | exported_entry_points()
    untested = sorted(n for n in names if n not in ALLOWLIST and not re.search(rf"\b{n}\b", tests))
    assert not untested, f"entry points no test names (test them directly or allowlist them): {untested}"


def test_allowlist_is_current():
    names = header_entry_points() | exported_entry_points()
    stale = sorted(n for n in ALLOWLIST if n not in names)
    assert not stale, f"allowlisted entry points that no longer exist: {stale}"
    tests = _test_code()
    covered = sorted(n for n in ALLOWLIST if not n.startswith("tdx_debug_") and re.search(rf"\b{n}\b", tests))
    assert not covered, f"allowlisted entry points that a test now names (drop them from the allowlist): {covered}"
