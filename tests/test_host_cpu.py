"""CPU-side checks (run with -m "not gpu"): host logic of the product package, the C ABI surface, loud failure."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import tiling as otile
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import tiling as ptile
from terrain_diffusion_b200.layout import from_nc8hw8, pack_weight_segments, to_nc8hw8
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.models.plan import block_plan, effective_weight, mp_concat_scales
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "reference_golden.npz")


def test_library_exports_every_symbol_declared_in_header():
    hdr = (ROOT / "include" / "tdx.h").read_text()
    names = sorted(set(re.findall(r"\b(tdx_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 20
    lib = L.lib()
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_abi_struct_sizes_match_ctypes():
    lib = L.lib()
    for i, st in enumerate(L.ABI_STRUCTS):
        assert lib.tdx_abi_sizeof(i) == C.sizeof(st), st.__name__


def test_descriptor_validation_runs_without_gpu():
    d = L.TdxIgemmDesc()
    assert L.lib().tdx_igemm_run(C.byref(d), None) == -1
    d.n_seg = 1
    d.a_ptr[0] = 16
    d.a_channels[0] = 48
    d.a_taps[0] = 9
    assert L.lib().tdx_igemm_run(C.byref(d), None) == -1
    assert b"multiple of 64" in L.lib().tdx_last_error()


def test_model_refuses_cpu_tensors_loudly():
    m = EDMUnet2D(**ounet.DECODER_CFG).eval()
    with pytest.raises(L.TdxError):
        m(torch.zeros(1, 5, 64, 64), torch.zeros(1), [])


def test_model_state_dict_layout_matches_reference():
    m = EDMUnet2D(**ounet.DECODER_CFG)
    shapes = ounet.state_shapes(ounet.DECODER_CFG)
    sd = m.state_dict()
    assert set(sd) == set(shapes)
    assert all(tuple(sd[k].shape) == tuple(shapes[k]) for k in sd)
    assert m.count_parameters() == 27922533
    assert m.config.model_channels == 64 and m.config.concat_balance == 0.5


def test_block_plan_and_folding_match_oracle():
    assert block_plan(ounet.DECODER_CFG) == ounet.block_plan(ounet.DECODER_CFG)
    w = torch.randn(64, 128, 3, 3)
    assert torch.equal(effective_weight(w, 0.7), ounet.effective_weight(w, 0.7))
    assert mp_concat_scales(256, 192, 0.5) == ounet.mp_concat_scales(256, 192, 0.5)
    # the closed-form scalars equal what mp_concat multiplies with
    a, b = torch.ones(1, 256, 1, 1), torch.ones(1, 192, 1, 1)
    cat = ounet.mp_concat([a, b], 0.5)
    s1, s2 = mp_concat_scales(256, 192, 0.5)
    assert abs(float(cat[0, 0, 0, 0]) - s1) < 1e-6 and abs(float(cat[0, -1, 0, 0]) - s2) < 1e-6


def test_layout_roundtrip_and_weight_packing_order():
    x = torch.randn(2, 64, 5, 7)
    assert torch.equal(from_nc8hw8(to_nc8hw8(x)), x.bfloat16().float())
    w = (torch.arange(128 * 128 * 9, dtype=torch.float32).reshape(128, 128, 3, 3) % 509) / 64
    w1 = (torch.arange(128 * 64, dtype=torch.float32).reshape(128, 64, 1, 1) % 251) / 32
    p = pack_weight_segments([w, w1]).float().reshape(2, -1)  # [split][stages...]
    p3 = p[:, :2 * 9 * 8 * 64 * 8].reshape(2, 2, 9, 8, 64, 8)  # [split, chunk, tap, kgroup, n, e]
    for (s_, ch, tap, kg, n, e) in [(0, 0, 0, 0, 0, 0), (1, 1, 4, 3, 17, 5), (0, 1, 8, 7, 63, 7), (1, 0, 2, 5, 40, 1)]:
        assert p3[s_, ch, tap, kg, n, e] == w[s_ * 64 + n, ch * 64 + kg * 8 + e, tap // 3, tap % 3].bfloat16().float()
    p1 = p[:, 2 * 9 * 8 * 64 * 8:].reshape(2, 1, 1, 8, 64, 8)
    assert p1[1, 0, 0, 2, 9, 3] == w1[64 + 9, 2 * 8 + 3, 0, 0].bfloat16().float()


def test_tiling_host_logic_is_bit_exact_with_reference_golden():
    cases, lens, flat = G["tile_starts.cases"], G["tile_starts.lens"], G["tile_starts.flat"]
    off = 0
    for (length, tile, stride), n in zip(cases.tolist(), lens.tolist()):
        assert ptile.tile_starts(length, tile, stride) == flat[off:off + n].tolist()
        off += n
    for size in (4, 8, 64):
        np.testing.assert_array_equal(ptile.linear_weight_window(size).numpy(), G[f"window{size}"])
    assert [ptile.padded_batch_size(n, 16) for n in (1, 2, 3, 5, 9, 16, 17)] == [1, 2, 4, 8, 16, 16, 16]
    rows = [list(ptile.shard_rows(23, 8, r)) for r in range(8)]
    assert sum(rows, []) == list(range(23))


def test_window_range_integer_rule_matches_oracle_everywhere():
    import random
    rnd = random.Random(0)
    for _ in range(3000):
        a = rnd.randint(-600, 600)
        b = a + rnd.randint(1, 700)
        size, stride, off = rnd.randint(1, 90), rnd.randint(1, 90), rnd.randint(-9, 9)
        assert list(ptile.window_range(a, b, size, stride, off)) == list(otile.window_range(a, b, size, stride, off))


def test_scheduler_tables_and_errors_on_cpu():
    for n in (4, 12, 20):
        s = EDMDPMSolverMultistepScheduler()
        s.set_timesteps(n)
        np.testing.assert_array_equal(s.sigmas.numpy(), G[f"sched{n}.sigmas"])
        np.testing.assert_array_equal(s.timesteps.numpy(), G[f"sched{n}.timesteps"])
        np.testing.assert_array_equal(s.trigflow_precondition_noise(s.sigmas[:-1]).numpy(), G[f"sched{n}.cnoise"])
        assert s.order_schedule() == [False] + [True] * (n - 2) + [False]
    s = EDMDPMSolverMultistepScheduler()
    with pytest.raises(ValueError):
        s.step(torch.zeros(1), torch.tensor(0.0), torch.zeros(1))
    s.set_timesteps(4)
    for mo, x in ((torch.zeros(1), torch.zeros(2)), (torch.zeros(2, 3), torch.zeros(3, 2)),
                  (torch.zeros(4), torch.zeros(1))):
        with pytest.raises(ValueError, match="model_output shape"):       # before the device check
            s.step(mo, s.timesteps[0], x)
    with pytest.raises(L.TdxError):
        s.step(torch.zeros(1), s.timesteps[0], torch.zeros(1))
    with pytest.raises(NotImplementedError):
        EDMDPMSolverMultistepScheduler(solver_order=3)


def test_first_convolution_weight_matrix_of_the_im2col_path_reproduces_the_3x3_convolution():
    """FoldedWeights lays the first MPConv's effective weights out as [cout][k_pad] with k = tap*ci + c, the channel order
    tdx_im2col_run writes (include/tdx.h): unfold(cat([x, ones])) @ W^T must equal conv2d(cat([x, ones]), w, padding=1)."""
    import torch.nn.functional as F

    from terrain_diffusion_b200.models.plan import FoldedWeights
    cfg = ounet.DECODER_CFG
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=3))
    fw = FoldedWeights(m, torch.device("cpu"))
    first = fw.enc[0]["name"]
    w_in = effective_weight(m.state_dict()[f"enc.{first}.weight"].float())       # [cout][ci][3][3]
    ci = w_in.shape[1]
    assert fw.conv_in_kpad == 64 and ci == 6
    w_mat = fw.segs["conv_in.im2col"][0]
    assert tuple(w_mat.shape) == (w_in.shape[0], 64, 1, 1) and torch.count_nonzero(w_mat[:, 9 * ci:]) == 0
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(2, ci - 1, 12, 10, generator=g), torch.ones(2, 1, 12, 10)], dim=1)
    cols = F.unfold(x, kernel_size=3, padding=1).view(2, ci, 9, 12, 10).permute(0, 2, 1, 3, 4).reshape(2, 9 * ci, 12, 10)
    got = torch.einsum("ok,nkhw->nohw", w_mat[:, :9 * ci, 0, 0], cols)
    ref = F.conv2d(x, w_in, padding=1)
    assert torch.allclose(got, ref, atol=1e-5, rtol=1e-5)


def test_new_entry_points_validate_their_arguments_without_a_gpu():
    """im2col / read-out primitives reject bad descriptors before any CUDA call (return codes + tdx_last_error)."""
    lib = L.lib()
    d = L.TdxIm2colDesc()
    assert lib.tdx_im2col_run(C.byref(d), None) != 0 and b"src[0]" in lib.tdx_last_error()
    d.src[0] = 16
    d.src_channels[0] = 3                       # 3 + ones = 4 input channels: not one of the shipped models
    d.out = 16
    d.k_pad = 64
    d.n_img, d.height, d.width = 1, 8, 8
    assert lib.tdx_im2col_run(C.byref(d), None) != 0 and b"input channels" in lib.tdx_last_error()
    d.src_channels[0] = 5
    d.k_pad = 128                               # 9 * 6 = 54 -> must be 64
    assert lib.tdx_im2col_run(C.byref(d), None) != 0 and b"k_pad" in lib.tdx_last_error()
    p = C.c_void_p(16)
    assert lib.tdx_gaussian_blur(p, 16, 16, p, 11, 5.0, None) != 0 and b"aliased" in lib.tdx_last_error()
    q = C.c_void_p(32)
    assert lib.tdx_gaussian_blur(p, 16, 16, q, 10, 5.0, None) != 0 and b"kernel size" in lib.tdx_last_error()
    assert lib.tdx_gaussian_blur(p, 5, 16, q, 11, 5.0, None) != 0 and b"reflect" in lib.tdx_last_error()
    assert lib.tdx_resize_aa_axis(p, 8, 8, q, 16, 2, None) != 0 and b"axis" in lib.tdx_last_error()
    assert lib.tdx_post_combine(p, 4, q, 8, q, None, 8, 8, 0, None) != 0      # pitch smaller than the width
    assert lib.tdx_lapse_rate(p, q, 10, 20, 15, -0.012, 0.0, -0.0065, 1e-6, 0.02, q, q, None) != 0
    assert b"window" in lib.tdx_last_error()
    assert lib.tdx_climate_sample(p, p, p, 4, 20, 20, 7, p, 0, 0, 8, 8, 256, 0, 0, q, None) != 0
    assert b"channels" in lib.tdx_last_error()


def test_latent_stage_seed_offsets_match_the_reference_call_sites():
    """ADVICE r1 (high): _build_latent_stage passes seed_offset 5819 to the init phase and 5820 + i to phase i
    (world_pipeline.py:1133-1203).  tests/golden/make_golden_stages.py reads both out of the reference SOURCE with ast
    and stores them; the pipeline's wiring constants must be those, or the same world seed gives different latents."""
    from pathlib import Path
    from terrain_diffusion_b200.inference import pipeline
    g = np.load(Path(__file__).resolve().parent / "golden" / "stages_golden.npz")
    offs = [int(v) for v in g["latent_seed_offsets"]]
    assert offs == [5819, 5820]
    assert [pipeline.LATENT_INIT_SEED_OFFSET, pipeline.LATENT_STEP_SEED_OFFSET] == offs


def test_integration_md_ctypes_stub_matches_the_library_abi(tmp_path):
    """VERDICT r1: the binding printed in INTEGRATION.md must be the real ABI.  The python block is taken FROM THE
    DOCUMENT TEXT, pointed at the built library and executed: its struct sizes must equal tdx_abi_sizeof (the stub
    asserts that itself) and its field list must be the header's."""
    import re
    from pathlib import Path
    from terrain_diffusion_b200 import _lib as L
    text = (Path(__file__).resolve().parent.parent / "INTEGRATION.md").read_text()
    blocks = re.findall(r"```python\n(.*?)```", text, flags=re.S)
    stub = next(b for b in blocks if "class TdxIgemmDesc" in b)
    stub = stub.replace('C.CDLL("libtdx.so")', f'C.CDLL({str(L.LIB_PATH)!r})')
    ns: dict = {}
    exec(compile(stub, "INTEGRATION.md", "exec"), ns)           # runs the stub's own sizeof assertion
    doc_fields = [f[0] for f in ns["TdxIgemmDesc"]._fields_]
    assert doc_fields == [f[0] for f in L.TdxIgemmDesc._fields_]
    assert C.sizeof(ns["TdxIgemmDesc"]) == C.sizeof(L.TdxIgemmDesc) == L.lib().tdx_abi_sizeof(1)
    header = (Path(__file__).resolve().parent.parent / "include" / "tdx.h").read_text()
    body = header[header.index("typedef struct TdxIgemmDesc {"):header.index("} TdxIgemmDesc;")]
    for name in doc_fields:
        assert re.search(r"\b" + re.escape(name) + r"\b", body), name


def test_blend_window_cache_and_device_constant_cache():
    """Round 2 host-side caches: the blend window is computed once per (size, device, dtype) and equals the reference
    formula (world_pipeline.py:117-124); small host constants of the stage functions are cached by CONTENT."""
    from terrain_diffusion_b200.inference import stages
    from terrain_diffusion_b200.inference.tiling import linear_weight_window
    w1, w2 = linear_weight_window(64), linear_weight_window(64, "cpu", torch.float32)
    assert w1 is w2 and w1.shape == (64, 64)
    mid = 31.5
    y = torch.arange(64).float()
    wy = 1 - (1 - 1e-3) * torch.clamp((y - mid).abs() / mid, 0, 1)
    assert torch.equal(w1, wy[:, None] * wy[None, :])
    assert linear_weight_window(32) is not w1 and float(w1.min()) > 0
    a = torch.tensor([1.0, 2.0, 3.0])
    c1 = stages._const_on(torch.device("cpu"), a)
    c2 = stages._const_on(torch.device("cpu"), a.clone())           # another object, the same content: the same entry
    c3 = stages._const_on(torch.device("cpu"), torch.tensor([1.0, 2.0, 4.0]))
    assert c1 is c2 and c3 is not c1 and torch.equal(c3, torch.tensor([1.0, 2.0, 4.0]))
    a[0] = 9.0                                                      # mutating the source later does not poison the cache
    assert float(stages._const_on(torch.device("cpu"), torch.tensor([1.0, 2.0, 3.0]))[0]) == 1.0
    s = stages._concat_scales([16, 16, 4, 16, 5, 1], torch.device("cpu"))
    assert s.shape == (58,) and abs(float((s[:16] ** 2).sum() * 6) - 58.0 / 6 * 6) < 1e-3


def test_batched_noise_entry_point_validates_without_a_gpu():
    import ctypes as C
    lib = L.lib()
    ys, xs = (C.c_int64 * 2)(0, 32), (C.c_int64 * 2)(0, 32)
    assert lib.tdx_noise_patches(1, 2, ys, xs, 64, 64, 5, 64, 64, None, None, 0, None) == -1
    assert b"null" in lib.tdx_last_error()
    need = lib.tdx_noise_patches_workspace_bytes(5, 64, 64)
    assert need >= 32 * lib.tdx_noise_patch_workspace_bytes(5, 64, 64) - 32 * 256
    assert lib.tdx_noise_patches(1, 2, ys, xs, 64, 64, 5, 64, 64, C.c_void_p(16), C.c_void_p(16), 8, None) == -1
    assert b"workspace" in lib.tdx_last_error()
