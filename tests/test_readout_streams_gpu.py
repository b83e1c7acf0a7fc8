"""Where the read-out launches: every libtdx call of the elevation, climate, terrain API, Minecraft API, relief and
river-routing entry points goes to the current stream of its tensors' device, with that device current.

`L.lib` is replaced by a proxy that records, for each `tdx_*` call, its last argument (the stream) and the current
device, and then forwards the call.
1. Under `torch.cuda.stream(side)` every launch of an entry point goes to `side`, and the outputs are bit for bit those
   of the same call on the default stream (NaN compared by position).
2. With two GPUs, inputs on cuda:1 while cuda:0 is current: every launch runs with device 1 current, on cuda:1's
   current stream, and the outputs are bit for bit those computed on cuda:0.  No stream context is entered here, since
   entering one makes the stream's device current."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import d8_flow, flow_accumulation, get_relief_map, plot_flow_indicator
from terrain_diffusion_b200.inference import minecraft as M
from terrain_diffusion_b200.inference import postproc as P
from tests._hydrology_inputs import hydrology_case
from tests._minecraft_inputs import case_world as minecraft_case
from tests._minecraft_inputs import stand_in_noise
from tests._post_inputs import (COASTAL_SCALE, COASTAL_WINDOW, ELEV_WINDOWS, RESIDUAL_MEAN, RESIDUAL_STD,
                                coastal_canvas, coastal_elev, elev_canvases, field, laplacian_case)
from tests._relief_inputs import relief_case
from tests._terrain_api_inputs import case_world as terrain_case

pytestmark = pytest.mark.gpu


class Recorder:
    """Stands in for the loaded library: records (name, last argument, current device) of every tdx_* call."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if not name.startswith("tdx_"):
            return fn

        def recorded(*args):
            self.calls.append((name, args[-1] if args else None, torch.cuda.current_device()))
            return fn(*args)
        return recorded


@pytest.fixture
def recorder(monkeypatch):
    rec = Recorder(L.lib())
    monkeypatch.setattr(L, "lib", lambda: rec)
    return rec


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


class DeviceCanvas:
    """canvas[:, a:b, c:d] of a tests._post_inputs.FakeCanvas as a tensor on `device`, like the pipeline's canvases."""

    def __init__(self, fake, device):
        self.fake, self.device = fake, device

    def __getitem__(self, key):
        _, ys, xs = key
        return _t(self.fake.planes(ys.start, ys.stop, xs.start, xs.stop), self.device)


def _resize(dev):
    return [P.resize_bilinear(_t(field(7, 12, 10), dev), (96, 80)), P.resize_bilinear(_t(field(8, 64, 136), dev), 17)]


def _pad(dev):
    return [P.pad_linear_extrapolation(_t(field(3, 13, 9, 1.0, 2.0), dev))]


def _blur(dev):
    return [P.gaussian_blur(_t(field(5, 17, 36, -30.0, 40.0), dev), 11, 5.0)]


def _decode(dev):
    r, low = (_t(a, dev) for a in laplacian_case("rect"))
    return [P.laplacian_decode(r, low), P.laplacian_decode(r, low, extrapolate=True)]


def _elev(dev):
    resid, lat = elev_canvases()
    return list(P.compute_elev(DeviceCanvas(resid, dev), DeviceCanvas(lat, dev), *ELEV_WINDOWS["neg_square"], 8,
                               RESIDUAL_MEAN, RESIDUAL_STD, as_int16=True))


def _climate(dev):
    return [P.compute_climate(DeviceCanvas(coastal_canvas(), dev), *COASTAL_WINDOW, _t(coastal_elev(), dev),
                              COASTAL_SCALE)]


def _upsample(dev):
    world, (i1, j1, i2, j2, scale) = terrain_case("specials_s8")
    ni1, nj1, ni2, nj2, oi, oj = P.terrain_window(i1, j1, i2, j2, scale)
    native = world.get(ni1, nj1, ni2, nj2)
    e, c = native["elev"].to(dev), native["climate"].to(dev)
    H, W = i2 - i1, j2 - j1
    return [P.upsample_crop(e, c, scale, oi, oj, H, W), P.upsample_crop(e, c, scale, oi, oj, H, W, payload=True),
            P.upsample_crop(e, None, scale, oi, oj, H, W)]


def _minecraft(dev):
    out = []
    for name in ("s1_16_nr30", "s2_64x96"):                # scale 1 reads a centre window; scale 2 adds detail noise
        world, (i1, j1, i2, j2, scale, noise) = minecraft_case(name)

        def get_device(*a, world=world):
            return {k: None if v is None else v.to(dev) for k, v in world.get(*a).items()}
        (planes, biome), _ = M.request(get_device, world.native_resolution, i1, j1, i2, j2, scale, noise,
                                       stand_in_noise, False)
        body, _ = M.request(get_device, world.native_resolution, i1, j1, i2, j2, scale, noise, stand_in_noise, True)
        out += [planes, biome, body]
    return out


def _relief(dev):
    out = []
    for name in ("nan", "vrange"):                         # the NaN-median fill; a user colour range
        elev, kw = relief_case(name)
        out.append(get_relief_map(_t(elev, dev), None, None, None, **kw))
    return out


def _rivers(dev):
    z = _t(hydrology_case("mixed")[0], dev)
    rr, cc, sink, kmax = d8_flow(z)
    return [rr, cc, sink, kmax, flow_accumulation(z, rr, cc, sink), plot_flow_indicator(z, 3)]


CASES = {"resize_bilinear": _resize, "pad_linear_extrapolation": _pad, "gaussian_blur": _blur,
         "laplacian_decode": _decode, "compute_elev": _elev, "compute_climate": _climate, "upsample_crop": _upsample,
         "minecraft_readout": _minecraft, "get_relief_map": _relief, "rivers": _rivers}


def _host(outs):
    assert outs and all(isinstance(t, torch.Tensor) and t.is_cuda for t in outs)
    return [t.cpu().numpy() for t in outs]


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for k, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.dtype == w.dtype, (what, k, g.shape, w.shape, g.dtype, w.dtype)
        if g.dtype.kind == "f":
            nan = np.isnan(w)
            assert np.array_equal(np.isnan(g), nan), f"{what} output {k}: NaN positions differ"
            g, w = np.where(nan, 0, g), np.where(nan, 0, w)
        assert g.tobytes() == w.tobytes(), f"{what} output {k}: bits differ"


@pytest.mark.parametrize("name", sorted(CASES))
def test_readout_launches_on_the_current_stream(name, recorder):
    dev = torch.device("cuda", torch.cuda.current_device())
    want = _host(CASES[name](dev))
    default = torch.cuda.current_stream(dev).cuda_stream
    assert recorder.calls and all(s == default for _, s, _ in recorder.calls), recorder.calls
    recorder.calls.clear()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        outs = CASES[name](dev)
    side.synchronize()
    assert recorder.calls
    for fn, stream, device in recorder.calls:
        assert stream == side.cuda_stream and device == dev.index, (fn, stream, side.cuda_stream, device)
    assert_same(_host(outs), want, name)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
@pytest.mark.parametrize("name", sorted(CASES))
def test_readout_launches_on_the_inputs_device(name, recorder):
    want = _host(CASES[name](torch.device("cuda:0")))
    recorder.calls.clear()
    with torch.cuda.device(0):
        got = _host(CASES[name](torch.device("cuda:1")))
    stream1 = torch.cuda.current_stream(1).cuda_stream
    assert recorder.calls
    for fn, stream, device in recorder.calls:
        assert device == 1 and stream == stream1, (fn, stream, stream1, device)
    assert_same(got, want, name)
