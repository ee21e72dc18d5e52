"""The output step of every frame (csrc/raster.cu write_pixel / store_pixel2, csrc/api.cu frame_out) on the GPU:

* cross-format exactness: per blend kernel and output mode, the RGBA16F frame is the round-to-nearest-even half of the
  RGBA32F frame bit for bit (in blend-over mode the f32 run blends over the half target's exact values), the RGBA8
  alpha bytes are the f32 restatement of the encoder applied to the RGBA32F alpha, and the RGBA8 colour bytes are the
  correctly rounded sRGB encoding of the RGBA32F colour outside the derived band (output_cases.SRGB8_BAND);
* pixels no splat blends keep their bytes when blending over ramp targets that hold every value a channel can take;
* compositing chains of 1-4 clouds against the float64 blend of the oracle's trace, identical across call orders
  (synchronous, queued, mixed) and target kinds (library frames, torch, exported and peer-buffer device memory);
* a blend-over frame whose pair list overflows a fresh context's buffer is composited once;
* device targets: RGBA8 at 4-byte but not 8-byte alignment renders the aligned frame; misaligned RGBA16F / RGBA32F
  targets are refused and left untouched.

The RGBA32F frames themselves are held to the oracle by test_gpu_blend.py.
"""
import ctypes as C
import os

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import kernel_paths as KP
import output_cases as OC
import test_gpu_blend as TB
from bevy_gaussian_splatting_b200 import abi

pytestmark = pytest.mark.gpu

FMTS = ("rgba32f", "rgba16f", "rgba8_srgb")
MODES = ("opaque", "premultiplied", "over")
GUARD = 256
BAND_COUNTS = {}


def _cu():
    cu = C.CDLL("libcuda.so.1")
    cu.cuMemcpyDtoH_v2.argtypes = [C.c_void_p, C.c_uint64, C.c_size_t]
    cu.cuMemcpyHtoD_v2.argtypes = [C.c_uint64, C.c_void_p, C.c_size_t]
    return cu


class Target:
    """A device frame of `fmt` at `offset` bytes past a 256-byte boundary, with guard bytes on both sides."""

    def __init__(self, view, fmt, offset=0, dst=None):
        import torch

        self.shape, self.dtype = (view.height, view.width, 4), B.GaussianSplattingPlugin.FORMATS[fmt][1]
        self.nbytes = int(np.prod(self.shape)) * np.dtype(self.dtype).itemsize
        self.offset = offset
        self.buf = torch.full((2 * GUARD + offset + self.nbytes,), 0xA5, dtype=torch.uint8, device="cuda")
        if dst is not None:
            self.write(dst)
        torch.cuda.synchronize()

    @property
    def ptr(self):
        return self.buf.data_ptr() + GUARD + self.offset

    def write(self, a):
        import torch

        a = np.ascontiguousarray(a, self.dtype).reshape(-1).view(np.uint8)
        self.buf[GUARD + self.offset: GUARD + self.offset + self.nbytes].copy_(torch.from_numpy(a.copy()))
        torch.cuda.synchronize()

    def read(self):
        import torch

        torch.cuda.synchronize()
        b = self.buf.cpu().numpy()
        assert np.all(b[:GUARD + self.offset] == 0xA5) and np.all(b[GUARD + self.offset + self.nbytes:] == 0xA5), "guard bytes written"
        return b[GUARD + self.offset: GUARD + self.offset + self.nbytes].copy().view(self.dtype).reshape(self.shape)


def render_to(p, h, s, view, fmt, mode, targets, asynchronous=False):
    """bgs_render (one target) or bgs_render_aux (three) into device targets -> status (no raise)."""
    code = B.GaussianSplattingPlugin.FORMATS[fmt][0]
    u, st = p._uniform_and_settings(h, s, None, asynchronous, mode == "premultiplied", mode == "over")
    v = view.to_abi()
    ptrs = [C.c_void_p(t.ptr) for t in targets]
    if len(targets) == 3:
        return p._lib.bgs_render_aux(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(st), *ptrs, code, 1)
    return p._lib.bgs_render(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(st), ptrs[0], code, 1)


def assert_path(c, p, before, fs):
    """The frame just rendered took the case's kernel: `before` = the stats of the frame before it (None: fresh context)."""
    if c.path == "rounds":
        assert fs.rounds > 1
    else:
        assert fs.rounds == 1
    if c.path == "r2":
        assert before is not None and KP.large_footprint_raster(before.n_visible, before.n_pairs)
    elif GEOM_MODE0(c) and before is not None:
        assert not KP.large_footprint_raster(before.n_visible, before.n_pairs)


def GEOM_MODE0(c):
    return OC.GEOM[c.path] == "obb3d"


def run_case(p, h, c, fmt, mode, dst=None, offset=0):
    """Render the case's frame once into fresh device targets (three for aux) -> list of frames; asserts the path."""
    before = p.frame_stats() if p._rendered else None
    ts = [Target(c.view, fmt, offset, dst) for _ in range(3 if c.aux else 1)]
    p._check(render_to(p, h, c.settings, c.view, fmt, mode, ts))
    p._rendered = True
    assert_path(c, p, before, p.frame_stats())
    return [t.read() for t in ts]


def open_case(c):
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(c.cloud)
    p._rendered = False
    if c.hinted:
        p.render_view(h, c.settings, c.view, fmt="rgba32f")        # the hints that select raster2_kernel<false>
        p._rendered = True
    return p, h


def f32_of_target(dst):
    """The RGBA32F target to blend over that holds what the kernel reads from `dst` (RGBA16F exactly; RGBA8 alpha
    exactly, colour to within its decode error)."""
    if dst.dtype == np.float16:
        return dst.astype(np.float32)
    return np.concatenate([OC.srgb_decode64(dst[..., :3] / 255.0).astype(np.float32), OC.alpha_decode_f32(dst[..., 3:])], -1)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("path", OC.PATHS)
def test_formats_are_the_rounding_of_the_f32_frame(path, mode):
    c = OC.case(path)
    dst16 = OC.seeded_target("rgba16f", c.view.height, c.view.width, 17) if mode == "over" else None
    dst8 = OC.seeded_target("rgba8_srgb", c.view.height, c.view.width, 18) if mode == "over" else None
    p, h = open_case(c)
    try:
        a16 = run_case(p, h, c, "rgba32f", mode, None if dst16 is None else f32_of_target(dst16))
        a8 = a16 if mode != "over" else run_case(p, h, c, "rgba32f", mode, f32_of_target(dst8))
        q16 = run_case(p, h, c, "rgba16f", mode, dst16)
        q8 = run_case(p, h, c, "rgba8_srgb", mode, dst8)
    finally:
        p.destroy()
    for k, (f16, h16, f8, g8) in enumerate(zip(a16, q16, a8, q8)):
        name = f"{path}/{mode}/{['colour', 'depth', 'normal'][k]}"
        want16 = OC.pack_rgba16f(f16)
        bad = ~OC.same_bytes(h16, want16, allow_negzero=False)
        assert not bad.any(), f"{name}: {bad.sum()} RGBA16F channels differ from the half of the f32 frame, first {np.argwhere(bad)[0]}"
        # alpha: the encoder's f32 steps applied to the f32 frame's alpha (opaque frames: 255)
        want_a = np.full(g8.shape[:2], 255, np.uint8) if mode == "opaque" else OC.pack_srgb8(f8)[..., 3]
        assert np.array_equal(g8[..., 3], want_a), f"{name}: RGBA8 alpha bytes differ"
        # colour: the correctly rounded encoding outside the band; over: the f32 run read the float64 decode of the
        # target, the kernel its own decode, so the band widens by the decode error times the encoder's slope
        extra = 0.0
        if mode == "over":
            extra = OC.srgb_encode_slope(np.maximum(f8[..., :3] - OC.srgb_decode_err(dst8[..., :3]), 0)) * OC.srgb_decode_err(dst8[..., :3])
        band = OC.in_band(f8[..., :3], extra)
        want8 = OC.srgb8_round64(f8[..., :3])
        off = (g8[..., :3] != want8) & ~band
        assert not off.any(), f"{name}: {off.sum()} RGBA8 colour bytes off the correctly rounded encoding, first {np.argwhere(off)[0]}"
        assert np.all(np.abs(g8[..., :3].astype(np.float64) - want8) <= 1)
        BAND_COUNTS[name] = (int(band.sum()), int((g8[..., :3] != want8).sum()), band.size)
        print(f"\n{name}: {band.sum()} of {band.size} colour channels in the band, {(g8[..., :3] != want8).sum()} of them off by one")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("path", OC.PATHS)
def test_pixels_no_splat_blends_keep_their_bytes(oracle, path, fmt):
    """Blend-over onto ramp targets: every pixel the oracle's trace blends no splat into keeps its bytes (empty tiles,
    uncovered pixels of non-empty tiles, raster2_kernel's read-back through decode / encode)."""
    c = OC.case(path)
    u = B.GaussianSplattingPlugin.cloud_uniform(c.settings)
    untouched = oracle.blend_trace(c.cloud, c.view.to_abi(), u, c.settings.to_abi())["n_blended"] == 0
    ramp = OC.ramp_target(fmt, c.view.height, c.view.width)
    p, h = open_case(c)
    try:
        got = run_case(p, h, c, fmt, "over", ramp)
    finally:
        p.destroy()
    for k, g in enumerate(got):
        ok = OC.same_bytes(g, ramp).all(-1)
        bad = untouched & ~ok
        assert not bad.any(), f"{path}/{fmt}/{k}: {bad.sum()} unblended pixels changed, first {np.argwhere(bad)[0]}: {ramp[tuple(np.argwhere(bad)[0])]} -> {g[tuple(np.argwhere(bad)[0])]}"
        assert (~ok & ~untouched).any()                       # (the blended ones did change)


# ---------------------------------------------------------------------------------------------------------------------
# compositing chains

CHAIN_VIEW = (OC.W, OC.H)


def _chain_setup():
    view = B.headless_view(*CHAIN_VIEW)
    s = BC.settings_for("obb3d", saturated=False, binning_rounds=False)
    return view, s, OC.chain_clouds(view)


def _lib_order(p, hs, s, view, fmt, order):
    """The chain into the context's own frame, host copies out -> the frame after each step."""
    outs = [np.empty((view.height, view.width, 4), B.GaussianSplattingPlugin.FORMATS[fmt][1]) for _ in hs]
    decoy = np.empty_like(outs[0])

    def call(j, mode, queued, out):
        p.render_view(hs[j], s, view, fmt=fmt, out=out, asynchronous=queued, premultiplied=mode == "premultiplied",
                      blend_over=mode == "over")

    if order == "sync":
        for j in range(len(hs)):
            call(j, "over", False, outs[j])
    elif order == "queued":
        for j in range(len(hs)):
            call(j, "over", True, outs[j])
    elif order == "sync_then_queued":          # a synchronous frame that does not blend over, then queued blend-over
        call(0, "premultiplied", False, outs[0])
        for j in range(1, len(hs)):
            call(j, "over", True, outs[j])
    elif order == "queued_then_sync":          # two queued frames, then blend-over alternating synchronous / queued
        call(len(hs) - 1, "premultiplied", True, decoy)
        call(0, "premultiplied", True, outs[0])
        for j in range(1, len(hs)):
            call(j, "over", j % 2 == 0, outs[j])
    assert p.sync()
    return outs


def _device_chain(p, hs, s, view, fmt, ptr, read, queued):
    outs = []
    for j in range(len(hs)):
        p.render_view_to_device(hs[j], s, view, ptr, fmt=fmt, asynchronous=queued, blend_over=True)
        if not queued:
            outs.append(read())
    if queued:
        assert p.sync()
        return None
    return outs


@pytest.mark.parametrize("fmt", FMTS)
def test_compositing_chains(oracle, fmt):
    import torch

    view, s, clouds = _chain_setup()
    aabb = False
    u = B.GaussianSplattingPlugin.cloud_uniform(s)
    traces = [oracle.blend_trace(cl, view.to_abi(), u, s.to_abi()) for cl in clouds]
    dcs = []
    for cl in clouds:                                    # the colour records' difference from the oracle's, per cloud
        p = B.GaussianSplattingPlugin(0)
        try:
            h = p.add_cloud(cl)
            p.render_view(h, s, view)
            dcs.append(TB.check_records(p, oracle, cl, s, view, h)[1])
            h.destroy()
        finally:
            p.destroy()
    dtype = B.GaussianSplattingPlugin.FORMATS[fmt][1]
    nbytes = view.height * view.width * 4 * np.dtype(dtype).itemsize
    frames = {}
    for order in ("sync", "queued", "sync_then_queued", "queued_then_sync"):
        p = B.GaussianSplattingPlugin(0)
        try:
            hs = [p.add_cloud(cl) for cl in clouds]
            frames["library/" + order] = _lib_order(p, hs, s, view, fmt, order)
        finally:
            p.destroy()
    cu = _cu()
    for kind in ("torch", "exported", "peer_slot1"):
        for queued in (False, True):
            p = B.GaussianSplattingPlugin(0)
            base, fd, alloc, handle = C.c_void_p(), C.c_int(-1), C.c_size_t(0), (C.c_ubyte * 64)()
            try:
                hs = [p.add_cloud(cl) for cl in clouds]
                if kind == "torch":
                    t = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
                    ptr = t.data_ptr()
                elif kind == "exported":
                    assert p._lib.bgs_frame_export_create(0, nbytes, C.byref(base), C.byref(fd), C.byref(alloc)) == abi.BGS_OK
                    ptr = base.value
                else:                                   # slot 1 of a two-slot frame stack: base + W * H * bpp
                    assert p._lib.bgs_peer_buffer_create(0, 2 * nbytes, C.byref(base), handle) == abi.BGS_OK
                    ptr = base.value + nbytes
                zeros = np.zeros(nbytes, np.uint8)
                assert cu.cuMemcpyHtoD_v2(C.c_uint64(ptr), zeros.ctypes.data_as(C.c_void_p), nbytes) == 0

                def read():
                    got = np.empty(nbytes, np.uint8)
                    torch.cuda.synchronize()
                    assert cu.cuMemcpyDtoH_v2(got.ctypes.data_as(C.c_void_p), C.c_uint64(ptr), nbytes) == 0
                    return got.view(dtype).reshape(view.height, view.width, 4)

                outs = _device_chain(p, hs, s, view, fmt, ptr, read, queued)
                frames[f"{kind}/{'queued' if queued else 'sync'}"] = outs if outs is not None else [None] * 3 + [read()]
            finally:
                if kind == "exported" and base.value:
                    p._lib.bgs_frame_export_destroy(base)
                    os.close(fd.value)
                elif kind == "peer_slot1" and base.value:
                    p._lib.bgs_peer_buffer_release(base, 0)
                p.destroy()
    ref = frames["library/sync"]
    # every step against the float64 blend over the previous GPU frame
    prev = np.zeros_like(ref[0])
    for j, got in enumerate(ref):
        if fmt == "rgba32f":
            TB.assert_within_bound(f"chain/{fmt}/{j}", got, traces[j], aabb, "over", dcs[j], prev)
        else:
            TB.assert_quantised(got, traces[j], aabb, "over", fmt, dcs[j], prev)
        assert j == 0 or np.abs(got.astype(np.float64) - prev.astype(np.float64)).max() > 0     # it blended
        prev = got
    # every order and target kind: the same bytes at every step it exposes
    for name, outs in frames.items():
        for j, (a, b) in enumerate(zip(outs, ref)):
            if a is not None:
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"{fmt}: {name} step {j} differs from library/sync"


# ---------------------------------------------------------------------------------------------------------------------
# regrow

@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("fmt", FMTS)
def test_blend_over_frame_that_regrows_the_pair_buffer(fmt, rounds):
    """The first frame of a fresh context overflows its pair buffer (> initial_pair_capacity(n) pairs) and is rendered
    again after the buffer grows: blended over once, i.e. byte-identical to the frame of a context grown beforehand.
    Queued, the overflowed attempt leaves the target as it was (bgs_sync -> BGS_NOT_READY)."""
    c = OC.regrow_case(rounds)
    view, s = c.view, c.settings
    dst = OC.seeded_target(fmt, view.height, view.width, 23)
    grown = B.GaussianSplattingPlugin(0)
    try:
        h = grown.add_cloud(c.cloud)
        grown.render_view(h, s, view, to_host=False)                       # grows the buffer
        fs = grown.frame_stats()
        assert fs.n_pairs > KP.initial_pair_capacity(len(c.cloud)) and (fs.rounds > 1) == rounds
        # a light frame next, so that its hints keep the frame under test on raster_kernel<0> like a fresh context's
        light = OC.case("r0")
        h_light = grown.add_cloud(light.cloud)
        grown.render_view(h_light, light.settings, light.view, to_host=False)
        fs = grown.frame_stats()
        assert not KP.large_footprint_raster(fs.n_visible, fs.n_pairs)
        t = Target(view, fmt, 0, dst)
        grown._check(render_to(grown, h, s, view, fmt, "over", [t]))
        want = t.read()
        assert (want != dst).any()
    finally:
        grown.destroy()
    for queued in (False, True):
        p = B.GaussianSplattingPlugin(0)
        try:
            h = p.add_cloud(c.cloud)
            t = Target(view, fmt, 0, dst)
            if not queued:
                p._check(render_to(p, h, s, view, fmt, "over", [t]))
            else:
                p._check(render_to(p, h, s, view, fmt, "over", [t], asynchronous=True))
                assert p._lib.bgs_sync(p._ctx) == abi.BGS_NOT_READY
                assert np.array_equal(t.read().view(np.uint8), dst.view(np.uint8)), "the overflowed attempt wrote the target"
                p._check(render_to(p, h, s, view, fmt, "over", [t], asynchronous=True))
                assert p.sync()
            assert (p.frame_stats().rounds > 1) == rounds
            got = t.read()
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), f"{fmt} queued={queued}: {(got != want).sum()} channels differ"
        finally:
            p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# alignment

@pytest.mark.parametrize("mode", ["opaque", "over"])
@pytest.mark.parametrize("path", ["r0", "r2", "rounds", "r0aux", "aabb3d-aux"])
def test_align_rgba8_at_4_bytes(path, mode):
    c = OC.case(path)
    dst = OC.seeded_target("rgba8_srgb", c.view.height, c.view.width, 29) if mode == "over" else None
    p, h = open_case(c)
    try:
        want = run_case(p, h, c, "rgba8_srgb", mode, dst, offset=0)
        got = run_case(p, h, c, "rgba8_srgb", mode, dst, offset=4)
    finally:
        p.destroy()
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_align_rgba8_peer_slot_with_odd_pixel_count():
    """Slot 1 of a frame stack of odd W * H RGBA8 frames starts 4 bytes off an 8-byte boundary; raster2_kernel<false>
    renders straight into it."""
    import torch

    c = OC.case("r2")
    assert (c.view.width * c.view.height) % 2 == 1
    nbytes = c.view.width * c.view.height * 4
    p, h = open_case(c)
    base, handle = C.c_void_p(), (C.c_ubyte * 64)()
    assert p._lib.bgs_peer_buffer_create(0, 2 * nbytes, C.byref(base), handle) == abi.BGS_OK
    try:
        want = p.render_view(h, c.settings, c.view, fmt="rgba8_srgb")
        before = p.frame_stats()
        assert (base.value + nbytes) % 8 == 4
        p.render_view_to_device(h, c.settings, c.view, base.value + nbytes, fmt="rgba8_srgb")
        assert KP.large_footprint_raster(before.n_visible, before.n_pairs) and p.frame_stats().rounds == 1
        torch.cuda.synchronize()
        got = np.empty(2 * nbytes, np.uint8)
        assert _cu().cuMemcpyDtoH_v2(got.ctypes.data_as(C.c_void_p), C.c_uint64(base.value), 2 * nbytes) == 0
        assert np.array_equal(got[nbytes:].reshape(want.shape), want)
        assert not got[:nbytes].any()                                  # slot 0 untouched (the allocation starts cleared)
    finally:
        p._lib.bgs_peer_buffer_release(base, 0)
        p.destroy()


@pytest.mark.parametrize("fmt,offset", [("rgba16f", 4), ("rgba32f", 4), ("rgba32f", 8)])
@pytest.mark.parametrize("path", ["r0", "r0aux"])
def test_align_misaligned_float_targets_are_refused(path, fmt, offset):
    c = OC.case(path)
    dst = OC.seeded_target(fmt, c.view.height, c.view.width, 31)
    p, h = open_case(c)
    try:
        ts = [Target(c.view, fmt, offset if k == 2 or not c.aux else 0, dst) for k in range(3 if c.aux else 1)]
        for mode in ("opaque", "over"):
            assert render_to(p, h, c.settings, c.view, fmt, mode, ts) == abi.BGS_EINVAL
            assert b"aligned" in p._lib.bgs_last_error(p._ctx)
        for t in ts:                                                    # guards and targets untouched
            assert np.array_equal(t.read().view(np.uint8), dst.view(np.uint8))
    finally:
        p.destroy()
