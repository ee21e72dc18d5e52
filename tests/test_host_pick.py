"""bgs_render_entities_pick and bgs_cloud_select_in_view without a GPU: the ctypes prototypes against the header, the pick
record's layout, the C calls' refusals of a NULL context, the plugin's ValueErrors before any call, and pick_oracle on
hand-built records."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import GaussianSplattingPlugin
from pick_oracle import pick_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _params(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bgs.h")).read(), flags=re.S)
    return [p.strip() for p in re.search(rf"bgs_status {name}\((.*?)\);", src, flags=re.S).group(1).split(",")]


def test_prototypes_match_the_header():
    (pick,) = [a for n, _, a in abi.SYMBOLS if n == "bgs_render_entities_pick"]
    params = _params("bgs_render_entities_pick")
    assert len(pick) == len(params) == 14 and params[-1] == "void* out_pick"
    (sel,) = [a for n, _, a in abi.SYMBOLS if n == "bgs_cloud_select_in_view"]
    params = _params("bgs_cloud_select_in_view")
    assert len(sel) == len(params) == 8
    assert params[4:7] == ["const uint8_t* mask", "int mask_is_device_ptr", "uint32_t mode"]
    assert sel[5] is C.c_int and sel[6] is C.c_uint32


def test_pick_record_layout():
    assert C.sizeof(abi.bgs_pick) == 16 == abi.PICK_DTYPE.itemsize
    assert B.PICK_DTYPE is abi.PICK_DTYPE
    assert [abi.PICK_DTYPE.fields[f][1] for f in ("entity", "index", "weight", "depth")] == [0, 4, 8, 12]
    assert abi.BGS_PICK_NONE == 0xFFFFFFFF
    assert "#define BGS_PICK_NONE 0xFFFFFFFFu" in open(os.path.join(ROOT, "include", "bgs.h")).read()


def test_null_context():
    lib = abi.load()
    assert lib.bgs_render_entities_pick(None, None, None, None, None, 0, None, None, None, None, None, 0, 0, None) == abi.BGS_EINVAL
    assert lib.bgs_cloud_select_in_view(None, None, None, None, None, 0, 0, None) == abi.BGS_EINVAL


class _Handle:
    temporal = False
    precompute_covariance = False
    n = 4


def test_plugin_validation_raises_before_any_call():
    p = GaussianSplattingPlugin.__new__(GaussianSplattingPlugin)   # (no context: any C call would fail)
    view = B.headless_view(8, 4)
    with pytest.raises(ValueError, match="no entities"):
        p.render_entities_pick([], view)
    ok = [(_Handle(), B.CloudSettings(), None)]
    bad = ok + [(_Handle(), B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits.Bits16), None)]
    with pytest.raises(ValueError, match="depth sort"):
        p.render_entities_pick(bad, view)
    with pytest.raises(ValueError, match="mode"):
        p.select_in_view(_Handle(), view, np.ones((4, 8), bool), mode="xor")
    with pytest.raises(ValueError, match="shape"):
        p.select_in_view(_Handle(), view, np.ones((8, 4), bool))
    with pytest.raises(TypeError, match="bool or uint8"):
        p.select_in_view(_Handle(), view, np.ones((4, 8), np.float32))
    pick = np.zeros((4, 8), abi.PICK_DTYPE)
    with pytest.raises(ValueError, match="mode"):
        p.select_picked(ok, pick, mode="xor")
    with pytest.raises(ValueError, match="PICK_DTYPE"):
        p.select_picked(ok, np.zeros((4, 8), np.float32))
    with pytest.raises(ValueError, match="shape"):
        p.select_picked(ok, pick, mask=np.ones((8, 4), bool))
    pick["entity"] = 3
    with pytest.raises(ValueError, match="entity 3"):
        p.select_picked(ok, pick)


def _rec(cx, cy, half, op, conic=False, colour=(0.5, 0.5, 0.5)):
    """One record: an axis-aligned quad-uv square of half-side `half` px (u = dx / half), or a conic of quad half-side
    2 half in half-pixels with a tiny conic (power ~ 0 inside), bbox the covered pixels."""
    lo_x, hi_x = int(np.floor(cx - half)), int(np.ceil(cx + half))
    lo_y, hi_y = int(np.floor(cy - half)), int(np.ceil(cy + half))
    bx, by = lo_x | hi_x << 16, lo_y | hi_y << 16
    q = [cx, cy, 1e-6, 0.0, 1e-6, 2.0 * half] if conic else [cx, cy, 1.0 / half, 0.0, 0.0, 1.0 / half]
    words = struct.pack("<6f2I4f", *q, bx, by, *colour, op)
    return np.frombuffer(words, np.float32)


def _frame(recs, W=16, H=16, order=None):
    n = len(recs)
    order = list(range(n)) if order is None else order
    return dict(n_vis=n, records=np.stack(recs), tile_ranges=np.array([[0, n]], np.uint32),
                tile_entries=np.array(order, np.uint32), depths=np.linspace(0.5, 0.1, n).astype(np.float32))


def test_pick_oracle_picks_the_hand_computed_pair():
    # rank 0: faint and wide; rank 1: strong, small, centred at (8, 8); rank 2: a conic behind both
    recs = [_rec(8.0, 8.0, 6.0, 0.2), _rec(8.0, 8.0, 2.0, 0.9), _rec(8.0, 8.0, 7.0, 0.9, conic=True)]
    pr = PO.pairs(_frame(recs), np.array([0, 0, 1], np.uint8), 16, 16, BC.alpha_error_coefs(False))
    off = pr["offsets"]
    pix = 8 * 16 + 8                       # centre (8.5, 8.5): inside all three
    a, b = int(off[pix]), int(off[pix + 1])
    assert pr["rank"][a:b].tolist() == [0, 1, 2]
    a0 = 0.2 * np.exp(-4.5 * ((0.5 / 6) ** 2 * 2))
    a1 = min(0.9 * np.exp(-4.5 * ((0.5 / 2) ** 2 * 2)), 0.999)
    w = [a0, a1 * (1 - a0)]
    assert np.allclose(pr["w"][a:a + 2], w, rtol=1e-6)
    assert int(np.argmax(pr["w"][a:b])) == 1
    assert (pr["bound"][a:b] > 0).all() and (pr["bound"][a:b] < 1e-5).all()
    # a corner pixel only the wide quad and the conic cover
    pix = 3 * 16 + 3
    a, b = int(off[pix]), int(off[pix + 1])
    assert pr["rank"][a:b].tolist() == [0, 2]
    # a scene depth between ranks: d = 0.5, 0.3, 0.1 -> only d >= 0.35 blends
    pr = PO.pairs(_frame(recs), np.array([0, 0, 1], np.uint8), 16, 16, BC.alpha_error_coefs(False),
                  scene=np.full((16, 16), 0.35, np.float32))
    pix = 8 * 16 + 8
    assert pr["rank"][int(pr["offsets"][pix]):int(pr["offsets"][pix + 1])].tolist() == [0]
    # the overlay: rank 1 with its boxes; a pixel on its edge band takes w = T and stops the walk
    pr = PO.pairs(_frame(recs), np.array([0, 4, 1], np.uint8), 16, 16, BC.alpha_error_coefs(False))
    pix = 6 * 16 + 6                       # (6.5, 6.5): u = v = -0.75 -> s = 0.125, inside the quad, not an edge
    a, b = int(pr["offsets"][pix]), int(pr["offsets"][pix + 1])
    assert pr["rank"][a:b].tolist() == [0, 1, 2]
    recs[1] = _rec(8.0, 8.0, 1.6, 0.9)
    pr = PO.pairs(_frame(recs), np.array([0, 4, 1], np.uint8), 16, 16, BC.alpha_error_coefs(False))
    pix = 6 * 16 + 6                       # u = v = -1.5 / 1.6: s = 0.03 -> an edge pair, w = T, nothing after it
    a, b = int(pr["offsets"][pix]), int(pr["offsets"][pix + 1])
    assert pr["rank"][a:b].tolist() == [0, 1]
    assert pr["w"][a + 1] == pytest.approx(1.0 - pr["w"][a])
    # saturated pixel: a ~ 0.938 each, so T = 1.4e-5 < 1e-4 after the fourth pair and the walk stops there
    many = [_rec(8.0, 8.0, 6.0, 1.0) for _ in range(6)]
    pr = PO.pairs(_frame(many), np.zeros(6, np.uint8), 16, 16, BC.alpha_error_coefs(False))
    pix = 8 * 16 + 8
    assert int(pr["offsets"][pix + 1] - pr["offsets"][pix]) == 4
    # a surfel rank needs the frame's surfel extras
    with pytest.raises(ValueError):
        PO.pairs(_frame(recs), np.array([0, 0, 2], np.uint8), 16, 16, BC.alpha_error_coefs(False))
