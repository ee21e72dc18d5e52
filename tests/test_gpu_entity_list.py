"""bgs_entity_list on the H100: every list frame is bgs_render_entities_many (_pick_many) of the list as it stands, on
every key test_gpu_entities_many.capture compares, with one more launch (the expansion): every entity_cases case in every
output variant and target, a seeded sequence of 30 edits on a mixed list of 300 entities, transforms set from host arrays
and from torch CUDA tensors in both layouts (identity and -0.0 matrices, entity 0 moved from the device only), queued
frames with edits, transform updates and a particle step between them, a cloud split into 65 536 entities against the
whole, refusals that change nothing, and the detach rule of a destroyed cloud."""
import ctypes as C

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import entities_many_cases as EM
import entity_cases as E
import scene4d_cases as S4
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.particles import random_particle_behaviors
from test_gpu_entities_many import CODES, H, PICK_VARIANTS, SV, VARIANTS, VIEW, W, _depth, _extras, _load, _same, capture

pytestmark = pytest.mark.gpu


def _create(p, ents):
    """A bgs_entity_list on p of EM.Entities' arrays."""
    h = C.c_void_p()
    EM.ok(p, p._lib.bgs_entity_list_create(p._ctx, ents.clouds, ents.unis, ents.ents, ents.flags, ents.k, C.byref(h)))
    return h


def _list_call(p, h, ents, out, code, frame_flags=0, depth=None, ex=None, device=False, pick=None, view=None):
    """bgs_render_entity_list (or _pick with `pick`) of list h on p, with ents' frame settings and view."""
    s = ents.frame(frame_flags)
    v = (view or ents.view).to_abi()
    zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * int(v.viewport[2]))
    args = [p._ctx, h, C.byref(v), C.byref(s), None if ex is None else C.byref(ex), None if zd is None else C.byref(zd),
            EM.addr(out), code, int(device)]
    if pick is None:
        return p._lib.bgs_render_entity_list(*args)
    return p._lib.bgs_render_entity_list_pick(*args, EM.addr(pick))


def _twin(pm, pl, many, listed, make_out, depth_tested, asynchronous=False):
    """many(out) on pm and listed(out) on pl, each into its own make_out() and complete: their captures are equal, and
    the list frame takes one launch more."""
    caps = []
    for p, call in ((pm, many), (pl, listed)):
        out = make_out()
        EM.ok(p, call(out))
        if asynchronous:
            assert p.sync()
        cap = capture(p, out, depth_tested)
        cap["launches"] = p.last_launch_count
        caps.append(cap)
    caps[1]["launches"] -= 1
    _same(caps[1], caps[0])


def _host(dtype):
    return np.full((H, W, 4), 0.25 if dtype != np.uint8 else 64, dtype)


# ---- 1. every entity_cases case, in every output variant and target, as a list

@pytest.mark.parametrize("case", list(E.CASES))
def test_cases_as_lists(case):
    pm, pl = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(0)
    h = None
    try:
        ents, _ = _load(pm, E.entities(case), flags=[j & 1 for j in range(6)])
        h = _create(pl, ents)
        for i, (dtype, flags, with_depth) in enumerate(VARIANTS):
            depth = _depth(i) if with_depth else None
            code = CODES[np.dtype(dtype)]
            _twin(pm, pl, lambda o: ents.call("many", o, code, flags, depth, _extras()),
                  lambda o: _list_call(pl, h, ents, o, code, flags, depth, _extras()), lambda: _host(dtype), depth is not None,
                  bool(flags & abi.BGS_FLAG_ASYNC))
        for i, (dtype, flags, with_depth, device) in enumerate(PICK_VARIANTS):
            depth = _depth(10 + i) if with_depth else None
            code = CODES[np.dtype(dtype)]
            got = []
            for p, call in ((pm, lambda o, pk: ents.call("pick_many", o, code, flags, depth, _extras(), device=device, pick=pk)),
                            (pl, lambda o, pk: _list_call(pl, h, ents, o, code, flags, depth, _extras(), device=device, pick=pk))):
                if device:
                    tdt = {np.dtype(np.uint8): torch.uint8, np.dtype(np.float16): torch.float16}.get(np.dtype(dtype), torch.float32)
                    out = torch.zeros((H, W, 4), dtype=tdt, device="cuda")
                    pick = torch.zeros((H, W, 4), dtype=torch.int32, device="cuda")
                else:
                    out, pick = _host(dtype), np.zeros((H, W), abi.PICK_DTYPE)
                EM.ok(p, call(out, pick))
                cap = capture(p, out, True)
                torch.cuda.synchronize()
                cap["pick"] = pick.tobytes() if isinstance(pick, np.ndarray) else pick.cpu().numpy().tobytes()
                cap["launches"] = p.last_launch_count
                got.append(cap)
            got[1]["launches"] -= 1
            _same(got[1], got[0])
    finally:
        if h is not None:
            pl._lib.bgs_entity_list_destroy(h)
        pl.destroy()
        pm.destroy()


# ---- 2. a seeded sequence of 30 edits on a mixed list of 300 entities

def _subset_arrays(p, handles, unis, sts, flags):
    k = len(handles)
    return ((C.c_void_p * k)(*[x._h.value for x in handles]), (abi.bgs_cloud_uniform * k)(*unis),
            (abi.bgs_entity_settings * k)(*[B.plugin.entity_settings(st) for st in sts]), (C.c_uint32 * k)(*flags))


def test_edit_sequence():
    rng = np.random.default_rng(7)
    pm, pl = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(0)
    h = None
    try:
        # the pool: every case's six entities (their clouds uploaded once), by case name
        pool = {}
        for case in E.CASES:
            pool[case], up = [], {}   # (per case: the ids of an earlier case's collected clouds may be reused)
            for cloud, layout, tr, st in E.entities(case, n4=2000):
                if id(cloud) not in up:
                    up[id(cloud)] = pm.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
                pool[case].append((up[id(cloud)], st))
        cases = list(E.CASES)
        # (slot i of every case is a copy of the same cloud, so its gaussian count is the same)
        slots = {hw.serial: i for case in cases for i, (hw, _) in enumerate(pool[case])}

        def draw(case=None, slot=None):
            c = case or cases[rng.integers(len(cases))]
            hw, st = pool[c][slot if slot is not None else rng.integers(6)]
            tr = SC.transform(tuple(rng.uniform(-1.2, 1.2, 3) * (1.0, 0.5, 0.8)), float(rng.uniform(0.5, 1.2)),
                              float(rng.uniform(0, 6.28)))
            return hw, pm.cloud_uniform(st, tr, hw.aabb), st, int(rng.integers(4) == 0)

        state = [draw() for _ in range(300)]
        mirror = EM.Entities(pm, *zip(*[s[:3] for s in state]), VIEW, [s[3] for s in state])
        h = _create(pl, mirror)
        lib = pl._lib
        for step in range(30):
            kind = ("set", "set_counts", "uniform", "append", "truncate", "depth")[step % 6]
            k = len(state)
            if kind in ("set", "set_counts", "depth"):
                idx = sorted(rng.choice(k, size=int(rng.integers(1, 12)), replace=False).tolist())
                # (set: each entity keeps its cloud, so no gaussian count changes; set_counts and depth: any cloud)
                new = [draw(case="agree_aabb" if kind == "depth" else None, slot=slots[state[j][0].serial] if kind == "set" else None)
                       for j in idx]
            elif kind == "uniform":   # every entity one blend kind (quad-uv, no overlay), or back to a mixed list
                idx = list(range(k))
                new = [(*draw(case="agree")[:3], 0) for _ in idx] if step % 12 == 2 else [draw() for _ in idx]
            if kind in ("set", "set_counts", "depth", "uniform"):
                arrays = _subset_arrays(pm, *zip(*[n_[:3] for n_ in new]), [n_[3] for n_ in new])
                EM.ok(pl, lib.bgs_entity_list_set(h, (C.c_uint32 * len(idx))(*idx), len(idx), *arrays))
                for j, n_ in zip(idx, new):
                    state[j] = n_
            elif kind == "append":
                new = [draw() for _ in range(int(rng.integers(1, 40)))]
                arrays = _subset_arrays(pm, *zip(*[n_[:3] for n_ in new]), [n_[3] for n_ in new])
                EM.ok(pl, lib.bgs_entity_list_append(h, len(new), *arrays))
                state += new
            else:
                k2 = int(rng.integers(200, k))
                EM.ok(pl, lib.bgs_entity_list_truncate(h, k2))
                del state[k2:]
            assert lib.bgs_entity_list_size(h) == len(state)
            mirror = EM.Entities(pm, *zip(*[s[:3] for s in state]), VIEW, [s[3] for s in state])
            depth = _depth(50 + step) if step % 3 == 0 else None
            flags = (0, abi.BGS_FLAG_NO_CHUNKS, abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX)[(step // 3) % 3]
            _twin(pm, pl, lambda o: mirror.call("many", o, abi.BGS_FORMAT_RGBA32F, flags, depth, _extras()),
                  lambda o: _list_call(pl, h, mirror, o, abi.BGS_FORMAT_RGBA32F, flags, depth, _extras()),
                  lambda: _host(np.float32), depth is not None)
    finally:
        if h is not None:
            pl._lib.bgs_entity_list_destroy(h)
        pl.destroy()
        pm.destroy()


# ---- 3. transforms from host arrays and from torch CUDA tensors, in both layouts

def _instances(k, seed=3):
    rng = np.random.default_rng(seed)
    return [SC.transform((float(x), float(y), -2.0 + float(z)), float(s), float(a))
            for x, y, z, s, a in zip(rng.uniform(-1.8, 1.8, k), rng.uniform(0.8, 2.2, k), rng.uniform(-0.5, 0.5, k),
                                     rng.uniform(0.6, 1.3, k), rng.uniform(0, 6.28, k))]


def _compare(p, lst, entities, **kw):
    want_img = p.render_entities_many(entities, VIEW, **kw)
    want = capture(p, want_img, False)
    launches = p.last_launch_count
    got = capture(p, p.render_entity_list(lst, VIEW, **kw), False)
    _same(got, want)
    assert p.last_launch_count == launches + 1


def test_set_transforms():
    p = B.GaussianSplattingPlugin(0)
    try:
        hw = p.add_cloud(SC.cloud_in_box(600, 4, centre=(0.0, 0.0, 0.0), half=0.15, scale=0.05, sh_degree=1))
        h4 = p.add_cloud(S4.performer(800, 9))
        st = B.CloudSettings(aabb=True)
        k = 240
        entities = [(hw, st if j % 3 else B.CloudSettings(), tr) for j, tr in enumerate(_instances(k))]
        entities[5] = (h4, S4.settings_4d(B.CloudSettings(), 0.4, -0.2, 1.1), entities[5][2])
        lst = p.entity_list(entities)
        _compare(p, lst, entities)

        def apply(first, mats):   # the transforms as the uniforms take them: CloudTransform(M) for row-major M
            for i, m in enumerate(mats):
                h_, s_, _ = entities[first + i]
                entities[first + i] = (h_, s_, B.CloudTransform(np.asarray(m, np.float32)))

        keep = []   # (device arrays stay allocated until the context's stream has read them)
        host = np.stack([t.matrix for t in _instances(40, 5)])
        lst.set_transforms(20, host)
        apply(20, host)
        _compare(p, lst, entities)
        # row-major torch tensor written on a side stream
        side = torch.cuda.Stream()
        rows = np.stack([t.matrix for t in _instances(50, 6)])
        with torch.cuda.stream(side):
            # (the producer is held back on its stream: read unordered, the list would take the matrices unwritten)
            keep.append(torch.zeros((50, 4, 4), device="cuda"))
            torch.cuda._sleep(50_000_000)
            keep[-1].copy_(torch.tensor(rows, device="cuda"))
            lst.set_transforms(100, keep[-1])
        apply(100, rows)
        _compare(p, lst, entities)
        # column-major: the .mT of a contiguous tensor (each matrix transposed in memory)
        base = np.stack([t.matrix for t in _instances(30, 7)])
        with torch.cuda.stream(side):
            keep.append(torch.zeros((30, 4, 4), device="cuda"))
            torch.cuda._sleep(50_000_000)
            keep[-1].copy_(torch.tensor(base.transpose(0, 2, 1).copy(), device="cuda"))
            lst.set_transforms(150, keep[-1].mT)
        apply(150, base)
        _compare(p, lst, entities)
        # identity from the device (model_identity's fast path) and -0.0 entries (the general path)
        keep.append(torch.eye(4, device="cuda").repeat(3, 1, 1))
        lst.set_transforms(60, keep[-1])
        apply(60, [np.eye(4)] * 3)
        neg = np.eye(4, dtype=np.float32)
        neg[0, 1] = neg[2, 3] = -0.0
        keep.append(torch.tensor(np.stack([neg] * 2), device="cuda"))
        lst.set_transforms(63, keep[-1])
        apply(63, [neg] * 2)
        _compare(p, lst, entities)
        # entity 0 moved from the device only: the host's copy of its uniform is stale
        m0 = _instances(1, 8)[0].matrix
        keep.append(torch.tensor(m0[None], device="cuda"))
        lst.set_transforms(0, keep[-1])
        apply(0, [m0])
        _compare(p, lst, entities)
        _compare(p, lst, entities, fmt="rgba8_srgb", premultiplied=True)
        lst.close()
    finally:
        p.destroy()


# ---- 4. ordering with queued frames

def test_queued_frames_with_device_transform_updates():
    """Three queued frames of a 1000-instance list into their own device targets, the transforms rewritten on the device
    between each pair: each frame is _many of its own transforms."""
    p = B.GaussianSplattingPlugin(0)
    try:
        k = 1000
        hw = p.add_cloud(SC.cloud_in_box(300, 5, centre=(0.0, 0.0, 0.0), half=0.1, scale=0.05, sh_degree=0))
        st = B.CloudSettings()
        sets = [np.stack([t.matrix for t in _instances(k, 20 + i)]) for i in range(3)]
        entities = [(hw, st, B.CloudTransform(m)) for m in sets[0]]
        lst = p.entity_list(entities)
        ents = EM.Entities(p, [hw] * k, [p.cloud_uniform(st, B.CloudTransform(m), hw.aabb) for m in sets[0]], [st] * k, SV)
        targets = [torch.zeros((SV.height, SV.width, 4), dtype=torch.float32, device="cuda") for _ in range(3)]
        keep = [torch.tensor(m, device="cuda") + 0.0 for m in sets]
        for i in range(3):
            if i:
                lst.set_transforms(0, keep[i])
            EM.ok(p, _list_call(p, lst._h, ents, targets[i], abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC | abi.BGS_FLAG_NO_CHUNKS,
                                device=True))
        assert p.sync()
        for i in range(3):
            want = EM.Entities(p, [hw] * k, [p.cloud_uniform(st, B.CloudTransform(m), hw.aabb) for m in sets[i]], [st] * k, SV)
            out = torch.zeros_like(targets[0])
            EM.ok(p, want.call("many", out, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_NO_CHUNKS, device=True))
            torch.cuda.synchronize()
            assert out.cpu().numpy().tobytes() == targets[i].cpu().numpy().tobytes(), i
        lst.close()
    finally:
        p.destroy()


def test_edit_and_particle_step_between_queued_frames():
    p = B.GaussianSplattingPlugin(0)
    try:
        n, k = 400, 1000
        hw = p.add_cloud(SC.cloud_in_box(n, 5, centre=(0.0, 0.0, 0.0), half=0.1, scale=0.05, sh_degree=0))
        other = p.add_cloud(SC.cloud_in_box(700, 6, centre=(0.0, 0.0, 0.0), half=0.2, scale=0.04, sh_degree=2))
        st = B.CloudSettings()
        trs = [SC.transform(((j % 40) * 0.09 - 1.8, 1.5 + (j // 40) * 0.06 - 0.75, -2.0), 1.0, 0.01 * j) for j in range(k)]
        entities = [(hw, st, tr) for tr in trs]
        lst = p.entity_list(entities)
        behaviors = p.add_particles(random_particle_behaviors(n, 3))
        ents = EM.Entities(p, [hw] * k, [p.cloud_uniform(st, tr, hw.aabb) for tr in trs], [st] * k, SV)

        def many(es):
            img = np.zeros((SV.height, SV.width, 4), np.float32)
            EM.ok(p, EM.Entities(p, [e[0] for e in es], [p.cloud_uniform(e[1], e[2], e[0].aabb) for e in es],
                                 [e[1] for e in es], SV).call("many", img, abi.BGS_FORMAT_RGBA32F))
            return img

        edited = list(entities)
        edited[7], edited[500] = (other, st, trs[7]), (other, st, trs[500])
        before, unstepped = many(entities), many(edited)
        q = [np.zeros((SV.height, SV.width, 4), np.float32) for _ in range(3)]
        EM.ok(p, _list_call(p, lst._h, ents, q[0], abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        lst.set([7, 500], [edited[7], edited[500]])   # an edit between two queued frames
        EM.ok(p, _list_call(p, lst._h, ents, q[1], abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        p.step_particles(hw, behaviors, 0.25)         # a particle step between two queued frames
        EM.ok(p, _list_call(p, lst._h, ents, q[2], abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        assert p.sync()
        stepped = many(edited)
        assert q[0].tobytes() == before.tobytes()
        assert q[1].tobytes() == unstepped.tobytes()
        assert q[2].tobytes() == stepped.tobytes()
        assert len({before.tobytes(), unstepped.tobytes(), stepped.tobytes()}) == 3
        lst.close()
    finally:
        p.destroy()


# ---- 5. a cloud split into 65 536 subsets as a list is the whole

def test_split_65536_equals_the_whole():
    k = 65536
    n = max(40 * k, 3 * 8 * EM.KG_TILE + 33 * k)
    st = B.CloudSettings()
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = SC.cloud_in_box(n, 66, half=1.6, scale=0.03, sh_degree=0)
        hw = p.add_cloud(cloud)
        u = p.cloud_uniform(st, SC.transform((0.1, 0.0, 0.2), 1.05, 0.3), hw.aabb)
        depth = _depth(26, SV.width, SV.height)
        want_img = np.zeros((SV.height, SV.width, 4), np.float32)
        s = st.to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        zd = abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * SV.width)
        EM.ok(p, p._lib.bgs_render_depth_test(p._ctx, hw._h, C.byref(SV.to_abi()), C.byref(u), C.byref(s), None, C.byref(zd),
                                              want_img.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0))
        want = capture(p, want_img, True)
        parts = [p.subset(hw, ix) for ix in EM.pieces(n, k, 6)]
        ents = EM.Entities(p, parts, [u] * k, [st] * k, SV)
        h = _create(p, ents)
        img = np.zeros((SV.height, SV.width, 4), np.float32)
        EM.ok(p, _list_call(p, h, ents, img, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_NO_CHUNKS, depth))
        _same(capture(p, img, True), want)
        p._lib.bgs_entity_list_destroy(h)
    finally:
        p.destroy()


# ---- 6. refusals change nothing; 7. lifetime

def test_refusals_change_nothing_and_destroyed_clouds_detach():
    p = B.GaussianSplattingPlugin(0)
    lib = p._lib
    try:
        hw = p.add_cloud(SC.cloud_in_box(3000, 9, half=1.6, scale=0.03, sh_degree=0))
        small = p.add_cloud(SC.cloud_in_box(50, 10, sh_degree=0))
        st = B.CloudSettings()
        k = 300
        trs = _instances(k, 30)
        entities = [(hw if j % 7 else small, st, tr) for j, tr in enumerate(trs)]
        lst = p.entity_list(entities)
        h = lst._h
        ents = EM.Entities(p, [e[0] for e in entities], [p.cloud_uniform(st, tr, e[0].aabb) for e, tr in zip(entities, trs)],
                           [st] * k, SV)
        img = np.zeros((SV.height, SV.width, 4), np.float32)
        EM.ok(p, _list_call(p, h, ents, img, abi.BGS_FORMAT_RGBA32F))
        hooks = capture(p, img, False)

        def unchanged():
            assert lib.bgs_entity_list_size(h) == k
            again = np.zeros_like(img)
            EM.ok(p, ents.call("many", again, abi.BGS_FORMAT_RGBA32F))
            want = capture(p, again, False)
            EM.ok(p, _list_call(p, h, ents, again, abi.BGS_FORMAT_RGBA32F))
            _same(capture(p, again, False), want)

        bad = B.CloudSettings(rasterize_mode=B.RasterizeMode.Classification, num_classes=0)
        one = lambda s_, c_=hw: _subset_arrays(p, [c_], [p.cloud_uniform(s_, None, c_.aabb)], [s_], [0])   # noqa: E731
        refusals = [
            lambda: lib.bgs_entity_list_set(h, (C.c_uint32 * 1)(3), 1, *one(bad)),
            lambda: lib.bgs_entity_list_set(h, (C.c_uint32 * 1)(k), 1, *one(st)),
            lambda: lib.bgs_entity_list_set(h, (C.c_uint32 * 2)(4, 4), 2, *_subset_arrays(p, [hw, hw], [ents.unis[0]] * 2, [st] * 2, [0, 0])),
            lambda: lib.bgs_entity_list_set(h, (C.c_uint32 * 1)(3), 1, *_subset_arrays(p, [hw], [ents.unis[0]], [st], [8])),
            lambda: lib.bgs_entity_list_append(h, 1, *one(bad)),
            lambda: lib.bgs_entity_list_append(h, abi.BGS_ENTITIES_MANY_MAX, None, None, None, None),
            lambda: lib.bgs_entity_list_truncate(h, k + 1),
            lambda: lib.bgs_entity_list_set_transforms(h, k - 1, 2, np.eye(4, dtype=np.float32).ctypes.data, 0, 0),
            lambda: lib.bgs_entity_list_set_transforms(h, 0, 1, None, 0, 0),
            lambda: lib.bgs_entity_list_set_transforms(h, 0, 1, np.eye(4, dtype=np.float32).ctypes.data, 2, 0),
            lambda: lib.bgs_entity_list_set_transforms(h, 0, 1, np.eye(4, dtype=np.float32).ctypes.data, 0, 1),
            lambda: _list_call(p, h, ents, img, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_SORT_ALL),
            lambda: _list_call(p, h, ents, img, 7),
        ]
        for i, call in enumerate(refusals):
            assert call() == abi.BGS_EINVAL, (i, EM.error(p))
            _same(capture(p, img, False), hooks)
        refusals[0]()
        assert "entities[3]" in EM.error(p)
        unchanged()
        c = B.CloudSettings(rasterize_mode=B.RasterizeMode.Classification, num_classes=3)
        c_bad = lib.bgs_entity_list_create(p._ctx, *one(bad), 1, C.byref(C.c_void_p()))
        assert c_bad == abi.BGS_EINVAL and "entities[0]" in EM.error(p)
        flow = B.CloudSettings(rasterize_mode=B.RasterizeMode.OpticalFlow)
        lst2 = p.entity_list([(hw, flow, None), (hw, c, None)])
        e2 = EM.Entities(p, [hw, hw], [p.cloud_uniform(flow, None, hw.aabb), p.cloud_uniform(c, None, hw.aabb)], [flow, c], SV)
        assert e2.call("many", img, abi.BGS_FORMAT_RGBA32F) == _list_call(p, lst2._h, e2, img, abi.BGS_FORMAT_RGBA32F) == abi.BGS_EINVAL
        lst2.truncate(0)
        assert _list_call(p, lst2._h, e2, img, abi.BGS_FORMAT_RGBA32F) == abi.BGS_EINVAL
        lst2.close()
        # lifetime: a destroyed listed cloud detaches its entities until set replaces them
        gone = p.add_cloud(SC.cloud_in_box(80, 12, sh_degree=0))
        lst.set([5], [(gone, st, trs[5])])
        gone.destroy()
        assert _list_call(p, h, ents, img, abi.BGS_FORMAT_RGBA32F) == abi.BGS_EINVAL
        assert "entities[5]" in EM.error(p)
        lst.set([5], [entities[5]])
        unchanged()
        # destroying a list with a queued frame drains it
        q = np.zeros_like(img)
        EM.ok(p, _list_call(p, h, ents, q, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        lst.close()
        assert C.CDLL("libcuda.so.1").cuStreamQuery(C.c_void_p(p.stream_ptr)) == 0   # (drained by the destroy itself)
        p.sync()
        want = np.zeros_like(img)
        EM.ok(p, ents.call("many", want, abi.BGS_FORMAT_RGBA32F))
        assert q.tobytes() == want.tobytes()
    finally:
        p.destroy()


# ---- 8. the C++ host

def test_cpp_host_instances_match_python(tmp_path):
    """examples/headless.cpp --instances (include/bgs.hpp's EntityList: one cloud instanced on a grid, then moved by one
    row-major set_transforms) gives the Python host's frame of the same list, which is render_entities_many's."""
    import os
    import subprocess

    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    exe = os.path.join(root, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(root, "examples")], check=True)
    n, w, h, scale, k = 3000, 320, 200, 0.3, 2500
    raw, cloud_f = tmp_path / "f.raw", tmp_path / "cloud.bin"
    run = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--raw", str(raw), "--instances", str(k),
                          "--dump-cloud", str(cloud_f)], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    assert f"instances: {k}" in run.stdout and "rendered=1" in run.stdout
    got = np.fromfile(raw, np.uint8)
    g = np.fromfile(cloud_f, np.uint8)[8:].view(np.float32)
    p = B.GaussianSplattingPlugin(0)
    try:
        hd = p.add_cloud(B.PlanarGaussian3d(g[: n * 4].reshape(n, 4), g[n * 4: n * 52].reshape(n, 48),
                                            g[n * 52: n * 56].reshape(n, 4), g[n * 56: n * 60].reshape(n, 4)))
        view, st = B.headless_view(w, h), B.CloudSettings(global_scale=scale)
        j = np.arange(k)
        t = np.stack([(j % 32) * 0.25 - 4.0, 1.5 + (j // 32 % 32) * 0.125 - 2.0, -2.0 - (j // 1024) * 0.5], 1).astype(np.float32)
        mats = np.tile(np.eye(4, dtype=np.float32), (k, 1, 1))
        mats[:, :3, 3] = t
        lst = p.entity_list([(hd, st, B.CloudTransform(m)) for m in mats])
        mats[:, 0, 3] += np.float32(0.5)
        lst.set_transforms(0, mats)
        for _ in range(3):   # (the C++ host renders three frames: the same hints)
            img = p.render_entity_list(lst, view, fmt="rgba8_srgb")
        assert got.tobytes() == img.tobytes()
        assert img.any()
        want = None
        for _ in range(3):
            want = p.render_entities_many([(hd, st, B.CloudTransform(m)) for m in mats], view, fmt="rgba8_srgb")
        assert want.tobytes() == img.tobytes()
        lst.close()
    finally:
        p.destroy()
