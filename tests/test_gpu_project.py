"""The projection (project.cu) and key-gen (keygen.cu over project_math.cuh) on the constructions of
`project_cases.py`, against the oracle: sorted keys and permutation bit-exact, n_visible equal, every record's drawn /
undrawn decision equal, drawn geometry and bboxes bit-exact (sign of zero counted, NaN compared as a class), colours
within the per-record bound `project_cases.colour_bound`, Depth colours from the literal sorted[1] / sorted[N-1] range."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import project_cases as PC

pytestmark = pytest.mark.gpu

f32 = np.float32
# (sort_all, key bits, queued).  Every case except the one-hot SH ones runs under all six; the SH cases (which are
# about the colour path, the same in every variant) take one each, cycled.
VARIANTS = [(False, 32, False), (True, 32, True), (False, 24, True), (True, 16, False), (False, 16, True), (True, 24, False)]


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


@pytest.fixture(scope="module")
def cases(oracle):
    return {c.name: c for c in PC.all_cases(oracle)}


WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst_colour_ratio():
    """After the module: the largest colour err / bound per variant (shown with -s)."""
    yield
    for k in sorted(WORST):
        print(f"COLOUR_ERR_BOUND {k}: {WORST[k]:.3f}")


def _params():
    out = []
    for i, (name, geoms) in enumerate(PC.case_index()):
        for j, g in enumerate(geoms):
            vs = [(i + j) % len(VARIANTS)] if name.startswith("sh_") else range(len(VARIANTS))
            out += [(name, g, v) for v in vs]
    return out


PARAMS = _params()


def render(plugin, case, s, queued):
    h = plugin.add_cloud(case.cloud, f16=case.layout == "f16", precompute_covariance=case.layout == "cov")
    try:
        if not queued:
            plugin.render_view(h, s, case.view, transform=case.transform, fmt="rgba32f")
        else:
            out = np.empty((case.view.height, case.view.width, 4), np.float32)
            for _ in range(3):
                plugin.render_view(h, s, case.view, transform=case.transform, fmt="rgba32f", out=out, asynchronous=True)
                if plugin.sync():
                    break
            else:
                raise AssertionError("a queued frame kept outgrowing the pair buffer")
        return h
    except BaseException:
        h.destroy()
        raise


def depth_colours(case, u, keys_order, ids):
    """numpy f32 restatement of depth_range + material/depth.wgsl:3-11 (sorted[1] and sorted[N-1] of the full order)."""
    p = case.oracle_cloud().position_visibility[:, :3].astype(f32)
    m = np.asarray(u.transform, f32).reshape(4, 4).T                      # row-major
    cam = np.asarray(case.view.world_position, f32)

    def dist(i):
        pw = [((m[r, 0] * p[i, 0] + m[r, 1] * p[i, 1]) + m[r, 2] * p[i, 2]) + m[r, 3] for r in range(3)]
        d = [f32(pw[r] - cam[r]) for r in range(3)]
        return np.sqrt(f32((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))

    n = len(p)
    dmin, dmax = dist(keys_order[n - 1]), dist(keys_order[1])
    out = []
    for i in ids:
        nd = f32(f32(dist(i) - dmin) / f32(dmax - dmin))
        nd = f32(min(max(nd, f32(0)), f32(1))) if nd == nd else f32(0)

        def smooth(e0, e1, x):
            t = f32(f32(x - f32(e0)) / f32(f32(e1) - f32(e0)))
            t = f32(min(max(t, f32(0)), f32(1)))
            return f32(f32(t * t) * f32(f32(3) - f32(2) * t))

        out.append((smooth(0.5, 1.0, nd), f32(1) - f32(abs(f32(nd - f32(0.5))) * f32(2)), f32(1) - smooth(0.0, 0.5, nd)))
    return np.array(out, f32).reshape(-1, 3), float(dmin), float(dmax)


def check_case(plugin, oracle, case, geom, variant, **kw):
    sort_all, bits, queued = VARIANTS[variant]
    s = PC.settings(geom, sort_all=sort_all, radix_sort_depth_bits=B.RadixSortDepthBits(bits), **{**case.settings, **kw})
    oc = case.oracle_cloud()
    s_abi = s.to_abi()
    s_abi.reserved = 1 if case.layout == "cov" else 0
    h = render(plugin, case, s, queued)
    try:
        u = plugin.cloud_uniform(s, case.transform, h.aabb)
        keys = oracle.keygen(oc.position_visibility, case.view.to_abi(), u, bits)
        sk, si = oracle.radix_sort(keys, bits)
        got = plugin.sorted_entries()
        assert np.array_equal(got[:, 0], sk), "sorted keys differ (must be bit-exact)"
        assert np.array_equal(got[:, 1], si), "sort permutation differs (must be bit-exact)"
        til = oracle.render_tiles(oc, case.view.to_abi(), u, s_abi, want_image=s.rasterize_mode == B.RasterizeMode.Depth)
        fs = plugin.frame_stats()
        assert fs.n_visible == til["n_vis"], "n_visible differs"
        rec, ids = plugin.projected()
        assert np.array_equal(ids, til["rank_to_id"])
        if not len(ids):
            return
        orec = oracle.project(oc, case.view.to_abi(), u, s_abi, ids)
        drawn = orec["xlo"] <= orec["xhi"]
        bb = rec[:, 6:8].view(np.uint32)
        gdrawn = ((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)) & ((bb[:, 1] & 0xFFFF) <= (bb[:, 1] >> 16))
        bad = np.flatnonzero(gdrawn != drawn)
        assert not len(bad), f"drawn decision differs for gaussians {ids[bad][:8]} (oracle drawn: {drawn[bad][:8]})"
        if s.aabb and s.gaussian_mode == B.GaussianMode.Gaussian3d:
            geo = np.stack([orec["cx"], orec["cy"]] + [orec["extra"][:, j] for j in range(4)], 1)
        else:
            geo = np.stack([orec[k] for k in ("cx", "cy", "ux", "uy", "vx", "vy")], 1)
        ok = PC.bits_agree(rec[drawn, :6], geo[drawn])
        if not ok.all():
            r, c = np.argwhere(~ok)[0]
            raise AssertionError(f"geometry of gaussian {ids[drawn][r]} field {c}: {rec[drawn][r, c]!r} vs {geo[drawn][r, c]!r}")
        assert np.array_equal(bb[drawn, 0], orec["xlo"][drawn].astype(np.uint32) | (orec["xhi"][drawn].astype(np.uint32) << 16))
        assert np.array_equal(bb[drawn, 1], orec["ylo"][drawn].astype(np.uint32) | (orec["yhi"][drawn].astype(np.uint32) << 16))
        assert PC.bits_agree(rec[drawn, 11], orec["op"][drawn]).all(), "opacity differs"
        col = rec[drawn, 8:11]
        if s.rasterize_mode == B.RasterizeMode.Color:
            want = np.stack([orec[k] for k in ("r", "g", "b")], 1)[drawn]
            bound = PC.colour_bound(oc, case.view, case.model, int(s.color_space), ids[drawn])
            lit = (s.draw_mode == B.DrawMode.HighlightSelected) & (oc.position_visibility[ids[drawn], 3] > 0.5)
            bound[lit] = 0.0
            ok = PC.colours_agree(col, want, bound)
            if not ok.all():
                r, c = np.argwhere(~ok)[0]
                raise AssertionError(f"colour of gaussian {ids[drawn][r]} channel {c}: {col[r, c]!r} vs {want[r, c]!r} "
                                     f"(bound {bound[r, c]:.3g})")
            with np.errstate(invalid="ignore", divide="ignore"):
                ratio = np.abs(col.astype(np.float64) - want) / bound
            ratio = ratio[np.isfinite(ratio) & (bound > 0)]
            key = f"{geom} {case.layout} {'identity' if case.model is None else 'model'} cs{int(s.color_space)}"
            if len(ratio):
                WORST[key] = max(WORST.get(key, 0.0), float(ratio.max()))
        elif s.rasterize_mode == B.RasterizeMode.Depth:
            want, dmin, dmax = depth_colours(case, u, si, ids[drawn])
            assert np.abs(col - want).max() <= 2e-6, f"Depth colours differ (dmin {dmin}, dmax {dmax})"
            img = plugin.render_view(h, s, case.view, transform=case.transform, fmt="rgba32f")
            assert np.abs(img - til["image"]).max() <= 1e-3
        return rec, orec, ids
    finally:
        h.destroy()


@pytest.mark.parametrize("name,geom,variant", PARAMS, ids=[f"{n}-{g}-v{v}" for n, g, v in PARAMS])
def test_projection_vs_oracle(plugin, oracle, cases, name, geom, variant):
    check_case(plugin, oracle, cases[name], geom, variant)
