"""The projection and key-gen constructions of `project_cases.py`, checked on the CPU: every class is reached (each
knife class on both sides of its threshold), the oracle decides the constructed inputs the way the classes say, and
the derived colour bound holds for the oracle's own f32 colour against the float64 WGSL restatement."""
import math

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import project_cases as PC
import wgsl_emu as W

f32 = np.float32

# classes each case must reach (at least one gaussian each)
REACH = {
    "draw_Selected": ["DRAW_HALF", "DRAW_BELOW", "DRAW_ABOVE", "DRAW_NEGZERO", "DRAW_NEG", "DRAW_NAN", "DRAW_INF"],
    "cutoff": ["CUT_LAST_CLAMPED", "CUT_FIRST_KEPT", "CUT_A_ZERO", "O_ZERO", "O_NEG", "O_NAN", "O_GT1", "O_SUBNORMAL"],
    "sigma": ["SIG_SHORTCUT", "SIG_ZERO", "SIG_NEGZERO", "SIG_SUBNORMAL", "SIG_INF", "SIG_NAN", "SIG_SIGNZERO"],
    "obb_identity": ["B0_ANEC", "EV_NAN", "MINOR_NONFINITE", "DET_ZERO", "DET_NAN"],
    "obb_affine": ["EV_NAN", "MINOR_NONFINITE", "DET_ZERO", "DET_NAN"],
    "obb_mirror": ["EV_NAN", "MINOR_NONFINITE", "DET_ZERO", "DET_NAN"],
    "bbox": ["BB_ON", "BB_UP", "BB_DOWN", "BB_SLACK", "BB_HUGE", "BB_OFFCENTRE", "BB_CLAMPED_EMPTY"],
    "surfel": ["SURFEL_D_BELOW", "SURFEL_D_ABOVE_NEAR", "SURFEL_FLOOR", "SURFEL_EXTENT", "SURFEL_REJECTED"],
    "surfel_extent": ["EX_ON", "EX_ABOVE", "EX_BELOW", "EY_ON", "EY_ABOVE", "EY_BELOW"],
    "keygen_far": ["KEY_D2_INF", "KEY_DEN_WINDOW", "KEY_DEN_OVER", "KEY_SUM_OVERFLOW", "KEY_NONFINITE"],
    "f16_specials": ["F16_ROT_INF", "F16_ROT_NAN", "F16_ROT_SUB", "F16_SCALE_INF", "F16_SCALE_NAN", "F16_SCALE_SUB",
                     "F16_SH_INF", "F16_SH_NAN", "F16_SH_SUB"],
    "cov_nonpd": ["COV_NONPD", "COV_INF", "COV_NAN", "COV_SUB", "COV_PD"],
}


@pytest.fixture(scope="module")
def cases(oracle):
    return {c.name: c for c in PC.all_cases(oracle)}


@pytest.mark.parametrize("name", sorted(REACH))
def test_every_class_reached(cases, name):
    c = cases[name]
    missing = [k for k in REACH[name] if not c.tags[k].any()]
    assert not missing, f"{name}: classes not reached: {missing}"


def test_case_index_matches_the_cases(cases):
    assert [(c.name, tuple(c.geoms)) for c in cases.values()] == [(n, tuple(g)) for n, g in PC.case_index()]


def test_surfel_restatement_is_the_oracle(oracle, cases):
    """`surfel_f32` (which the ex / ey knife is walked with) gives the oracle's 2DGS record bit for bit: the means,
    the radius max(sqrt ex, sqrt ey, cutoff 0.707106), and the rejection at ex or ey < 1e-4."""
    for name in ("surfel", "surfel_extent"):
        c = cases[name]
        rec = PC.oracle_records(oracle, c, "aabb2d")
        q = PC.surfel_f32(c.cloud, c.view, c.model, 3.0)
        dr = PC.drawn_of(rec)
        assert PC.bits_agree(q["mean0"][dr], rec["extra"][dr, 4]).all() and PC.bits_agree(q["mean1"][dr], rec["extra"][dr, 5]).all()
        with np.errstate(invalid="ignore"):
            rq = np.maximum(np.maximum(np.sqrt(q["ex"]), np.sqrt(q["ey"])), f32(3.0) * f32(0.707106))
            rejected = ~(np.abs(q["d"]) >= f32(1e-4)) | (q["ex"] < f32(1e-4)) | (q["ey"] < f32(1e-4))
        assert PC.bits_agree(rq[dr], rec["extra"][dr, 3]).all()
        vis = ~np.isnan(rec["cx"])
        assert np.array_equal(dr[vis], ~rejected[vis] & dr[vis]) and not (dr & rejected).any()
        if name == "surfel_extent":
            # the knife: exactly 1e-4f and one ulp above are kept (`<` is strict), one ulp below is rejected
            for k in ("EX", "EY"):
                assert dr[c.tags[k + "_ON"]].all() and dr[c.tags[k + "_ABOVE"]].all() and not dr[c.tags[k + "_BELOW"]].any()


def test_zero_sigma_reaches_a_shortcut_sensitive_record(cases):
    """Some zero-Sigma splat's record differs between Sigma and T Sigma T^t (identity T): the identity shortcut must
    not be taken on a zero entry, and the GPU file shows whether it is."""
    hits = sum(int(cases[f"sigma_zero_{v}"].tags["SIG0_SHORTCUT_CHANGES"].sum()) for v in range(10))
    assert hits >= 5


def test_sh_onehot_reaches_every_coefficient_and_direction(cases):
    sh = [c for n, c in cases.items() if n.startswith("sh_")]
    assert len(sh) >= 2 * 30
    for k in range(48):
        assert all(c.tags[f"SH_C{k}"].sum() >= 3 for c in sh)
    # the axes and the basis functions' zeros are among the directions (centre gaussians: exactly the wanted one up to
    # the f32 rounding of the eye)
    dl = np.concatenate([PC.local_direction64(c.cloud, c.view, c.model)[:1] for c in sh if "identity" in c.name])
    for axis in np.eye(3):
        for sgn in (1, -1):
            assert (np.abs(dl - sgn * axis).max(1) < 1e-6).any()
    b = PC.sh_basis64(dl)
    assert all((np.abs(b[:, k]) < 1e-6).any() for k in range(1, 16)), "a zero of every non-constant basis function"


def test_cutoff_knife_straddles_the_clamp(oracle, cases):
    c = cases["cutoff"]
    o = c.cloud.scale_opacity[:, 3]
    a, cut = PC.cutoff_f32(oracle, o)
    last = a[c.tags["CUT_LAST_CLAMPED"]]
    first = a[c.tags["CUT_FIRST_KEPT"]]
    assert np.all(last == f32(2.0 ** -20)) and np.all(first == f32(2.0 ** -19))
    assert np.all(cut[c.tags["CUT_LAST_CLAMPED"]] == np.sqrt(f32(1e-6)))
    # a never equals 1e-6f near the knife: `>` and `>=` decide every f32 opacity alike
    walk = PC.ulp_walk(f32(math.exp(-4.5)), np.arange(-20000, 20001, 13))[0]
    aw, _ = PC.cutoff_f32(oracle, walk)
    assert not np.any(aw == f32(1e-6)) and np.any(aw < f32(1e-6)) and np.any(aw > f32(1e-6))
    assert np.all((aw.astype(np.float64) / 2.0 ** -20) % 1.0 == 0.0)


def test_draw_mode_decisions_on_the_oracle(oracle, cases):
    """Selected draws w >= 0.5 (w < 0.5 discards; NaN is drawn); HighlightSelected recolours w > 0.5 only."""
    c = cases["draw_Selected"]
    rec = PC.oracle_records(oracle, c, "obb3d")
    vis = ~np.isnan(rec["cx"]) & PC.drawn_of(PC.oracle_records(oracle, c, "obb3d", draw_mode=B.DrawMode.All))
    drawn = PC.drawn_of(rec)
    w = c.cloud.position_visibility[:, 3]
    assert np.all(drawn[vis & c.tags["DRAW_HALF"]]) and np.all(drawn[vis & c.tags["DRAW_ABOVE"]])
    assert not drawn[c.tags["DRAW_BELOW"]].any() and not drawn[c.tags["DRAW_NEG"]].any()
    assert np.all(drawn[vis & c.tags["DRAW_NAN"]]) and (vis & c.tags["DRAW_HALF"]).sum() > 20
    h = PC.oracle_records(oracle, cases["draw_HighlightSelected"], "obb3d")
    lit = (h["r"] == f32(0.3)) & (h["g"] == f32(1.0)) & (h["b"] == f32(0.1)) & (h["op"] == f32(1.0))
    with np.errstate(invalid="ignore"):
        assert np.array_equal(lit[vis], (w > 0.5)[vis])


def test_sigma_classes_on_the_oracle(oracle, cases):
    """Feeding Sigma itself (what the identity shortcut uses) through the covariance path gives the full path's record
    bit for bit wherever the shortcut is taken."""
    c = cases["sigma"]
    assert c.tags["SIG_SIGNZERO"].sum() >= 4
    S = PC.sigma_f32(c.cloud.rotation, c.cloud.scale_opacity)
    e = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    raw = PC.RawCovariance(c.cloud.position_visibility, c.cloud.spherical_harmonic, e[:, :4],
                           np.concatenate([e[:, 4:], c.cloud.scale_opacity[:, 3:], c.cloud.scale_opacity[:, 3:]], 1))
    differ = np.zeros(len(raw), bool)
    for geom in ("obb3d", "aabb3d"):
        full = PC.oracle_records(oracle, c, geom)
        s = PC.settings(geom, **c.settings).to_abi()
        s.reserved = 1
        u = B.GaussianSplattingPlugin.cloud_uniform(PC.settings(geom, **c.settings))
        short = oracle.project(raw, c.view.to_abi(), u, s, np.arange(len(raw), dtype=np.uint32))
        for k in ("cx", "cy", "ux", "uy", "vx", "vy"):
            differ |= ~PC.bits_agree(full[k], short[k])
        for j in range(4):
            differ |= ~PC.bits_agree(full["extra"][:, j], short["extra"][:, j])
    assert not differ[c.tags["SIG_SHORTCUT"]].any(), "the shortcut must be exact where it is taken"


def test_depth_cases_shape(oracle, cases):
    """n_vis 0 / 1 / 2 / many, with and without culled gaussians at the lowest and highest index."""
    got = {}
    for name in ("depth_culled", "depth_all_visible", "depth_one_visible", "depth_none_visible", "depth_two_visible"):
        c = cases[name]
        u = B.GaussianSplattingPlugin.cloud_uniform(PC.settings("obb3d", **c.settings))
        keys = oracle.keygen(c.cloud.position_visibility, c.view.to_abi(), u, 32)
        got[name] = (int((keys != 0xFFFFFFFF).sum()), bool(keys[0] == 0xFFFFFFFF), bool(keys[-1] == 0xFFFFFFFF))
    assert got["depth_culled"][0] >= 2 and got["depth_culled"][1:] == (True, True)
    assert got["depth_all_visible"] == (62, False, False)
    assert got["depth_one_visible"] == (1, True, True)
    assert got["depth_none_visible"] == (0, True, True)
    assert got["depth_two_visible"] == (2, True, False)


def _f64_colour(dl, sh, color_space):
    sh_ = W.Shader.__new__(W.Shader)
    v = sh_.spherical_harmonics_lookup(W.Vec(*dl), [float(x) for x in sh])
    out = np.array([v[0], v[1], v[2]], np.float64)
    if color_space == 0:
        out = np.where(out <= 0.04045, out / 12.92, np.abs((out + 0.055) / 1.055) ** 2.4)
    return out


def test_colour_bound_holds_for_the_oracle(oracle, cases):
    """The oracle's f32 colour against the float64 SH lookup of wgsl_emu.py at the float64 direction: within the
    derived bound (which also covers the CUDA side's rsqrt.approx and __powf).  Largest err / bound recorded."""
    worst = 0.0
    n = 0
    for name, c in cases.items():
        if not (name.startswith("sh_") or name.startswith("general_")):
            continue
        s = PC.settings("obb3d", **c.settings)
        cs = int(s.color_space)
        oc = c.oracle_cloud()
        rec = PC.oracle_records(oracle, c, "obb3d")
        keep = np.flatnonzero(PC.drawn_of(rec))[:150]
        bound = PC.colour_bound(oc, c.view, c.model, cs, keep)
        dl = PC.local_direction64(oc, c.view, c.model)[keep]
        want = np.array([_f64_colour(d, oc.spherical_harmonic[i], cs) for d, i in zip(dl, keep)])
        got = np.stack([rec["r"], rec["g"], rec["b"]], 1)[keep].astype(np.float64)
        err = np.abs(got - want)
        assert np.all(err <= bound), f"{name}: colour error {err.max():.3g} above its bound"
        worst = max(worst, float((err / np.maximum(bound, 1e-30)).max()))
        n += len(keep)
    assert n > 5000 and 0.0 < worst <= 1.0


def test_colour_bound_separates_a_wrong_sh_constant(cases):
    """For every basis function, the one-hot gaussians of its coefficients see a colour change above their bound when
    the SH constant is off by one unit in its fifth significant digit."""
    sh = [c for n, c in cases.items() if n.startswith("sh_")]
    for k in range(16):
        d = 10.0 ** (math.floor(math.log10(abs(PC.SHC[k]))) - 4)
        seen = 0
        for c in sh:
            sel = np.flatnonzero(c.tags[f"SH_C{3 * k}"] | c.tags[f"SH_C{3 * k + 1}"] | c.tags[f"SH_C{3 * k + 2}"])
            bound = PC.colour_bound(c.cloud, c.view, c.model, 1, sel)
            b = PC.sh_basis64(PC.local_direction64(c.cloud, c.view, c.model)[sel])[:, k]
            change = np.abs(c.cloud.spherical_harmonic[sel].reshape(-1, 16, 3)[:, k, :] * d * b[:, None])
            seen += int((change > bound).any(1).sum())
        assert seen >= 8, f"SH constant {k}: a change in its fifth digit hides under the bound"
