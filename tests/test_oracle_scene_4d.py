"""bgs_render_scene_4d's CPU oracle (scene4d_oracle/) against the oracles it joins: one Gaussian4d cloud is
temporal_oracle's frame bit for bit, 3D clouds alone are scene_oracle's frame, a split 4D cloud is the whole cloud, and
a 3D cloud in a Velocity frame is drawn as nothing.  Also the plugin's check of a 4D entity list."""
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import scene4d_cases as S4
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import check_scene_entities_4d
from scene4d_oracle import scene4d_oracle as S4O
from scene_oracle import scene_oracle as SO
from temporal_oracle import temporal_oracle as T

VIEW = B.headless_view(160, 96)
PREV = B.perspective_view((0.1, 1.45, 5.1), (0.0, 1.5, 4.0), 160, 96)
M = B.RasterizeMode
KEYS = ("sorted", "records", "rank_to_id", "depths", "tile_ranges", "tile_entries", "image")


def _uniform(settings, tr=None, cloud=None):
    return B.GaussianSplattingPlugin.cloud_uniform(settings, tr, None if cloud is None else cloud.compute_aabb())


def _extras(mode):
    ex = abi.bgs_render_extras(num_classes=3)
    if mode == M.OpticalFlow:
        ex.previous_clip_from_world[:] = PREV.to_abi().clip_from_world[:]
        ex.delta_time = 1.0 / 30.0
    return ex


def _depth_buffer(seed):
    return np.random.default_rng(seed).random((96, 160), np.float32) * np.float32(0.04)


@pytest.mark.parametrize("aabb", [False, True])
@pytest.mark.parametrize("mode", [M.Color, M.Depth, M.Position, M.Classification, M.OpticalFlow, M.Velocity])
def test_one_4d_cloud_is_the_temporal_oracle_frame(mode, aabb):
    cloud = S4.performer(2500, 3)
    st = S4.settings_4d(B.CloudSettings(rasterize_mode=mode, aabb=aabb, num_classes=3), 0.4, -0.2, 1.3)
    u = _uniform(st, SC.transform((0.2, -0.1, 0.3), 1.1, 0.4), cloud)
    s, ex = st.to_abi(), _extras(mode)
    zs = _depth_buffer(1) if mode == M.Color else None
    got = S4O.frame([(cloud, u, (st.time_start, st.time_stop))], VIEW.to_abi(), s, ex, scene=zs)
    want = T.frame(cloud, VIEW.to_abi(), u, s, st.time_start, st.time_stop, extras=ex, scene=zs)
    for key in ("records", "rank_to_id", "depths", "image"):
        assert got[key].tobytes() == want[key].tobytes(), key
    assert 0 < S4.drawn(got["records"]).sum() < len(got["records"])   # some are masked by time


@pytest.mark.parametrize("mode", [M.Color, M.Depth, M.Position])
def test_3d_clouds_alone_are_the_scene_oracle_frame(mode):
    listed = []
    for cloud, layout, _, tr, kw in S4.room():
        st = B.CloudSettings(rasterize_mode=mode, **kw)
        listed.append((SC.oracle_cloud(cloud, layout), _uniform(st, tr, cloud), layout == "cov"))
    s = B.CloudSettings(rasterize_mode=mode).to_abi()
    got = S4O.frame(listed, VIEW.to_abi(), s, _extras(mode))
    want = SO.render_tiles(listed, VIEW.to_abi(), s)
    assert np.array_equal(got["sorted"], SO.sorted_entries(listed, VIEW.to_abi()))
    for key in ("tile_ranges", "tile_entries", "rank_to_id", "image"):
        assert got[key].tobytes() == want[key].tobytes(), key


@pytest.mark.parametrize("k", [2, 3, 7])
@pytest.mark.parametrize("mode", [M.Color, M.Depth, M.Velocity])
def test_split_4d_cloud_is_the_whole_cloud(mode, k):
    cloud = S4.performer(2500, 4)
    st = S4.settings_4d(B.CloudSettings(rasterize_mode=mode), 0.6)
    u = _uniform(st, SC.transform((0.0, 0.1, -0.3), 0.9, -0.3), cloud)
    s, w = st.to_abi(), (st.time_start, st.time_stop)
    zs = _depth_buffer(2)
    whole = S4O.frame([(cloud, u, w)], VIEW.to_abi(), s, _extras(mode), scene=zs)
    split = S4O.frame([(cloud.subset(ix), u, w) for ix in SC.pieces(len(cloud), k)], VIEW.to_abi(), s, _extras(mode), scene=zs)
    for key in KEYS:
        assert split[key].tobytes() == whole[key].tobytes(), key


def test_3d_clouds_in_a_velocity_frame_draw_nothing():
    room = S4.room()
    listed = [(SC.oracle_cloud(c, layout), _uniform(B.CloudSettings(**kw), tr, c), layout == "cov") for c, layout, _, tr, kw in room]
    n3 = sum(len(c) for c, _, _ in listed)
    cloud = S4.performer(2000, 5)
    st = S4.settings_4d(B.CloudSettings(rasterize_mode=M.Velocity), 0.5)
    listed.append((cloud, _uniform(st, None, cloud), (st.time_start, st.time_stop)))
    got = S4O.frame(listed, VIEW.to_abi(), B.CloudSettings(rasterize_mode=M.Velocity).to_abi(), _extras(M.Velocity))
    three = got["rank_to_id"] < n3
    assert three.any() and not S4.drawn(got["records"][three]).any()
    assert (got["records"][three][:, 2:6] == 0).all() and (got["records"][three][:, 8:11] == 0).all()
    assert not np.isin(got["tile_entries"], np.flatnonzero(three)).any()


class _H3:
    aabb = None


class _H4(_H3):
    temporal = True


def test_entity_check_of_4d_lists():
    g4 = S4.settings_4d(B.CloudSettings(), 0.3)
    base = B.CloudSettings()
    h3, h4 = _H3(), _H4()
    # per-entity: the times, windows and playback, and a 4D entity's gaussian_mode
    other = dataclasses.replace(g4, time=0.9, time_start=-1.0, time_stop=2.0, time_scale=0.5, playback_mode=B.PlaybackMode.Loop,
                                global_opacity=0.5)
    frame = check_scene_entities_4d([(h3, base, None), (h4, g4, None), (h4, other, SC.transform((1, 0, 0)))])
    assert frame.gaussian_mode == B.GaussianMode.Gaussian3d and frame.time == base.time
    assert check_scene_entities_4d([(h4, g4, None), (h4, other, None)]).gaussian_mode == B.GaussianMode.Gaussian4d
    g2 = dataclasses.replace(base, gaussian_mode=B.GaussianMode.Gaussian2d)
    assert check_scene_entities_4d([(h3, g2, None), (h4, dataclasses.replace(g4, gaussian_mode=B.GaussianMode.Gaussian4d), None)]).gaussian_mode == B.GaussianMode.Gaussian2d
    bad = [
        [(h3, base, None), (h4, dataclasses.replace(g4, gaussian_mode=B.GaussianMode.Gaussian3d), None)],   # 4D entity not 4D
        [(h3, dataclasses.replace(base, gaussian_mode=B.GaussianMode.Gaussian4d), None), (h4, g4, None)],   # 3D entity as 4D
        [(h3, base, None), (h3, g2, None), (h4, g4, None)],                                                  # 2D and 3D mixed
        [(h3, dataclasses.replace(g2, aabb=True), None), (h4, dataclasses.replace(g4, aabb=True), None)],   # 2D + AABB + 4D
        [(h3, base, None), (h4, dataclasses.replace(g4, rasterize_mode=M.Depth), None)],                    # frame-wide field
        [],
        [(h4, g4, None)] * 65,
    ]
    for entities in bad:
        with pytest.raises(ValueError):
            check_scene_entities_4d(entities)
