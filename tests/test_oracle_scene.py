"""bgs_render_scene's CPU oracle (scene_oracle/) against the single-cloud oracle: one cloud is the existing frame bit for
bit, a split cloud is the whole cloud bit for bit, depth-separated clouds are the reference's far-first composite, and
interpenetrating clouds are not (the case the joint sort exists for).  Also the plugin's check of its entity list."""
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import scene_cases as SC
from bevy_gaussian_splatting_b200.plugin import check_scene_entities
from scene_oracle import scene_oracle as SO

VIEW = B.headless_view(160, 96)


def _uniform(settings, tr=None, cloud=None):
    return B.GaussianSplattingPlugin.cloud_uniform(settings, tr, None if cloud is None else cloud.compute_aabb())


@pytest.mark.parametrize("mode", [B.RasterizeMode.Color, B.RasterizeMode.Depth, B.RasterizeMode.Position])
@pytest.mark.parametrize("aabb", [False, True])
def test_one_cloud_is_the_oracle_frame(oracle, mode, aabb):
    cloud = SC.cloud_in_box(3000, 1)
    st = B.CloudSettings(rasterize_mode=mode, aabb=aabb)
    u = _uniform(st, SC.transform((0.3, -0.2, 0.5), 1.1, 0.4), cloud)
    s = st.to_abi()
    keys = oracle.keygen(cloud.position_visibility, VIEW.to_abi(), u, 32)
    order = oracle.stable_sort(keys)
    se = SO.sorted_entries([(cloud, u, False)], VIEW.to_abi(), 32)
    assert np.array_equal(se[:, 0], keys[order]) and np.array_equal(se[:, 1], order)
    want = oracle.render_tiles(cloud, VIEW.to_abi(), u, s)
    got = SO.render_tiles([(cloud, u, False)], VIEW.to_abi(), s)
    for key in ("tile_ranges", "tile_entries", "rank_to_id"):
        assert np.array_equal(got[key], want[key]), key
    assert got["image"].tobytes() == want["image"].tobytes()
    if mode != B.RasterizeMode.Depth:   # (orc_project leaves Depth colours to the frame pass)
        rec = oracle.project(cloud, VIEW.to_abi(), u, s, want["rank_to_id"])
        assert got["records"].tobytes() == rec.tobytes()
    assert SO.render_ref([(cloud, u, False)], VIEW.to_abi(), s).tobytes() == oracle.render_ref(cloud, VIEW.to_abi(), u, s).tobytes()


@pytest.mark.parametrize("k", [2, 3, 7])
@pytest.mark.parametrize("mode", [B.RasterizeMode.Color, B.RasterizeMode.Depth])
def test_split_cloud_is_the_whole_cloud(mode, k):
    cloud = SC.cloud_in_box(2500, 2)
    st = B.CloudSettings(rasterize_mode=mode)
    u = _uniform(st, SC.transform((0.0, 0.1, -0.3), 0.9, -0.3), cloud)
    s = st.to_abi()
    whole = [(cloud, u, False)]
    split = [(cloud.subset(ix), u, False) for ix in SC.pieces(len(cloud), k)]
    assert np.array_equal(SO.sorted_entries(split, VIEW.to_abi()), SO.sorted_entries(whole, VIEW.to_abi()))
    a, b = SO.render_tiles(split, VIEW.to_abi(), s), SO.render_tiles(whole, VIEW.to_abi(), s)
    for key in ("tile_ranges", "tile_entries", "rank_to_id", "records", "image"):
        assert a[key].tobytes() == b[key].tobytes(), key


def _far_first_chain(oracle, listed, settings):
    """The reference's per-entity order: each cloud a draw of its own, the farthest first, each over the last."""
    cam = VIEW.to_abi().world_position
    def dist(item):
        cloud, u, _ = item
        m = np.array(u.transform, np.float32).reshape(4, 4).T
        c = m @ np.append(cloud.position_visibility[:, :3].mean(0), 1.0)
        return float(np.linalg.norm(c[:3] - np.array(cam[:3])))
    img = None
    for cloud, u, _ in sorted(listed, key=dist, reverse=True):
        img = oracle.render_ref(cloud, VIEW.to_abi(), u, settings, dst=img)
    return img


def test_depth_separated_clouds_match_the_far_first_composite(oracle):
    st = B.CloudSettings()
    near = SC.cloud_in_box(1500, 3, centre=(0.0, 1.5, 1.0), half=0.8)
    far = SC.cloud_in_box(1500, 4, centre=(0.0, 1.5, -3.0), half=0.8)
    listed = [(near, _uniform(st, None, near), False), (far, _uniform(dataclasses.replace(st, global_opacity=0.7), None, far), False)]
    chain = _far_first_chain(oracle, listed, st.to_abi())
    assert np.abs(SO.render_ref(listed, VIEW.to_abi(), st.to_abi()) - chain).max() <= 1e-5
    assert np.abs(SO.render_tiles(listed, VIEW.to_abi(), st.to_abi())["image"] - chain).max() <= 1e-3


def test_interpenetrating_clouds_differ_from_the_far_first_composite(oracle):
    st = B.CloudSettings()
    a = SC.cloud_in_box(2000, 5, centre=(0.0, 1.5, -1.0), half=1.0, scale=0.1)
    b = SC.cloud_in_box(2000, 6, centre=(0.1, 1.5, -1.1), half=1.0, scale=0.1)
    listed = [(a, _uniform(st, None, a), False), (b, _uniform(st, SC.transform(yaw=0.5), b), False)]
    chain = _far_first_chain(oracle, listed, st.to_abi())
    joint = SO.render_ref(listed, VIEW.to_abi(), st.to_abi())
    assert np.abs(joint - chain).max() > 0.05
    assert np.abs(SO.render_tiles(listed, VIEW.to_abi(), st.to_abi())["image"] - joint).max() <= 1e-3


class _Handle:
    aabb = None


def test_entity_check_rejects_disagreeing_frame_fields():
    base = B.CloudSettings()
    h = _Handle()
    ok = [(h, base, None), (h, dataclasses.replace(base, global_opacity=0.5, global_scale=2.0, color_space=B.GaussianColorSpace.LinRec709Display), SC.transform((1, 0, 0)))]
    assert check_scene_entities(ok) is base
    for field, value in [("rasterize_mode", B.RasterizeMode.Depth), ("draw_mode", B.DrawMode.Selected), ("aabb", True),
                         ("gaussian_mode", B.GaussianMode.Gaussian2d), ("opacity_adaptive_radius", False), ("num_classes", 3),
                         ("radix_sort_depth_bits", B.RadixSortDepthBits.Bits16)]:
        with pytest.raises(ValueError, match=field):
            check_scene_entities([(h, base, None), (h, dataclasses.replace(base, **{field: value}), None)])
    with pytest.raises(ValueError):
        check_scene_entities([])
    with pytest.raises(ValueError):
        check_scene_entities([(h, base, None)] * 65)
