"""Python host mirror of the plugin surface for the forward splat path.

Reference: `GaussianSplattingPlugin` (src/lib.rs:48-80) wires, for this path, the render-world
system `run_radix_sort` (src/sort/radix.rs:616-756) and the `DrawGaussians` render command
(src/render/mod.rs:986-992,1501-1569), both invoked once per `GaussianCamera` view per frame over
entities holding `(PlanarGaussian3dHandle, CloudSettings)`.  Here the same roles exist with the
same names, but the per-view work is ONE call across the C ABI (`bgs_render`).

This module is test/bench plumbing above the ABI (the production host stays Rust, see
INTEGRATION.md); it never computes anything itself and has no fallback path.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import warnings

import numpy as np

from . import abi
from .camera import GaussianCamera, View
from .gaussian import SH_WIDTHS, PlanarGaussian3d, PlanarGaussian4d, aabb_of_extent, compute_aabb
from .particles import PARTICLE_BEHAVIOR_DTYPE, as_particle_behaviors
from .settings import CloudSettings, GaussianMode, RasterizeMode, SparseSelect


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def scene_depth_arg(scene_depth, width: int, height: int) -> tuple[abi.bgs_scene_depth | None, int | None]:
    """(`bgs_scene_depth`, producer stream) for any object with `__cuda_array_interface__` (a torch CUDA tensor, a CuPy
    array, ...): float32, shape (height, width), rows contiguous, the row stride taken from the interface.  The producer
    stream is the interface's (v3) "stream" entry, None when it names none.  None -> (None, None)."""
    if scene_depth is None:
        return None, None
    cai = getattr(scene_depth, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError("scene_depth must expose __cuda_array_interface__ (device memory)")
    if np.dtype(cai["typestr"]) != np.dtype("<f4"):
        raise TypeError(f"scene_depth must be float32, not {cai['typestr']}")
    if tuple(cai["shape"]) != (height, width):
        raise ValueError(f"scene_depth must have shape ({height}, {width}), not {tuple(cai['shape'])}")
    strides = cai.get("strides")
    pitch = 4 * width
    if strides is not None:
        if strides[1] != 4 and width > 1:
            raise ValueError("scene_depth rows must be contiguous")
        pitch = int(strides[0])
    return abi.bgs_scene_depth(depth=int(cai["data"][0]), pitch_bytes=pitch), cai.get("stream")


_cuda_driver = None


def _stream_wait(consumer: int, producer: int) -> None:
    """Order `consumer` (a CUstream) after the work queued so far on `producer` (a CUstream, or the interface's 1 / 2 for
    the legacy / per-thread default stream, which are also the driver's handles for them): one event, recorded on the
    producer and waited for on the device, as __cuda_array_interface__ v3 asks of a consumer."""
    global _cuda_driver
    if _cuda_driver is None:
        _cuda_driver = C.CDLL("libcuda.so.1")
    cu, ev = _cuda_driver, C.c_void_p()
    for call in (lambda: cu.cuEventCreate(C.byref(ev), C.c_uint(2)),        # CU_EVENT_DISABLE_TIMING
                 lambda: cu.cuEventRecord(ev, C.c_void_p(producer)),
                 lambda: cu.cuStreamWaitEvent(C.c_void_p(consumer), ev, C.c_uint(0))):
        rc = call()
        if rc != 0:
            if ev.value:
                cu.cuEventDestroy_v2(ev)
            raise RuntimeError(f"scene_depth: ordering after the producer's stream failed (CUDA driver error {rc})")
    cu.cuEventDestroy_v2(ev)   # (released once the wait has been satisfied)


@dataclasses.dataclass
class CloudTransform:
    """GlobalTransform of the cloud entity -> CloudUniform.transform (render/mod.rs:1056-1072)."""

    matrix: np.ndarray = dataclasses.field(default_factory=lambda: np.eye(4, dtype=np.float32))


def similarity_transform(translation=(0.0, 0.0, 0.0), rotation_wxyz=(1.0, 0.0, 0.0, 0.0), scale: float = 1.0,
                         pivot=(0.0, 0.0, 0.0)) -> np.ndarray:
    """The 4x4 f32 matrix (CloudTransform.matrix's convention; `transform` passes it column-major) that scales by
    `scale` and rotates by the quaternion `rotation_wxyz` (normalised here) about `pivot`, then translates by
    `translation`: T(pivot + translation) R S T(-pivot), built in f64.  A gizmo rotates a selection about its centre."""
    q = np.asarray(rotation_wxyz, np.float64)
    w, x, y, z = q / np.linalg.norm(q)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    p = np.asarray(pivot, np.float64)
    m = np.eye(4)
    m[:3, :3] = float(scale) * R
    m[:3, 3] = p + np.asarray(translation, np.float64) - m[:3, :3] @ p
    return m.astype(np.float32)


class PlanarGaussian3dHandle:
    """A cloud resident in HBM (the role of `Handle<PlanarGaussian3d>` + its prepared GPU planes)."""

    _next_serial = 0

    def __init__(self, plugin: "GaussianSplattingPlugin", cloud: PlanarGaussian3d, f16: bool = False,
                 precompute_covariance: bool = False):
        PlanarGaussian3dHandle._next_serial += 1
        self.serial = PlanarGaussian3dHandle._next_serial   # never reused (id() is, once a handle is collected)
        self._plugin = plugin
        self._lib = plugin._lib
        self.n = len(cloud)
        self.f16 = f16
        self.sh_degree = cloud.sh_degree        # stored at the cloud's own SH width (the _sh upload calls)
        self.aabb = cloud.compute_aabb()        # the entity's Aabb (calculate_bounds, src/gaussian/cloud.rs:45-62)
        self._h = C.c_void_p()
        self.precompute_covariance = precompute_covariance
        d = self.sh_degree
        if precompute_covariance:
            # the reference's `precompute_covariance_3d` feature: Covariance3dOpacityPacked128 in the second plane
            sh_p, cov_op = cloud.precomputed_covariance().pack_f16()
            st = self._lib.bgs_cloud_upload_f16_cov_sh(plugin._ctx, self.n, d, _ptr(cloud.position_visibility), _ptr(sh_p),
                                                       _ptr(cov_op), C.byref(self._h))
        elif f16:
            sh_p, rso = cloud.pack_f16()
            st = self._lib.bgs_cloud_upload_f16_sh(plugin._ctx, self.n, d, _ptr(cloud.position_visibility), _ptr(sh_p),
                                                   _ptr(rso), C.byref(self._h))
        else:
            st = self._lib.bgs_cloud_upload_f32_sh(plugin._ctx, self.n, d, _ptr(cloud.position_visibility),
                                                   _ptr(cloud.spherical_harmonic), _ptr(cloud.rotation),
                                                   _ptr(cloud.scale_opacity), C.byref(self._h))
        plugin._check(st)

    @classmethod
    def _adopt(cls, plugin: "GaussianSplattingPlugin", h: C.c_void_p, n: int, f16: bool,
               precompute_covariance: bool, aabb=None) -> "PlanarGaussian3dHandle":
        """A handle owning a `bgs_cloud*` the library made (bgs_cloud_subset, _upload_khr); its Aabb is `aabb`, or computed
        from the positions read back, as `calculate_bounds` would compute it for the cloud once saved and loaded."""
        self = cls.__new__(cls)
        PlanarGaussian3dHandle._next_serial += 1
        self.serial = PlanarGaussian3dHandle._next_serial
        self._plugin, self._lib = plugin, plugin._lib
        self.n, self.f16, self.precompute_covariance = n, f16, precompute_covariance
        self._h = h
        d = C.c_uint32()
        plugin._check(plugin._lib.bgs_cloud_sh_degree(h, C.byref(d)))
        self.sh_degree = int(d.value)
        self.aabb = compute_aabb(plugin.positions(self)) if aabb is None else aabb
        return self

    def destroy(self):
        if self._h:
            self._lib.bgs_cloud_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class PlanarGaussian4dHandle(PlanarGaussian3dHandle):
    """A Gaussian4d cloud resident in HBM (`bgs_cloud_upload_4d`); `render_view` draws it through `bgs_render_4d` at
    `settings.time` in the window [settings.time_start, settings.time_stop]."""

    temporal = True

    def __init__(self, plugin: "GaussianSplattingPlugin", cloud: PlanarGaussian4d):
        PlanarGaussian3dHandle._next_serial += 1
        self.serial = PlanarGaussian3dHandle._next_serial
        self._plugin, self._lib = plugin, plugin._lib
        self.n, self.f16, self.precompute_covariance = len(cloud), False, False
        self.sh_degree = 3                      # the spatial degree of the spherindrical colour
        self.aabb = cloud.compute_aabb()
        self._h = C.c_void_p()
        plugin._check(self._lib.bgs_cloud_upload_4d(plugin._ctx, self.n, *(_ptr(a) for a in cloud.planes()), C.byref(self._h)))


class ParticleBehaviorsHandle:
    """A `ParticleBehaviors` asset resident in HBM (`bgs_particles`): what the reference attaches to a cloud entity."""

    def __init__(self, plugin: "GaussianSplattingPlugin", behaviors):
        b = as_particle_behaviors(behaviors)
        self._plugin = plugin
        self._lib = plugin._lib
        self.count = len(b)
        self._h = C.c_void_p()
        plugin._check(self._lib.bgs_particles_create(plugin._ctx, _ptr(b), self.count, C.byref(self._h)))

    def get(self) -> np.ndarray:
        """The current records (velocity and acceleration advanced by every step queued so far)."""
        out = np.empty(self.count, PARTICLE_BEHAVIOR_DTYPE)
        self._plugin._check(self._lib.bgs_particles_get(self._plugin._ctx, self._h, _ptr(out)))
        return out

    def destroy(self):
        if self._h:
            self._lib.bgs_particles_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


@dataclasses.dataclass
class SceneHandles:
    """A KHR_gaussian_splatting scene resident on one GPU (`GaussianSplattingPlugin.add_scene`): one handle per primitive,
    shared by every node that places it, the scene's bundles and how many zero-length rotations each primitive had."""

    handles: list
    bundles: list
    zero_quats: list

    def entities(self) -> list:
        """(handle, settings, transform) per bundle: the entity list `render_entities`, `render_entities_aux` and
        `render_views` take."""
        return [(self.handles[b.primitive], b.settings, b.transform) for b in self.bundles]

    def destroy(self):
        for h in self.handles:
            h.destroy()


# CloudSettings fields a bgs_render_scene call takes from each entity (into its bgs_cloud_uniform); every other field is
# the frame's and must agree across the entities
SCENE_PER_ENTITY_FIELDS = frozenset({"global_opacity", "global_scale", "color_space"})


def check_scene_entities(entities) -> CloudSettings:
    """`entities`: a sequence of (handle, CloudSettings, transform or None), one bgs_render_scene call's clouds.  Returns
    the settings the frame-wide values come from (the first entity's); raises ValueError when there are none, too many,
    or two entities disagree on a frame-wide field (anything but global_opacity, global_scale and color_space)."""
    entities = list(entities)
    if not entities:
        raise ValueError("render_scene: no entities")
    if len(entities) > abi.BGS_SCENE_MAX_CLOUDS:
        raise ValueError(f"render_scene: {len(entities)} entities, at most {abi.BGS_SCENE_MAX_CLOUDS}")
    first = entities[0][1]
    for j, (_, st, _) in enumerate(entities[1:], 1):
        for f in dataclasses.fields(first):
            if f.name in SCENE_PER_ENTITY_FIELDS:
                continue
            a, b = getattr(first, f.name), getattr(st, f.name)
            if a != b:
                raise ValueError(f"render_scene: entity {j} has {f.name} = {b!r}, entity 0 {a!r}: frame-wide fields must agree")
    return first


# bgs_render_scene_4d also takes each entity's time and window, and its playback settings are its own
SCENE_4D_PER_ENTITY_FIELDS = SCENE_PER_ENTITY_FIELDS | {"time", "time_start", "time_stop", "time_scale", "playback_mode",
                                                        "gaussian_mode"}


def is_4d_handle(handle) -> bool:
    return bool(getattr(handle, "temporal", False))


def check_scene_entities_4d(entities) -> CloudSettings:
    """`check_scene_entities` for an entity list with Gaussian4d clouds (one bgs_render_scene_4d call).  time, time_start,
    time_stop, time_scale and playback_mode are per entity too.  A 4D entity's gaussian_mode must be Gaussian4d; the other
    entities' must agree and be Gaussian2d or Gaussian3d, and Gaussian2d with aabb takes no 4D entity.  Returns the
    frame's settings: the first entity's, with gaussian_mode the non-4D entities' (Gaussian4d when every entity is 4D).
    Raises ValueError on any disagreement."""
    entities = list(entities)
    if not entities:
        raise ValueError("render_scene: no entities")
    if len(entities) > abi.BGS_SCENE_MAX_CLOUDS:
        raise ValueError(f"render_scene: {len(entities)} entities, at most {abi.BGS_SCENE_MAX_CLOUDS}")
    first = entities[0][1]
    for j, (_, st, _) in enumerate(entities[1:], 1):
        for f in dataclasses.fields(first):
            if f.name in SCENE_4D_PER_ENTITY_FIELDS:
                continue
            a, b = getattr(first, f.name), getattr(st, f.name)
            if a != b:
                raise ValueError(f"render_scene: entity {j} has {f.name} = {b!r}, entity 0 {a!r}: frame-wide fields must agree")
    others = set()
    for j, (h, st, _) in enumerate(entities):
        gm = GaussianMode(st.gaussian_mode)
        if is_4d_handle(h):
            if gm != GaussianMode.Gaussian4d:
                raise ValueError(f"render_scene: entity {j} is a Gaussian4d cloud with gaussian_mode {gm.name}")
        elif gm == GaussianMode.Gaussian4d:
            raise ValueError(f"render_scene: entity {j} is not a Gaussian4d cloud but has gaussian_mode Gaussian4d")
        else:
            others.add(gm)
    if len(others) > 1:
        raise ValueError(f"render_scene: the non-4D entities disagree on gaussian_mode ({sorted(m.name for m in others)})")
    mode = others.pop() if others else GaussianMode.Gaussian4d
    if mode == GaussianMode.Gaussian2d and first.aabb and any(is_4d_handle(h) for h, _, _ in entities):
        raise ValueError("render_scene: Gaussian2d with aabb takes no Gaussian4d entity (its blend reads surfel records)")
    return dataclasses.replace(first, gaussian_mode=mode)


# CloudSettings fields a bgs_render_entities call takes for the whole frame: the one depth sort and its flags
ENTITIES_FRAME_FIELDS = ("radix_sort_depth_bits", "sort_mode", "sort_all", "binning_rounds")


def check_entities(entities) -> CloudSettings:
    """`entities`: a sequence of (handle, CloudSettings, transform or None), one bgs_render_entities call's clouds, each
    drawn with its own settings.  Returns the settings the frame-wide values (ENTITIES_FRAME_FIELDS) come from, the first
    entity's; raises ValueError when there are none, too many, or two entities disagree on a frame-wide field."""
    entities = list(entities)
    if not entities:
        raise ValueError("render_entities: no entities")
    if len(entities) > abi.BGS_SCENE_MAX_CLOUDS:
        raise ValueError(f"render_entities: {len(entities)} entities, at most {abi.BGS_SCENE_MAX_CLOUDS}")
    first = entities[0][1]
    for j, (_, st, _) in enumerate(entities[1:], 1):
        for name in ENTITIES_FRAME_FIELDS:
            a, b = getattr(first, name), getattr(st, name)
            if a != b:
                raise ValueError(f"render_entities: entity {j} has {name} = {b!r}, entity 0 {a!r}: the frame has one depth sort")
    return first


def check_entities_aux(entities) -> CloudSettings:
    """`check_entities` for one bgs_render_entities_aux call, which also raises ValueError for a Gaussian4d cloud (its
    layout has no Normal colour), a precomputed-covariance cloud (no rotation) and an entity in Velocity mode (it changes
    which splats draw, so the three frames would not share their alphas)."""
    entities = list(entities)
    first = check_entities(entities)
    for j, (h, st, _) in enumerate(entities):
        if is_4d_handle(h):
            raise ValueError(f"render_entities_aux: entity {j} is a Gaussian4d cloud")
        if getattr(h, "precompute_covariance", False):
            raise ValueError(f"render_entities_aux: entity {j} is a precomputed-covariance cloud")
        if RasterizeMode(st.rasterize_mode) == RasterizeMode.Velocity:
            raise ValueError(f"render_entities_aux: entity {j} is in Velocity mode")
    return first


def check_views(entities, views) -> CloudSettings:
    """`check_entities` for one bgs_render_views call of `views` (a sequence of View), which also raises ValueError when
    there are no views, when views x entities exceeds abi.BGS_SCENE_MAX_CLOUDS segments, and for an entity in Depth mode
    (its colour range would be per view) or OpticalFlow mode (one previous view per frame)."""
    entities, views = list(entities), list(views)
    first = check_entities(entities)
    if not views:
        raise ValueError("render_views: no views")
    if len(views) * len(entities) > abi.BGS_SCENE_MAX_CLOUDS:
        raise ValueError(f"render_views: {len(views)} views x {len(entities)} entities, at most {abi.BGS_SCENE_MAX_CLOUDS} segments")
    for j, (_, st, _) in enumerate(entities):
        mode = RasterizeMode(st.rasterize_mode)
        if mode in (RasterizeMode.Depth, RasterizeMode.OpticalFlow):
            raise ValueError(f"render_views: entity {j} is in {mode.name} mode")
    return first


def check_views_aux(entities, views) -> CloudSettings:
    """`check_entities_aux` and `check_views` for one bgs_render_views_aux call of `views` (a sequence of View): ValueError
    for no views, views x entities over abi.BGS_SCENE_MAX_CLOUDS segments, a Gaussian4d or precomputed-covariance cloud,
    and an entity in Velocity or OpticalFlow mode.  Depth entities are accepted: each view's Depth colours are over its own
    range."""
    entities, views = list(entities), list(views)
    first = check_entities(entities)
    if not views:
        raise ValueError("render_views_aux: no views")
    if len(views) * len(entities) > abi.BGS_SCENE_MAX_CLOUDS:
        raise ValueError(f"render_views_aux: {len(views)} views x {len(entities)} entities, at most {abi.BGS_SCENE_MAX_CLOUDS} segments")
    for j, (h, st, _) in enumerate(entities):
        if is_4d_handle(h):
            raise ValueError(f"render_views_aux: entity {j} is a Gaussian4d cloud")
        if getattr(h, "precompute_covariance", False):
            raise ValueError(f"render_views_aux: entity {j} is a precomputed-covariance cloud")
        mode = RasterizeMode(st.rasterize_mode)
        if mode in (RasterizeMode.Velocity, RasterizeMode.OpticalFlow):
            raise ValueError(f"render_views_aux: entity {j} is in {mode.name} mode")
    return first


def entity_settings(settings: CloudSettings) -> abi.bgs_entity_settings:
    """One entity's bgs_entity_settings."""
    s = settings.to_abi()
    return abi.bgs_entity_settings(gaussian_mode=s.gaussian_mode, rasterize_mode=s.rasterize_mode, aabb=s.aabb,
                                   opacity_adaptive_radius=s.opacity_adaptive_radius, draw_mode=s.draw_mode,
                                   num_classes=int(settings.num_classes),
                                   window=abi.bgs_time_window(float(settings.time_start), float(settings.time_stop)))


class GaussianSplattingPlugin:
    """Owns one `bgs_context` (one GPU).  `render_view` = run_radix_sort + DrawGaussians for one view."""

    FORMATS = {"rgba8_srgb": (abi.BGS_FORMAT_RGBA8_SRGB, np.uint8, 4), "rgba16f": (abi.BGS_FORMAT_RGBA16F, np.float16, 4),
               "rgba32f": (abi.BGS_FORMAT_RGBA32F, np.float32, 4)}

    def __init__(self, cuda_device: int = 0):
        self._lib = abi.load()
        self._ctx = C.c_void_p()
        st = self._lib.bgs_context_create(cuda_device, C.byref(self._ctx))
        if st != abi.BGS_OK:
            raise abi.BgsError(st, f"bgs_context_create(device={cuda_device}) failed (no usable CUDA device?)")
        self.device = cuda_device

    # -- resources
    def add_cloud(self, cloud: PlanarGaussian3d | PlanarGaussian4d, f16: bool = False,
                  precompute_covariance: bool = False) -> PlanarGaussian3dHandle:
        """A PlanarGaussian4d cloud gives a PlanarGaussian4dHandle (f32 only: the reference has no f16 4D layout)."""
        if isinstance(cloud, PlanarGaussian4d):
            if f16 or precompute_covariance:
                raise ValueError("add_cloud: a Gaussian4d cloud is stored in f32 only")
            return PlanarGaussian4dHandle(self, cloud)
        return PlanarGaussian3dHandle(self, cloud, f16, precompute_covariance)

    def add_scene(self, scene, f16: bool = False) -> SceneHandles:
        """A loaded KHR_gaussian_splatting scene (`B.load_scene`) made resident: each primitive is decoded on the GPU
        (`bgs_cloud_upload_khr`) into one cloud at its SH degree, f32 or f16, which every node placing it shares (a mesh
        placed by k nodes is one cloud and k entities).  Each handle's Aabb comes from the primitive's POSITION values.
        Zero-length rotations become the identity with a warning, as in the reference; a value the reference refuses
        raises BgsError (BGS_EINVAL) and leaves no cloud behind."""
        handles, zero_quats = [], []
        try:
            for prim in scene.primitives:
                h, zq, p = C.c_void_p(), C.c_uint32(), prim.to_abi()
                self._check(self._lib.bgs_cloud_upload_khr(self._ctx, C.byref(p), int(f16), C.byref(zq), C.byref(h)))
                handles.append(PlanarGaussian3dHandle._adopt(self, h, prim.n, f16, False,
                                                             aabb=compute_aabb(prim.position.array())))
                zero_quats.append(int(zq.value))
                if zq.value:
                    warnings.warn(f"mesh {prim.mesh} primitive {prim.primitive}: attribute 'KHR_gaussian_splatting:ROTATION' "
                                  f"contained {zq.value} zero-length quaternions; replacing them with identity rotations")
        except Exception:
            for h in handles:
                h.destroy()
            raise
        return SceneHandles(handles, list(scene.bundles), zero_quats)

    def save_scene(self, path, entities, cameras=(), names=None, metadata=None) -> None:
        """The reference's "G to save" for clouds resident here: `entities` (handle, settings, transform) -- e.g.
        `SceneHandles.entities()` after a selection edit, a subset or a particle step -- written by `B.write_scene` with
        `cameras` (SceneCamera), each distinct handle downloaded once.  `names` / `metadata`: per entity (default
        "cloud{j}" / the default extension values).  Gaussian4d and precomputed-covariance clouds raise ValueError."""
        from .khr import SceneExportCloud, write_scene

        entities = list(entities)
        clouds = {}
        for h, _, _ in entities:
            if is_4d_handle(h) or getattr(h, "precompute_covariance", False):
                raise ValueError("save_scene: Gaussian4d and precomputed-covariance clouds have no KHR_gaussian_splatting form")
            if h.serial not in clouds:
                clouds[h.serial] = self.download(h)
        names = names or [f"cloud{j}" for j in range(len(entities))]
        metadata = metadata or [None] * len(entities)
        write_scene(path, [SceneExportCloud(clouds[h.serial], nm, st, tr, md)
                           for (h, st, tr), nm, md in zip(entities, names, metadata)], cameras)

    def _check(self, st: int):
        if st != abi.BGS_OK:
            raise abi.BgsError(st, (self._lib.bgs_last_error(self._ctx) or b"").decode())

    @staticmethod
    def cloud_uniform(settings: CloudSettings, transform: CloudTransform | None = None, aabb=None) -> abi.bgs_cloud_uniform:
        """extract_gaussians (src/render/mod.rs:1056-1072); `aabb` = (min, max) of the entity's Aabb."""
        u = abi.bgs_cloud_uniform()
        lo, hi = aabb if aabb is not None else (np.zeros(3, np.float32), np.ones(3, np.float32))
        u.aabb_min[:] = [float(lo[0]), float(lo[1]), float(lo[2]), 1.0]
        u.aabb_max[:] = [float(hi[0]), float(hi[1]), float(hi[2]), 1.0]
        m = (transform.matrix if transform is not None else np.eye(4, dtype=np.float32)).astype(np.float32)
        u.transform[:] = m.T.reshape(-1).tolist()
        u.global_opacity = settings.global_opacity
        u.global_scale = settings.global_scale
        u.color_space = int(settings.color_space)
        u.time = settings.time
        return u

    # -- the per-view, per-frame call
    def render_view(self, handle: PlanarGaussian3dHandle, settings: CloudSettings, view: View,
                    camera: GaussianCamera | None = None, transform: CloudTransform | None = None,
                    fmt: str = "rgba32f", out: np.ndarray | None = None, to_host: bool = True,
                    asynchronous: bool = False, premultiplied: bool = False, blend_over: bool = False,
                    previous_view: View | None = None, delta_time: float | None = None, scene_depth=None):
        """Returns the (H, W, 4) frame (host) or None when `to_host` is False / the camera is warming up.
        `scene_depth`: the view's Depth32Float depth buffer on this GPU (see `scene_depth_arg`); splats behind it are
        hidden, as the reference's GreaterEqual depth test hides them (bgs_render_depth_test).  When its interface names
        a stream (v3), the frame waits on the device for the work queued there; without one the buffer must be complete
        when the call is made.  It must stay unchanged until an asynchronous frame completes.
        `asynchronous`: only enqueue the frame (BGS_FLAG_ASYNC); call `sync()` before reading anything.
        `premultiplied`: the splat layer alone, (C, 1 - T) (BGS_FLAG_PREMULTIPLIED_OUT).  `blend_over`: blend over what
        the context's frame already holds -- the previous call's result (BGS_FLAG_BLEND_OVER_TARGET): one call per
        cloud, far cloud first, like the reference's Transparent3d items (render/mod.rs:398-452, :944-948).
        `previous_view` / `delta_time`: RasterizeMode.OpticalFlow's camera of the previous frame and the seconds since
        it (the other modes ignore them); RasterizeMode.Classification reads `settings.num_classes`."""
        if camera is not None and camera.warmup:   # queue_gaussians skips warm-up cameras (render/mod.rs:361-371)
            return None
        code, dtype, ch = self.FORMATS[fmt]
        v = view.to_abi()
        u, s, ex = self._call_args(handle, settings, transform, asynchronous, premultiplied, blend_over, previous_view, delta_time)
        if to_host:
            if out is None:
                out = np.empty((view.height, view.width, ch), dtype)
            assert out.dtype == dtype and out.size == view.height * view.width * ch and out.flags.c_contiguous
        target = _ptr(out) if to_host else None
        zd = self._scene_depth(scene_depth, view)
        if getattr(handle, "temporal", False):
            st = self._render_4d(handle, v, u, s, ex, zd, settings, target, code, 0)
        elif zd is not None:
            st = self._lib.bgs_render_depth_test(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s),
                                                 None if ex is None else C.byref(ex), C.byref(zd), target, code, 0)
        elif ex is None:
            st = self._lib.bgs_render(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s), target, code, 0)
        else:
            st = self._lib.bgs_render_ex(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s), C.byref(ex), target, code, 0)
        self._check(st)
        return out if to_host else None

    def render_scene(self, entities, view: View, fmt: str = "rgba32f", scene_depth=None, previous_view: View | None = None,
                     delta_time: float | None = None, asynchronous: bool = False, premultiplied: bool = False,
                     blend_over: bool = False, out: np.ndarray | None = None) -> np.ndarray:
        """Every entity of one view in ONE frame (`bgs_render_scene`): `entities` is a sequence of (handle, CloudSettings,
        CloudTransform or None), the Bevy world's cloud entities.  Their splats share one depth sort, so clouds that
        interpenetrate are blended splat by splat instead of one painted over the other.  Each entity's global_opacity,
        global_scale, color_space, transform and handle.aabb go to its own uniform; every other settings field is the
        frame's and must agree across entities (`check_scene_entities`, ValueError before any call).  The other arguments
        are `render_view`'s.  Returns the (H, W, 4) host frame.
        A list with a PlanarGaussian4dHandle goes to `bgs_render_scene_4d`: each entity's time, time_start, time_stop,
        time_scale and playback_mode are its own, a 4D entity's gaussian_mode is Gaussian4d and the others' must agree
        (`check_scene_entities_4d`)."""
        entities = list(entities)
        temporal = any(is_4d_handle(h) for h, _, _ in entities)
        settings = check_scene_entities_4d(entities) if temporal else check_scene_entities(entities)
        code, dtype, ch = self.FORMATS[fmt]
        v = view.to_abi()
        _, s, ex = self._call_args(entities[0][0], settings, entities[0][2], asynchronous, premultiplied, blend_over,
                                   previous_view, delta_time)
        k = len(entities)
        clouds = (C.c_void_p * k)(*[h._h.value for h, _, _ in entities])
        unis = (abi.bgs_cloud_uniform * k)(*[self.cloud_uniform(st, tr, h.aabb) for h, st, tr in entities])
        if out is None:
            out = np.empty((view.height, view.width, ch), dtype)
        assert out.dtype == dtype and out.size == view.height * view.width * ch and out.flags.c_contiguous
        zd = self._scene_depth(scene_depth, view)
        if temporal:
            windows = (abi.bgs_time_window * k)(*[abi.bgs_time_window(float(st.time_start), float(st.time_stop)) for _, st, _ in entities])
            self._check(self._lib.bgs_render_scene_4d(self._ctx, clouds, unis, windows, k, C.byref(v), C.byref(s),
                                                      None if ex is None else C.byref(ex), None if zd is None else C.byref(zd),
                                                      _ptr(out), code, 0))
            return out
        self._check(self._lib.bgs_render_scene(self._ctx, clouds, unis, k, C.byref(v), C.byref(s), None if ex is None else C.byref(ex),
                                               None if zd is None else C.byref(zd), _ptr(out), code, 0))
        return out

    def render_entities(self, entities, view: View, fmt: str = "rgba32f", scene_depth=None, previous_view: View | None = None,
                        delta_time: float | None = None, asynchronous: bool = False, premultiplied: bool = False,
                        blend_over: bool = False, out: np.ndarray | None = None) -> np.ndarray:
        """`render_scene` with each entity drawn with its own CloudSettings (`bgs_render_entities`): gaussian_mode,
        rasterize_mode, aabb, opacity_adaptive_radius, draw_mode, num_classes and the 4D window are per entity, so a
        highlighted selection, a Classification object or a 2DGS surface drawn with aabb share one depth-sorted frame
        with the scan around them.  visualize_bounding_box is per entity too (`bgs_render_entities_ex`'s entity flags).
        radix_sort_depth_bits (and the other sort fields) are the frame's and must agree (`check_entities`, ValueError
        before any call).  The other arguments are `render_scene`'s."""
        entities = list(entities)
        first = check_entities(entities)
        code, dtype, ch = self.FORMATS[fmt]
        if out is None:
            out = np.empty((view.height, view.width, ch), dtype)
        assert out.dtype == dtype and out.size == view.height * view.width * ch and out.flags.c_contiguous
        args = self._entities_args(entities, first, view, previous_view, delta_time, asynchronous, premultiplied, blend_over)
        zd = self._scene_depth(scene_depth, view)
        self._check(self._lib.bgs_render_entities_ex(self._ctx, *args, None if zd is None else C.byref(zd), _ptr(out), code, 0))
        return out

    def render_entities_aux(self, entities, view: View, fmt: str = "rgba32f", scene_depth=None,
                            previous_view: View | None = None, delta_time: float | None = None, premultiplied: bool = False,
                            blend_over: bool = False) -> list[np.ndarray]:
        """`render_entities`' frame and its depth and normal frames in ONE pass (`bgs_render_entities_aux`): returns
        [rgba, depth, normal], the depth and normal frames being `render_entities`' with every entity's rasterize_mode
        replaced by Depth and by Normal.  Validates like `render_entities` (`check_entities_aux`: also ValueError, before
        any call, for a Gaussian4d or precomputed-covariance cloud and a Velocity entity).  Synchronous only.
        `blend_over`: each frame over the context's previous frame of its kind (rgba: the last frame; depth / normal: the
        last aux frame's)."""
        entities = list(entities)
        first = check_entities_aux(entities)
        code, dtype, ch = self.FORMATS[fmt]
        outs = [np.empty((view.height, view.width, ch), dtype) for _ in range(3)]
        args = self._entities_args(entities, first, view, previous_view, delta_time, False, premultiplied, blend_over)
        zd = self._scene_depth(scene_depth, view)
        self._check(self._lib.bgs_render_entities_aux(self._ctx, *args, None if zd is None else C.byref(zd), *(_ptr(o) for o in outs),
                                                      code, 0))
        return outs

    def render_entities_pick(self, entities, view: View, fmt: str = "rgba32f", scene_depth=None,
                             previous_view: View | None = None, delta_time: float | None = None, premultiplied: bool = False,
                             blend_over: bool = False) -> tuple[np.ndarray, np.ndarray]:
        """`render_entities`' frame and, from the same pass, its pick frame (`bgs_render_entities_pick`): returns (rgba,
        pick), pick an (h, w) array of abi.PICK_DTYPE -- per pixel the entity and gaussian index of the pair with the
        largest blend weight w = a T, that w and the splat's depth d (BGS_PICK_NONE, 0, 0 where nothing blends).  rgba is
        byte for byte `render_entities`' frame.  Validates like `render_entities` (`check_entities`, ValueError before any
        call).  Synchronous only; `blend_over` applies to rgba only."""
        entities = list(entities)
        first = check_entities(entities)
        code, dtype, ch = self.FORMATS[fmt]
        out = np.empty((view.height, view.width, ch), dtype)
        pick = np.empty((view.height, view.width), abi.PICK_DTYPE)
        args = self._entities_args(entities, first, view, previous_view, delta_time, False, premultiplied, blend_over)
        zd = self._scene_depth(scene_depth, view)
        self._check(self._lib.bgs_render_entities_pick(self._ctx, *args, None if zd is None else C.byref(zd), _ptr(out), code, 0,
                                                       _ptr(pick)))
        return out, pick

    def render_views(self, entities, views, fmt: str = "rgba32f", scene_depths=None, asynchronous: bool = False,
                     premultiplied: bool = False, outs=None) -> list[np.ndarray]:
        """`render_entities` of every view in `views` (a sequence of View) in ONE frame (`bgs_render_views`): returns one
        (H_i, W_i, 4) host frame per view, each byte for byte `render_entities`' frame of that view.  Stereo eyes, cube-map
        faces or split-screen cameras share one key-gen, sort, projection, binning and blend.  `scene_depths`: one depth
        buffer per view (as `render_view`'s `scene_depth`), or None.  `outs`: the host frames to fill (one per view).
        `asynchronous`: only enqueue the frame; the frames are filled once `sync()` returns.  Validates with `check_views`
        (ValueError before any call)."""
        entities, views = list(entities), list(views)
        first = check_views(entities, views)
        code, dtype, ch = self.FORMATS[fmt]
        if outs is None:
            outs = [np.empty((v.height, v.width, ch), dtype) for v in views]
        assert len(outs) == len(views)
        for o, v in zip(outs, views):
            assert o.dtype == dtype and o.size == v.height * v.width * ch and o.flags.c_contiguous
        clouds, unis, ents, eflags, k, _, s, _ = self._entities_args(entities, first, views[0], None, None, asynchronous,
                                                                     premultiplied, False)
        n = len(views)
        vs = (abi.bgs_view * n)(*[v.to_abi() for v in views])
        zds = None
        if scene_depths is not None:
            assert len(scene_depths) == n
            zds = (abi.bgs_scene_depth * n)(*[self._scene_depth(d, v) for d, v in zip(scene_depths, views)])
        targets = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        self._check(self._lib.bgs_render_views(self._ctx, clouds, unis, ents, eflags, k, vs, n, s, zds, targets, code, 0))
        return outs

    def render_views_aux(self, entities, views, fmt: str = "rgba32f", scene_depths=None, premultiplied: bool = False,
                         outs=None) -> list[list[np.ndarray]]:
        """`render_entities_aux` of every view in `views` in ONE frame (`bgs_render_views_aux`): returns [rgba, depth,
        normal] per view, each byte for byte `render_entities_aux`' frames of that view.  Entities in Depth mode are drawn
        over each view's own depth range.  `scene_depths`: one depth buffer per view, or None.  `outs`: the host frames to
        fill, [[rgba, depth, normal] per view].  Synchronous only.  Validates with `check_views_aux` (ValueError before any
        call)."""
        entities, views = list(entities), list(views)
        first = check_views_aux(entities, views)
        code, dtype, ch = self.FORMATS[fmt]
        if outs is None:
            outs = [[np.empty((v.height, v.width, ch), dtype) for _ in range(3)] for v in views]
        assert len(outs) == len(views)
        for trio, v in zip(outs, views):
            assert len(trio) == 3
            for o in trio:
                assert o.dtype == dtype and o.size == v.height * v.width * ch and o.flags.c_contiguous
        clouds, unis, ents, eflags, k, _, s, _ = self._entities_args(entities, first, views[0], None, None, False,
                                                                     premultiplied, False)
        n = len(views)
        vs = (abi.bgs_view * n)(*[v.to_abi() for v in views])
        zds = None
        if scene_depths is not None:
            assert len(scene_depths) == n
            zds = (abi.bgs_scene_depth * n)(*[self._scene_depth(d, v) for d, v in zip(scene_depths, views)])
        targets = [(C.c_void_p * n)(*[trio[f].ctypes.data for trio in outs]) for f in range(3)]
        self._check(self._lib.bgs_render_views_aux(self._ctx, clouds, unis, ents, eflags, k, vs, n, s, zds, *targets, code, 0))
        return outs

    def _entities_args(self, entities, first, view, previous_view, delta_time, asynchronous, premultiplied, blend_over):
        """(clouds, uniforms, entities, entity flags, k, view, frame, extras) of a bgs_render_entities_ex or _aux call."""
        v = view.to_abi()
        s = first.to_abi()
        s.flags &= ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX   # (each entity's own, below)
        s.flags |= ((abi.BGS_FLAG_ASYNC if asynchronous else 0) | (abi.BGS_FLAG_PREMULTIPLIED_OUT if premultiplied else 0)
                    | (abi.BGS_FLAG_BLEND_OVER_TARGET if blend_over else 0))
        ex = None
        if previous_view is not None:
            ex = abi.bgs_render_extras(num_classes=1, delta_time=float(delta_time) if delta_time is not None else 0.0)
            ex.previous_clip_from_world[:] = previous_view.to_abi().clip_from_world[:]
        k = len(entities)
        eflags = (C.c_uint32 * k)(*[abi.BGS_ENTITY_VISUALIZE_BOUNDING_BOX if st.visualize_bounding_box else 0
                                    for _, st, _ in entities])
        clouds = (C.c_void_p * k)(*[h._h.value for h, _, _ in entities])
        unis = (abi.bgs_cloud_uniform * k)(*[self.cloud_uniform(st, tr, h.aabb) for h, st, tr in entities])
        ents = (abi.bgs_entity_settings * k)(*[entity_settings(st) for _, st, _ in entities])
        return clouds, unis, ents, eflags, k, C.byref(v), C.byref(s), None if ex is None else C.byref(ex)

    def _render_4d(self, handle, v, u, s, ex, zd, settings, target, code, is_device):
        return self._lib.bgs_render_4d(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s), None if ex is None else C.byref(ex),
                                       None if zd is None else C.byref(zd), target, code, is_device, float(settings.time_start),
                                       float(settings.time_stop))

    def _scene_depth(self, scene_depth, view):
        """The call's bgs_scene_depth; a buffer whose interface names its producer's stream is read only after the work
        queued on that stream so far (every launch of a frame is ordered after the context's stream)."""
        zd, producer = scene_depth_arg(scene_depth, view.width, view.height)
        if producer is not None:
            _stream_wait(self.stream_ptr, int(producer))
        return zd

    def _uniform_and_settings(self, handle, settings, transform, asynchronous=False, premultiplied=False, blend_over=False):
        """The uniform and settings structs of a call (see `_call_args`)."""
        return self._call_args(handle, settings, transform, asynchronous, premultiplied, blend_over)[:2]

    def _call_args(self, handle, settings, transform, asynchronous=False, premultiplied=False, blend_over=False,
                   previous_view=None, delta_time=None):
        """The uniform, settings and extras of a call; cached while (settings, transform, cloud, flags, extras) repeat
        from frame to frame.  The extras are None -- bgs_render, i.e. bgs_render_ex's NULL -- when they would say what NULL
        says: no previous view and num_classes = 1."""
        prev = None if previous_view is None else bytes(previous_view.to_abi().clip_from_world)
        key = (dataclasses.astuple(settings), None if transform is None else transform.matrix.tobytes(), asynchronous, handle.serial,
               premultiplied, blend_over, prev, delta_time)
        if getattr(self, "_us_cache", (None,))[0] != key:
            s_ = settings.to_abi()
            if asynchronous:
                s_.flags |= abi.BGS_FLAG_ASYNC
            if premultiplied:
                s_.flags |= abi.BGS_FLAG_PREMULTIPLIED_OUT
            if blend_over:
                s_.flags |= abi.BGS_FLAG_BLEND_OVER_TARGET
            ex = None
            if prev is not None or settings.num_classes != 1:
                ex = abi.bgs_render_extras(num_classes=int(settings.num_classes))
                if prev is not None:
                    ex.previous_clip_from_world[:] = previous_view.to_abi().clip_from_world[:]
                    ex.delta_time = float(delta_time) if delta_time is not None else 0.0
            self._us_cache = (key, self.cloud_uniform(settings, transform, handle.aabb), s_, ex)
        return self._us_cache[1], self._us_cache[2], self._us_cache[3]

    def render_view_aux(self, handle: PlanarGaussian3dHandle, settings: CloudSettings, view: View,
                        transform: CloudTransform | None = None, fmt: str = "rgba32f", scene_depth=None):
        """Colour, depth and normal frames of one view in ONE pass (`bgs_render_aux`, BASELINE.json config 4).
        `scene_depth` (as in `render_view`): the three frames depth-tested against it, through `bgs_render_entities_aux`
        with this one entity (the same frames `bgs_render_aux` draws, with the depth test)."""
        code, dtype, ch = self.FORMATS[fmt]
        v = view.to_abi()
        u = self.cloud_uniform(settings, transform, handle.aabb)
        s = settings.to_abi()
        outs = [np.empty((view.height, view.width, ch), dtype) for _ in range(3)]
        if scene_depth is None:
            st = self._lib.bgs_render_aux(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s), _ptr(outs[0]), _ptr(outs[1]),
                                          _ptr(outs[2]), code, 0)
        else:
            zd = self._scene_depth(scene_depth, view)
            e = entity_settings(settings)
            st = self._lib.bgs_render_entities_aux(self._ctx, (C.c_void_p * 1)(handle._h.value), C.byref(u), C.byref(e), None, 1,
                                                   C.byref(v), C.byref(s), None, C.byref(zd), *(_ptr(o) for o in outs), code, 0)
        self._check(st)
        return outs

    def render_view_to_device(self, handle: PlanarGaussian3dHandle, settings: CloudSettings, view: View, device_ptr: int,
                              transform: CloudTransform | None = None, fmt: str = "rgba8_srgb", asynchronous: bool = False,
                              premultiplied: bool = False, blend_over: bool = False, previous_view: View | None = None,
                              delta_time: float | None = None, scene_depth=None) -> None:
        """Render straight into caller-owned device memory: an exported frame target (`bgs_frame_export_create`), or
        another GPU's memory mapped into this process (`bgs_peer_buffer_open`) -- the blend kernel's pixel stores then
        travel over NVLink themselves.  The target must be aligned to one pixel (4 / 8 / 16 bytes).  `premultiplied` /
        `blend_over`, `previous_view`, `delta_time` and `scene_depth` as in `render_view`; blend-over reads what
        `device_ptr` holds."""
        code, _, _ = self.FORMATS[fmt]
        v = view.to_abi()
        u, s, ex = self._call_args(handle, settings, transform, asynchronous, premultiplied, blend_over, previous_view, delta_time)
        zd = self._scene_depth(scene_depth, view)
        if getattr(handle, "temporal", False):
            self._check(self._render_4d(handle, v, u, s, ex, zd, settings, C.c_void_p(device_ptr), code, 1))
        elif zd is not None:
            self._check(self._lib.bgs_render_depth_test(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s),
                                                        None if ex is None else C.byref(ex), C.byref(zd),
                                                        C.c_void_p(device_ptr), code, 1))
        elif ex is None:
            self._check(self._lib.bgs_render(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s), C.c_void_p(device_ptr), code, 1))
        else:
            self._check(self._lib.bgs_render_ex(self._ctx, handle._h, C.byref(v), C.byref(u), C.byref(s), C.byref(ex),
                                                C.c_void_p(device_ptr), code, 1))

    def sync(self) -> bool:
        """Complete the frames enqueued with `asynchronous=True`.  False = the last frame must be rendered again
        (its pair list outgrew the buffer, which has been grown)."""
        st = self._lib.bgs_sync(self._ctx)
        if st == abi.BGS_NOT_READY:
            return False
        self._check(st)
        return True

    # -- selection: the visibility lane DrawMode::Selected / HighlightSelected read, edited in place (no re-upload)
    def select_sparse(self, handle: PlanarGaussian3dHandle, query: SparseSelect | None = None) -> int:
        """SparseSelect (src/query/sparse.rs:24-54) on the GPU: visibility 1 where fewer than `neighbor_threshold`
        gaussians (itself included) lie within `radius`, else 0 (the exact rule: include/bgs.h).  Returns how many
        were selected.  The debug hooks and frame stats are not ready again until the next render."""
        q = query if query is not None else SparseSelect()
        sel = C.c_uint32()
        self._check(self._lib.bgs_cloud_select_sparse(self._ctx, handle._h, C.c_float(q.radius), C.c_uint32(q.neighbor_threshold),
                                                      C.byref(sel)))
        return int(sel.value)

    def select_in_mesh(self, handle: PlanarGaussian3dHandle, vertices, indices, mesh_from_cloud=None, mode: str = "replace") -> int:
        """Point-in-mesh selection (src/query/raycast.rs:54-124) on the GPU: a gaussian is inside when the +x ray from
        mesh_from_cloud * position hits an odd number of triangles (the exact rule: include/bgs.h).  vertices (nv, 3)
        float32, indices (nt, 3) uint32, mesh_from_cloud a 4x4 (row-major numpy, i.e. M @ p; None = identity).
        mode "replace": visibility 1 inside, 0 elsewhere; "add": 1 inside, the rest untouched.  Returns how many are inside."""
        modes = {"replace": abi.BGS_SELECT_REPLACE, "add": abi.BGS_SELECT_ADD}
        if mode not in modes:
            raise ValueError(f"mode must be one of {sorted(modes)}")
        v = np.ascontiguousarray(vertices, np.float32)
        i = np.ascontiguousarray(indices, np.uint32)
        if v.ndim != 2 or v.shape[1] != 3:
            raise ValueError("vertices must have shape (nv, 3)")
        if i.ndim != 2 or i.shape[1] != 3:
            raise ValueError("indices must have shape (nt, 3)")
        m = None
        if mesh_from_cloud is not None:
            m = np.asarray(mesh_from_cloud, np.float32)
            if m.shape != (4, 4):
                raise ValueError("mesh_from_cloud must be 4x4")
            m = np.ascontiguousarray(m.T)                     # column-major for the C ABI
        inside = C.c_uint32()
        self._check(self._lib.bgs_cloud_select_in_mesh(self._ctx, handle._h, _ptr(v), len(v), _ptr(i), len(i),
                                                       None if m is None else _ptr(m), modes[mode], C.byref(inside)))
        return int(inside.value)

    def select_in_view(self, handle: PlanarGaussian3dHandle, view: View, mask, transform: CloudTransform | None = None,
                       mode: str = "replace") -> int:
        """Rectangle, lasso and brush selection through the volume (`bgs_cloud_select_in_view`): a gaussian is inside when
        the projection with `transform` and `view` finds it in the frustum and the mask pixel under its centre is set (the
        exact rule: include/bgs.h).  `mask`: an (h, w) bool / uint8 numpy array, or an object with
        `__cuda_array_interface__` of that shape and type in device memory (read after its producer stream's work, as
        `scene_depth` is).  mode "replace": visibility 1 inside, 0 elsewhere; "add": 1 inside, the rest untouched.
        Returns how many are inside."""
        modes = {"replace": abi.BGS_SELECT_REPLACE, "add": abi.BGS_SELECT_ADD}
        if mode not in modes:
            raise ValueError(f"mode must be one of {sorted(modes)}")
        shape = (view.height, view.width)
        cai = getattr(mask, "__cuda_array_interface__", None)
        if cai is not None:
            if np.dtype(cai["typestr"]) not in (np.dtype(np.uint8), np.dtype(np.bool_)):
                raise TypeError(f"mask must be bool or uint8, not {cai['typestr']}")
            if tuple(cai["shape"]) != shape:
                raise ValueError(f"mask must have shape {shape}, not {tuple(cai['shape'])}")
            strides = cai.get("strides")
            if strides is not None and tuple(strides) != (view.width, 1):
                raise ValueError("mask must be C-contiguous")
            if cai.get("stream") is not None:
                _stream_wait(self.stream_ptr, int(cai["stream"]))
            ptr, is_device, keep = C.c_void_p(int(cai["data"][0])), 1, mask
        else:
            m = np.asarray(mask)
            if m.dtype not in (np.dtype(np.uint8), np.dtype(np.bool_)):
                raise TypeError(f"mask must be bool or uint8, not {m.dtype}")
            if m.shape != shape:
                raise ValueError(f"mask must have shape {shape}, not {m.shape}")
            keep = np.ascontiguousarray(m).view(np.uint8)
            ptr, is_device = _ptr(keep), 0
        u = self.cloud_uniform(CloudSettings(), transform, handle.aabb)
        v = view.to_abi()
        inside = C.c_uint32()
        self._check(self._lib.bgs_cloud_select_in_view(self._ctx, handle._h, C.byref(u), C.byref(v), ptr, is_device, modes[mode],
                                                       C.byref(inside)))
        del keep
        return int(inside.value)

    def select_picked(self, entities, pick: np.ndarray, mask=None, min_weight: float = 0.0, mode: str = "replace") -> int:
        """Select what a pick frame shows (host-side, over `set_visibility`): for each distinct handle among `entities`
        (the list `render_entities_pick` rendered), the gaussians picked at the pixels where `mask` ((h, w) bool; None:
        every pixel) is set, with weight >= min_weight.  Instances of one cloud select into that one cloud.  mode
        "replace": each handle's visibility 1 at its picked gaussians, 0 elsewhere; "add": 1 there, the rest untouched.
        Returns how many distinct (cloud, gaussian) pairs were picked."""
        if mode not in ("replace", "add"):
            raise ValueError("mode must be one of ['add', 'replace']")
        entities = list(entities)
        pick = np.asarray(pick)
        if pick.dtype != abi.PICK_DTYPE or pick.ndim != 2:
            raise ValueError("pick must be an (h, w) array of PICK_DTYPE")
        sel = (pick["entity"] != abi.BGS_PICK_NONE) & (pick["weight"] >= np.float32(min_weight))
        if mask is not None:
            mask = np.asarray(mask, bool)
            if mask.shape != pick.shape:
                raise ValueError(f"mask must have shape {pick.shape}, not {mask.shape}")
            sel &= mask
        ent, idx = pick["entity"][sel], pick["index"][sel]
        if ent.size and int(ent.max()) >= len(entities):
            raise ValueError(f"pick names entity {int(ent.max())}, but {len(entities)} entities were given")
        handles = []
        for h, _, _ in entities:
            if not any(h is o for o in handles):
                handles.append(h)
        total = 0
        for h in handles:
            js = [j for j, (e, _, _) in enumerate(entities) if e is h]
            mine = np.unique(idx[np.isin(ent, js)])
            total += mine.size
            vis = np.zeros(h.n, np.float32) if mode == "replace" else self.visibility(h)
            vis[mine] = 1.0
            self.set_visibility(h, vis)
        return total

    def visibility(self, handle: PlanarGaussian3dHandle) -> np.ndarray:
        """The visibility lane of every gaussian, (n,) float32."""
        out = np.empty(handle.n, np.float32)
        self._check(self._lib.bgs_cloud_visibility_get(self._ctx, handle._h, _ptr(out)))
        return out

    def set_visibility(self, handle: PlanarGaussian3dHandle, vis) -> None:
        vis = np.ascontiguousarray(vis, np.float32)
        if vis.shape != (handle.n,):
            raise ValueError(f"visibility must have shape ({handle.n},)")
        self._check(self._lib.bgs_cloud_visibility_set(self._ctx, handle._h, _ptr(vis)))

    def apply_selection(self, handle: PlanarGaussian3dHandle, indices) -> None:
        """src/query/select.rs:81-110: visibility 0 everywhere, 1 at `indices`."""
        idx = np.asarray(indices).reshape(-1)
        if idx.size and (idx.dtype.kind not in "iu" or idx.min() < 0 or idx.max() >= handle.n):
            raise IndexError(f"selection indices must be integers in [0, {handle.n})")
        vis = np.zeros(handle.n, np.float32)
        vis[idx] = 1.0
        self.set_visibility(handle, vis)

    def invert_selection(self, handle: PlanarGaussian3dHandle) -> None:
        """src/query/select.rs:116-150 on a 0/1 lane: visibility == 0.0 becomes 1, everything else 0."""
        self.set_visibility(handle, (self.visibility(handle) == 0.0).astype(np.float32))

    def selection(self, handle: PlanarGaussian3dHandle) -> np.ndarray:
        """Indices of the selected gaussians: visibility >= 0.5, the ones DrawMode::Selected draws."""
        return np.flatnonzero(self.visibility(handle) >= 0.5).astype(np.uint32)

    # -- keeping a selection as its own cloud, reading clouds back (src/query/select.rs:156-176; the rule: include/bgs.h)
    def subset(self, handle: PlanarGaussian3dHandle, indices=None) -> PlanarGaussian3dHandle | None:
        """A new resident cloud of `handle`'s gaussians, in its layout.  indices None: the selected ones, visibility
        !(w < 0.5) -- the set DrawMode::Selected draws, NaN included (unlike `selection()`) -- in index order; None when
        nothing is selected.  Otherwise gaussian j of the result is gaussian indices[j] (order kept, repeats allowed)."""
        out, n = C.c_void_p(), C.c_uint32()
        if indices is None:
            self._check(self._lib.bgs_cloud_subset(self._ctx, handle._h, None, 0, C.byref(out), C.byref(n)))
        else:
            idx = np.asarray(indices).reshape(-1)
            if idx.dtype.kind not in "iu" or (idx.size and (idx.min() < 0 or idx.max() >= 1 << 32)):
                raise IndexError("subset: indices must be non-negative integers")
            idx = np.ascontiguousarray(idx, np.uint32)
            self._check(self._lib.bgs_cloud_subset(self._ctx, handle._h, _ptr(idx), idx.size, C.byref(out), C.byref(n)))
        if not out:
            return None
        return type(handle)._adopt(self, out, int(n.value), handle.f16, handle.precompute_covariance)

    def download_planes(self, handle: PlanarGaussian3dHandle) -> tuple[np.ndarray, ...]:
        """The cloud's planes as the matching upload call takes them: f32 (pos_vis, sh (n, S_d), rotation,
        scale_opacity); f16 and precomputed-covariance clouds (pos_vis, sh_packed (n, S_d / 2), second plane words)."""
        pos = np.empty((handle.n, 4), np.float32)
        if getattr(handle, "temporal", False):   # (pos_vis, sh, rotations, scale_opacity, timestamp_timescale)
            planes = (pos, np.empty((handle.n, 144), np.float32), np.empty((handle.n, 8), np.float32),
                      np.empty((handle.n, 4), np.float32), np.empty((handle.n, 4), np.float32))
            self._check(self._lib.bgs_cloud_download_4d(self._ctx, handle._h, *(_ptr(a) for a in planes)))
            return planes
        width = SH_WIDTHS[handle.sh_degree]
        if handle.f16 or handle.precompute_covariance:
            sh, second = np.empty((handle.n, width // 2), np.uint32), np.empty((handle.n, 4), np.uint32)
            self._check(self._lib.bgs_cloud_download_f16_sh(self._ctx, handle._h, _ptr(pos), _ptr(sh), _ptr(second)))
            return pos, sh, second
        sh, rot, so = np.empty((handle.n, width), np.float32), np.empty((handle.n, 4), np.float32), np.empty((handle.n, 4), np.float32)
        self._check(self._lib.bgs_cloud_download_f32_sh(self._ctx, handle._h, _ptr(pos), _ptr(sh), _ptr(rot), _ptr(so)))
        return pos, sh, rot, so

    def download(self, handle: PlanarGaussian3dHandle) -> PlanarGaussian3d:
        """The cloud as a host PlanarGaussian3d: f16 planes widened to f32 (`PlanarGaussian3d.from_f16`); a
        precomputed-covariance cloud holds its covariance in the slots `precomputed_covariance()` uses."""
        planes = self.download_planes(handle)
        if len(planes) == 5:
            return PlanarGaussian4d(*planes)
        return PlanarGaussian3d.from_f16(*planes) if len(planes) == 3 else PlanarGaussian3d(*planes)

    def save_selection(self, handle: PlanarGaussian3dHandle, path) -> int:
        """The reference's save_selection (src/query/select.rs:156-176): the selected gaussians (`subset(handle)`)
        written to `path` as .gcloud or .ply by its extension.  Returns how many were written.  A precomputed-covariance
        cloud raises ValueError (its rotation and scale are gone, and the file holds those).  Nothing selected raises
        ValueError and writes nothing, where the reference would write an empty cloud."""
        from .gcloud import write_gcloud
        from .io import write_ply_3d

        ext = os.path.splitext(str(path))[1].lower()
        writers = {".gcloud": write_gcloud, ".ply": write_ply_3d}
        if ext not in writers:
            raise ValueError("save_selection: only .ply and .gcloud supported")
        if handle.precompute_covariance:
            raise ValueError("save_selection: a precomputed-covariance cloud has no rotation and scale to save")
        sub = self.subset(handle)
        if sub is None:
            raise ValueError("save_selection: nothing is selected")
        try:
            writers[ext](path, self.download(sub))
            return sub.n
        finally:
            sub.destroy()

    # -- particle behaviours (src/morph/particle.rs): an enqueued per-frame edit of the positions (the rule: include/bgs.h)
    def add_particles(self, behaviors) -> ParticleBehaviorsHandle:
        """Upload a ParticleBehaviors array (PARTICLE_BEHAVIOR_DTYPE records).  Duplicate active indices are refused."""
        return ParticleBehaviorsHandle(self, behaviors)

    def step_particles(self, handle: PlanarGaussian3dHandle, particles: ParticleBehaviorsHandle, delta_time: float) -> None:
        """One step of every behaviour over `delta_time` seconds, enqueued on this context: frames rendered before it
        (on any context) see the old positions, everything after it the new ones.  `sync()` completes it."""
        self._check(self._lib.bgs_cloud_particles_step(self._ctx, handle._h, particles._h, C.c_float(delta_time)))

    def positions(self, handle: PlanarGaussian3dHandle) -> np.ndarray:
        """The position plane, (n, 4) float32 (x, y, z, visibility), after every step queued on the cloud."""
        out = np.empty((handle.n, 4), np.float32)
        self._check(self._lib.bgs_cloud_positions_get(self._ctx, handle._h, _ptr(out)))
        return out

    # -- interpolation (src/morph/interpolate.rs): an enqueued per-frame blend of two clouds (the rule: include/bgs.h)
    def interpolate(self, out: PlanarGaussian3dHandle, lhs: PlanarGaussian3dHandle, rhs: PlanarGaussian3dHandle,
                    settings: CloudSettings) -> None:
        """`out` := the blend of `lhs` and `rhs` at `settings.time` between `settings.time_start` and `time_stop`,
        enqueued on this context: frames rendered before it (on any context) see the old `out`, everything after it the
        blend.  The three clouds hold the same number of gaussians in one layout; make `out` once as
        `subset(lhs, np.arange(lhs.n))`.  `sync()` completes it."""
        self._check(self._lib.bgs_cloud_interpolate(self._ctx, out._h, lhs._h, rhs._h, C.c_float(settings.time),
                                                    C.c_float(settings.time_start), C.c_float(settings.time_stop)))

    # -- transforms and bounds: a gizmo drag baked into the cloud, and its Aabb refreshed (the rule: include/bgs.h)
    def transform(self, handle: PlanarGaussian3dHandle, matrix, selected: bool = False) -> None:
        """Bake the similarity transform `matrix` (a 4x4 in CloudTransform.matrix's convention, or a CloudTransform),
        in the cloud's own frame, into every gaussian or, `selected`, the selected ones (visibility !(v < 0.5)):
        positions, rotations, scales or covariances, and SH bands 1-3.  Enqueued like `step_particles`: frames rendered
        before it (on any context) see the old cloud, everything after it the new one.  A world-space delta W of an
        entity with model matrix `model` is `inv(model) @ W @ model` here.  Shear, non-uniform scale, reflections and
        Gaussian4d clouds raise BgsError (BGS_EINVAL).  handle.aabb is not updated: call `update_aabb`."""
        m = matrix.matrix if isinstance(matrix, CloudTransform) else matrix
        m = np.asarray(m, np.float32)
        if m.shape != (4, 4):
            raise ValueError(f"transform: the matrix must be 4x4, not {m.shape}")
        cm = np.ascontiguousarray(m.T.reshape(16))
        mode = abi.BGS_TRANSFORM_SELECTED if selected else abi.BGS_TRANSFORM_ALL
        self._check(self._lib.bgs_cloud_transform(self._ctx, handle._h, _ptr(cm), mode))

    def bounds(self, handle: PlanarGaussian3dHandle, selected: bool = False) -> tuple[np.ndarray, np.ndarray, int]:
        """(min (3,) f32, max (3,) f32, count) of the positions of every gaussian, or of the selected ones, whose x, y
        and z are finite, after every write queued on the cloud; (+inf, -inf, 0) for none."""
        lo, hi, n = np.empty(3, np.float32), np.empty(3, np.float32), C.c_uint32()
        mode = abi.BGS_TRANSFORM_SELECTED if selected else abi.BGS_TRANSFORM_ALL
        self._check(self._lib.bgs_cloud_bounds(self._ctx, handle._h, mode, _ptr(lo), _ptr(hi), C.byref(n)))
        return lo, hi, int(n.value)

    def update_aabb(self, handle: PlanarGaussian3dHandle) -> tuple[np.ndarray, np.ndarray]:
        """handle.aabb := the entity's Aabb from the GPU bounds of every finite position, through compute_aabb's f32
        steps (for finite positions, bit for bit compute_aabb(positions(handle))).  Returns it."""
        lo, hi, _ = self.bounds(handle)
        handle.aabb = aabb_of_extent(lo, hi)
        return handle.aabb

    # -- parity / measurement hooks
    def frame_stats(self) -> abi.bgs_frame_stats:
        fs = abi.bgs_frame_stats()
        self._check(self._lib.bgs_frame_stats_get(self._ctx, C.byref(fs)))
        return fs

    def stage_times_us(self) -> np.ndarray:
        arr = (C.c_float * 6)()
        self._check(self._lib.bgs_stage_times_us(self._ctx, C.byref(arr)))
        return np.array(list(arr), np.float32)

    def sorted_entries(self) -> np.ndarray:
        n = self.frame_stats().n
        out = np.empty((n, 2), np.uint32)
        self._check(self._lib.bgs_debug_sorted_entries(self._ctx, _ptr(out)))
        return out

    def tile_ranges(self) -> np.ndarray:
        fs = self.frame_stats()
        out = np.empty((fs.tiles_x * fs.tiles_y, 2), np.uint32)
        self._check(self._lib.bgs_debug_tile_ranges(self._ctx, _ptr(out)))
        return out

    def tile_entries(self) -> np.ndarray:
        fs = self.frame_stats()
        out = np.empty((fs.n_pairs,), np.uint32)
        if fs.n_pairs:
            self._check(self._lib.bgs_debug_tile_entries(self._ctx, _ptr(out), fs.n_pairs))
        return out

    def projected(self):
        fs = self.frame_stats()
        rec = np.empty((fs.n_visible, 12), np.float32)
        ids = np.empty((fs.n_visible,), np.uint32)
        if fs.n_visible:
            self._check(self._lib.bgs_debug_projected(self._ctx, _ptr(rec), _ptr(ids)))
        return rec, ids

    def splat_depths(self) -> np.ndarray:
        """The last depth-tested frame's splat depths d, (n_visible,) float32 in front-to-back rank order."""
        fs = self.frame_stats()
        out = np.empty((fs.n_visible,), np.float32)
        if fs.n_visible:
            self._check(self._lib.bgs_debug_splat_depths(self._ctx, _ptr(out)))
        return out

    @property
    def stream_ptr(self) -> int:
        return int(self._lib.bgs_context_stream(self._ctx) or 0)

    @property
    def copy_stream_ptr(self) -> int:
        return int(self._lib.bgs_context_copy_stream(self._ctx) or 0)

    @property
    def frame_device_ptr(self) -> int:
        return int(self._lib.bgs_frame_device_ptr(self._ctx) or 0)

    @property
    def last_launch_count(self) -> int:
        return int(self._lib.bgs_last_launch_count(self._ctx))

    def destroy(self):
        if self._ctx:
            self._lib.bgs_context_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass
