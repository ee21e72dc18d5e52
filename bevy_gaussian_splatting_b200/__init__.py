"""bevy_gaussian_splatting_b200 -- H100-native (sm_90a) forward splat path behind the reference's plugin surface.

Product = `csrc/` (hand-written sm_90a kernels + the C ABI of include/bgs.h, built to libbgs.so).
The Python modules here are the host-side mirror of the reference interface for this path
(same names as mosure/bevy_gaussian_splatting: src/lib.rs:7-29 re-exports) used by tests and bench.
"""
from .abi import PICK_DTYPE, BgsError  # noqa: F401
from .camera import GaussianCamera, View, headless_view, orbit_view, perspective_view  # noqa: F401
from .gaussian import (PlanarGaussian3d, PlanarGaussian4d, random_gaussians_3d, random_gaussians_3d_seeded,  # noqa: F401
                       random_gaussians_4d_seeded, SH_COEFF_COUNT, SH_4D_COEFF_COUNT, SH_WIDTHS)
from .io import load_cloud, parse_ply_3d, parse_ply_4d, write_ply_4d  # noqa: F401
from .khr import (GaussianScene, KhrAccessor, KhrPrimitive, KhrSpec, SceneBundle, SceneCamera,  # noqa: F401
                  SceneExportCloud, load_scene, write_scene)
from .gcloud import decode_gcloud, encode_gcloud, read_gcloud, write_gcloud  # noqa: F401
from .particles import (PARTICLE_BEHAVIOR_DTYPE, PARTICLE_INACTIVE, ParticleBehaviors,  # noqa: F401
                        random_particle_behaviors)
from .plugin import (CloudTransform, GaussianSplattingPlugin, ParticleBehaviorsHandle, PlanarGaussian3dHandle,  # noqa: F401
                     PlanarGaussian4dHandle, SceneHandles, similarity_transform)
from .settings import (CloudSettings, DrawMode, GaussianColorSpace, GaussianMode, PlaybackMode,  # noqa: F401
                       RadixSortDepthBits, RasterizeMode, ShaderDefines, SortMode, SparseSelect, playback_update)
