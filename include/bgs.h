/*
 * bgs.h -- C ABI of the H100-native (sm_90a) forward splat path (libbgs.so).
 *
 * Drop-in boundary for mosure/bevy_gaussian_splatting's per-view, per-frame GPU work.
 * One Rust render-world system calls bgs_render() in place of BOTH reference call sites:
 *   - system  run_radix_sort::<R>                 (src/sort/radix.rs:616-756, scheduled :97-118)
 *   - command DrawGaussians<R> / DrawGaussianInstanced::render
 *                                                 (src/render/mod.rs:986-992, :1501-1569)
 * The Bevy plugin surface (GaussianSplattingPlugin, PlanarGaussian3dHandle, CloudSettings,
 * GaussianCamera) stays Rust; see INTEGRATION.md for the binding and the system that calls this.
 *
 * Conventions: plain pointers and sizes only; host arrays are borrowed for the duration of the
 * call; device memory is library-owned; every entry point returns a bgs_status and never
 * aborts or throws across the boundary.  A context is single-threaded (Bevy's render thread);
 * distinct contexts (one per GPU) may be used concurrently.  Matrices are column-major f32,
 * exactly as Bevy's `View` uniform / `CloudUniform` hold them.
 */
#ifndef BGS_H
#define BGS_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct bgs_context bgs_context; /* opaque, library-owned */
typedef struct bgs_cloud bgs_cloud;     /* opaque, library-owned */

typedef enum {
    BGS_OK = 0,
    BGS_NOT_READY = 1, /* maps to the reference's silent skip-frame (radix.rs:645-658, mod.rs:1533-1539) */
    BGS_EINVAL = 2,
    BGS_ECUDA = 3,
    BGS_ENOMEM = 4,
    BGS_ENCCL = 5
} bgs_status;

/* The Bevy `View` uniform fields the path reads (src/render/bindings.wgsl:3-9;
 * helpers.wgsl:18-38, transform.wgsl:6, gaussian_2d.wgsl:104, radix.wgsl:92). */
typedef struct {
    float view_from_world[16];
    float clip_from_view[16];
    float clip_from_world[16]; /* used as unjittered_clip_from_world and clip_from_world */
    float world_position[3];
    float viewport[4]; /* x, y, w, h (px); the frame is w x h */
} bgs_view;

/* CloudUniform (src/render/mod.rs:995-1009, bindings.wgsl:13-26), fields this path reads. */
typedef struct {
    float transform[16]; /* model -> world */
    float global_opacity;
    float global_scale;
    uint32_t color_space; /* GaussianColorSpace: 0 SrgbRec709Display, 1 LinRec709Display */
    float time;
    float aabb_min[4];    /* CloudUniform.min / .max = the entity's Aabb.min()/.max() extended with 1.0 */
    float aabb_max[4];    /* (render/mod.rs:1070-1071); read by RasterizeMode::Position only */
} bgs_cloud_uniform;

/* CloudSettings / CloudPipelineKey (src/gaussian/settings.rs:90-133, render/mod.rs:898-909). */
enum { BGS_GAUSSIAN_2D = 0, BGS_GAUSSIAN_3D = 1, BGS_GAUSSIAN_4D = 2 /* bgs_render_4d only */ };
enum {
    BGS_RASTERIZE_COLOR = 0, BGS_RASTERIZE_DEPTH = 1, BGS_RASTERIZE_NORMAL = 2, BGS_RASTERIZE_POSITION = 3,
    BGS_RASTERIZE_CLASSIFICATION = 4, BGS_RASTERIZE_OPTICAL_FLOW = 5,   /* bgs_render_ex */
    BGS_RASTERIZE_VELOCITY = 6                                           /* bgs_render_4d only */
};
enum { BGS_DRAW_ALL = 0, BGS_DRAW_SELECTED = 1, BGS_DRAW_HIGHLIGHT_SELECTED = 2 };
enum {
    BGS_FLAG_SORT_ALL = 1u, /* sort all N entries like the reference (culled keyed 0xFFFFFFFF)
                               instead of stream-compacting the visible ones first; same output */
    BGS_FLAG_ASYNC = 2u,    /* bgs_render only enqueues the frame on the context stream and returns;
                               bgs_sync() completes it (frames may be queued back to back, like the
                               reference's command-buffer submission: radix.rs / mod.rs never read back) */
    BGS_FLAG_NO_CHUNKS = 4u,/* never split the frame into front-to-back binning rounds (see BGS_FLAG_CHUNKS);
                               the tile debug hooks need a one-round frame */
    BGS_FLAG_PREMULTIPLIED_OUT = 16u, /* frame = the splat layer alone, premultiplied: (C, 1 - T) -- no implicit black clear,
                               alpha = coverage.  What a compositor needs to put the layer over anything later. */
    BGS_FLAG_BLEND_OVER_TARGET = 32u, /* blend over what the target already holds, dst = src + (1 - src.a) * dst on all four
                               channels -- the reference's PREMULTIPLIED_ALPHA_BLENDING on the view target
                               (render/mod.rs:944-948): several clouds per view (one bgs_render each, far cloud first,
                               mod.rs:398-452) and a scene behind the splats.  Target = out_rgba when it is a device
                               pointer, else the context's frame that the previous call rendering into the context's
                               frames wrote, synchronous or queued (frames delivered to host memory are copied out
                               after blending).  A pixel no splat blends keeps its bytes, except that -0.0 becomes +0.0
                               in RGBA16F / RGBA32F targets (and a NaN may come back as another NaN).  A frame whose
                               (splat, tile) pair list outgrew the buffer (BGS_NOT_READY) leaves the target as it was:
                               a synchronous call renders such a frame again by itself and composites it once; after a
                               queued one, bgs_sync's BGS_NOT_READY means the overflowed frames did not touch their
                               targets, so rendering them again composites each once. */
    BGS_FLAG_CHUNKS = 8u,   /* bin / tile-sort / blend in front-to-back rank rounds that stop emitting (splat, tile)
                               pairs once every tile has saturated.  Same pixels, bit for bit.  Only USE_OBB frames from
                               bgs_render (not USE_AABB ones, not bgs_render_aux, not BGS_FLAG_VISUALIZE_BOUNDING_BOX
                               ones) of at most 65536 tiles are ever split
                               into rounds; other frames ignore the flag and run one round.  Without either flag the
                               library picks rounds for such frames when the previous frame had >= 32 (splat, tile)
                               pairs per visible splat and >= 2^24 pairs. */
    BGS_FLAG_VISUALIZE_BOUNDING_BOX = 64u /* CloudSettings.visualize_bounding_box (the reference's VISUALIZE_BOUNDING_BOX
                               shader def, gaussian.wgsl:486-495): draw a band around each splat's quad, opaque green.
                               Honoured by bgs_render, _ex, _depth_test, _aux, _4d, _scene and _scene_4d (every listed
                               cloud) and bgs_render_entities (every entity).  The rule, exactly:
                               - For a (pixel, splat) pair whose coverage decision holds (after the aabb power > 0
                                 discard) and, under a depth buffer, whose depth test holds, take uv: the quad uv of the
                                 coverage test |u|, |v| <= 1 for quad-uv splats (USE_OBB: 3DGS, 2DGS, 4D); (mx / R, my / R)
                                 for conic (3DGS / 4D with aabb) and surfel (2DGS with aabb) splats, m the quad-space
                                 offset in half-pixels (y up) and R the half-side the coverage test compares |m| against,
                                 IEEE division.
                               - s = uv * 0.5f + 0.5f per component in f32 (the multiply is exact: one rounding).  The
                                 pair is an edge iff s.x < 0.08f || s.x > 1.0f - 0.08f || s.y < 0.08f || s.y > 1.0f - 0.08f
                                 (the subtraction in f32; a NaN component is not an edge).
                               - An edge pair blends (0.3f, 1.0f, 0.1f) at alpha exactly 1: C += T * colour, T := 0, so
                                 the pixel stops.  Any other covered pair blends as without the flag.  The test comes
                                 before the opacity, so boxes are drawn whatever the splat's opacity or colour (opacity
                                 0, global_opacity 0, Velocity's zeroed splats); a splat with no quad (culled, unselected
                                 under BGS_DRAW_SELECTED, time-masked 4D) has none.
                               - bgs_render_aux: the depth and normal frames get the same edges, in the same colour.
                               - Unchanged: key-gen, both sorts, records, binning, tile ranges and slices, splat depths
                                 and every debug hook.  An overlay frame runs in one round (BGS_FLAG_CHUNKS is ignored),
                                 so bgs_frame_stats is that of the same frame with BGS_FLAG_NO_CHUNKS.
                               - Unpinned: the reference interpolates uv across the quad in fixed function; whether that
                                 equals this uv (or its negation on one axis) is unpinned to the last ulp, so decisions
                                 within an ulp of a band edge may differ from the reference's. */
};
typedef struct {
    uint32_t gaussian_mode;           /* BGS_GAUSSIAN_* */
    uint32_t rasterize_mode;          /* BGS_RASTERIZE_* */
    uint32_t aabb;                    /* 0 = USE_OBB (default), 1 = USE_AABB */
    uint32_t opacity_adaptive_radius; /* default 1 */
    uint32_t draw_mode;               /* BGS_DRAW_* */
    uint32_t radix_sort_depth_bits;   /* 16 | 24 | 32 (RadixSortDepthBits) */
    uint32_t flags;                   /* BGS_FLAG_* */
    uint32_t reserved;
} bgs_settings;

/* Output frame formats.  RGBA8_SRGB / RGBA16F mirror the reference targets
 * (Rgba8UnormSrgb / Rgba16Float, render/mod.rs:917-921); RGBA32F is the premultiplied linear
 * accumulator parity is judged on. */
enum { BGS_FORMAT_RGBA8_SRGB = 0, BGS_FORMAT_RGBA16F = 1, BGS_FORMAT_RGBA32F = 2 };

typedef struct {
    uint32_t n;          /* gaussians in the cloud */
    uint32_t n_visible;  /* in-frustum gaussians this frame */
    uint64_t n_pairs;    /* (splat, tile) pairs emitted this frame (multi-round frames: summed over the rounds;
                            fewer than a one-round frame's when the frame saturated early) */
    uint32_t tiles_x, tiles_y;
    uint32_t width, height;
    uint32_t rounds;          /* binning rounds of the frame: 1, or > 1 on chunked frames (BGS_FLAG_CHUNKS) */
    uint32_t tiles_saturated; /* chunked frames: tiles whose every pixel saturated before the last round */
} bgs_frame_stats;

bgs_status bgs_context_create(int cuda_device, bgs_context** out);
void bgs_context_destroy(bgs_context* ctx);

/* Planar SoA upload, f32 layout (240 B/gaussian): planar_3d.rs:45-54, f32.rs:53-175.
 * pos_vis n*4 (x,y,z,visibility); sh n*48 (interleaved RGB x16); rot n*4 (w,x,y,z);
 * scale_opacity n*4 (linear scale xyz, linear opacity). */
bgs_status bgs_cloud_upload_f32(bgs_context* ctx, uint32_t n, const float* pos_vis, const float* sh,
                                const float* rot_wxyz, const float* scale_opacity, bgs_cloud** out);
/* f16 planar layout (128 B/gaussian): f16.rs:30-56,244-263; planar.wgsl:117-176.
 * sh_packed n*24 words (even coefficient in the low half); rot_scale_opacity n*4 words. */
bgs_status bgs_cloud_upload_f16(bgs_context* ctx, uint32_t n, const float* pos_vis, const uint32_t* sh_packed,
                                const uint32_t* rot_scale_opacity, bgs_cloud** out);
/* f16 planar layout with PRECOMPUTED 3D covariance (the reference's `precompute_covariance_3d` feature): the second plane
 * holds Covariance3dOpacityPacked128 {cov3d: [u32; 3], opacity: u32} (f16.rs:131-170; decode planar.wgsl:133-152)
 * instead of rotation + scale.  Projection then skips quat/scale -> Sigma3D; as in the reference shader
 * (gaussian_3d.wgsl:78-79) neither global_scale nor the model 3x3 touch the stored covariance.  Gaussian3d with
 * RasterizeMode Color / Depth / Position only (Normal and 2DGS need the rotation). */
bgs_status bgs_cloud_upload_f16_cov(bgs_context* ctx, uint32_t n, const float* pos_vis, const uint32_t* sh_packed,
                                    const uint32_t* cov3d_opacity, bgs_cloud** out);
void bgs_cloud_destroy(bgs_cloud* cloud);

/* Spherical-harmonic degree (the reference's build features sh0 .. sh3, src/material/spherical_harmonics.rs:41-87,
 * chosen here per cloud at upload).  The calls above store degree 3.  The rule, for d in {0, 1, 2, 3}:
 *   - K_d = (d + 1)^2 coefficients per channel; the SH plane holds S_d = pad4(3 K_d) floats per gaussian: 4, 12, 28, 48.
 *     Coefficient k of channel c is sh[3k + c] for k < K_d; lanes 3 K_d .. S_d - 1 are padding (lane 3 at degree 0,
 *     lane 27 at degree 2; degrees 1 and 3 have none).
 *   - f16 layouts hold S_d / 2 words per gaussian: 2, 6, 14, 24; the even coefficient in the low half.
 *   - colour = 0.5 + sum over k < K_d of shc[k] * basis_k(dir) * sh[3k + c] (the bands spherical_harmonics.wgsl:34-68
 *     keeps for SH_COEFF_COUNT > 11 / > 26 / > 47), then the sRGB decode as at degree 3.  Padding lanes are stored,
 *     downloaded, subset and interpolated, and never evaluated.  A degree-d cloud therefore renders exactly like the
 *     same cloud with its coefficients zero-padded to 48 (an FMA with a zero coefficient and a finite basis is exact).
 *   - Degree 3 is exactly the storage and the kernels of the calls above.
 * bgs_cloud_upload_f32_sh / _f16_sh / _f16_cov_sh take the arguments of the call without _sh plus sh_degree, and the SH
 * plane at the degree's width.  bgs_cloud_download_f32_sh / _f16_sh give the planes back at the cloud's width, bit for
 * bit as uploaded, padding lanes included; the downloads without _sh refuse a cloud of degree < 3.  Every other call
 * takes a cloud of any degree with unchanged semantics: the render calls in every geometry, mode, format and flag,
 * bgs_cloud_subset (the new cloud keeps the degree), selection, visibility, positions, particle steps, and
 * bgs_cloud_interpolate (over all S_d lanes or S_d / 2 words; lhs, rhs and out must share the degree).
 * bgs_cloud_sh_degree: the cloud's degree (3 for clouds of the calls without _sh, and for Gaussian4d clouds, whose
 * spatial degree it is).
 * sh_degree > 3, a null out for bgs_cloud_sh_degree, an _sh download of a cloud of the other precision or of a 4D
 * cloud, or an interpolation of clouds of different degrees -> BGS_EINVAL, with nothing allocated or enqueued.
 * Block sizes per gaussian (resident, besides the 16 B position plane): f32 64 / 128 / 256 / 256 B and f16 64 / 64 /
 * 128 / 128 B for degrees 0 / 1 / 2 / 3. */
bgs_status bgs_cloud_upload_f32_sh(bgs_context* ctx, uint32_t n, uint32_t sh_degree, const float* pos_vis,
                                   const float* sh /* n * S_d */, const float* rot_wxyz, const float* scale_opacity,
                                   bgs_cloud** out);
bgs_status bgs_cloud_upload_f16_sh(bgs_context* ctx, uint32_t n, uint32_t sh_degree, const float* pos_vis,
                                   const uint32_t* sh_packed /* n * S_d / 2 */, const uint32_t* rot_scale_opacity,
                                   bgs_cloud** out);
bgs_status bgs_cloud_upload_f16_cov_sh(bgs_context* ctx, uint32_t n, uint32_t sh_degree, const float* pos_vis,
                                       const uint32_t* sh_packed /* n * S_d / 2 */, const uint32_t* cov3d_opacity,
                                       bgs_cloud** out);
bgs_status bgs_cloud_download_f32_sh(bgs_context* ctx, const bgs_cloud* cloud, float* pos_vis /* n*4 */,
                                     float* sh /* n * S_d */, float* rot_wxyz /* n*4 */, float* scale_opacity /* n*4 */);
bgs_status bgs_cloud_download_f16_sh(bgs_context* ctx, const bgs_cloud* cloud, float* pos_vis /* n*4 */,
                                     uint32_t* sh_packed /* n * S_d / 2 */, uint32_t* second_plane /* n*4 */);
bgs_status bgs_cloud_sh_degree(const bgs_cloud* cloud, uint32_t* out);

/* A KHR_gaussian_splatting glTF primitive decoded into a resident cloud on the GPU (the reference's scene loader,
 * src/io/scene.rs).  The caller parses the glTF and describes each attribute's accessor; the call copies each
 * accessor's span, (n - 1) * byte_stride + element size bytes from `data`, once to the device, decodes it there and
 * repacks it as bgs_cloud_upload_f32_sh / _f16_sh (f16 != 0) would from the decoded planes, at sh_degree.
 *
 * bgs_khr_accessor: `data` is the host address of element 0, byte_stride the distance between elements (the
 * bufferView's byteStride, or the element size when tightly packed), component_type the glTF code (5120 i8, 5121 u8,
 * 5122 i16, 5123 u16, 5126 f32), components 1 (SCALAR), 3 (VEC3) or 4 (VEC4).  Accepted, as the reference accepts them:
 *   POSITION  VEC3 f32;
 *   ROTATION  VEC4 f32, or normalised i8 / i16;
 *   SCALE     VEC3 f32, i8 or i16, normalised or not (a log scale);
 *   OPACITY   SCALAR f32, or normalised u8 / u16;
 *   COLOR_0   VEC3 / VEC4 f32, u8 or u16 (u8 / u16 read as normalised whatever `normalized` says; alpha dropped);
 *   sh[k]     VEC3 f32, coefficient k = d*d + c of degree d, present for every k < (sh_degree + 1)^2.
 * With sh_degree 0 and sh[0].data NULL the primitive has no SH: the DC coefficients are COLOR_0 / 0.282095 when COLOR_0
 * is present (its data non-NULL), else 0.  COLOR_0 is ignored when SH are present; sh[k] beyond the degree are ignored.
 * The decode, every f32 operation round-to-nearest without FMA: a normalised value is max(v / 127, -1), max(v / 32767,
 * -1), v / 255 or v / 65535; the quaternion, in its stored order, becomes q * (1 / sqrt(((q0 q0 + q1 q1) + q2 q2) +
 * q3 q3)), or (1, 0, 0, 0) when that sum is <= FLT_EPSILON (such quaternions are counted in *out_zero_quats, which may
 * be NULL); scale = exp(raw) evaluated in f64 and rounded once to f32; position w = 1; f16 clouds round each value to
 * nearest even.  The rotation plane holds the four stored lanes in order (the reference reads (1, 0, 0, 0) as identity).
 * Refused with BGS_EINVAL, naming the attribute, before anything reaches the device: a NULL required accessor, an
 * unaccepted (components, component_type, normalized), byte_stride below the element size or not a multiple of the
 * component size, n outside [1, 2^30), sh_degree > 3.  Refused with BGS_EINVAL after the decode, the cloud released and
 * *out left NULL: a non-finite position, rotation (after normalising), exp(scale), SH coefficient or COLOR_0 value, and
 * an opacity that is NaN or outside [0, 1].  Synchronous; the context stays usable after any refusal. */
typedef struct {
    const void* data;
    uint32_t byte_stride;
    uint32_t component_type;
    uint32_t normalized;
    uint32_t components;
} bgs_khr_accessor;
typedef struct {
    uint32_t n;
    bgs_khr_accessor position, rotation, scale, opacity;
    bgs_khr_accessor color_0; /* optional: data NULL when absent */
    bgs_khr_accessor sh[16];
    uint32_t sh_degree;
} bgs_khr_primitive;
bgs_status bgs_cloud_upload_khr(bgs_context* ctx, const bgs_khr_primitive* primitive, uint32_t f16, uint32_t* out_zero_quats,
                                bgs_cloud** out);

/* Selection edits of a resident cloud: the visibility lane (pos_vis[4i + 3]) that DrawMode::Selected and
 * HighlightSelected read, changed in place without a re-upload.  All three calls are synchronous.
 *
 * bgs_cloud_select_sparse: SparseSelect (src/query/sparse.rs:24-54).  Sets each gaussian's visibility to 1.0 when
 * fewer than neighbor_threshold gaussians (itself included) lie within `radius` of it, else to 0.0.  Returns how many
 * were set to 1 in *out_selected (may be NULL).  The rule, exactly:
 *   - positions are the plane's x, y, z as uploaded (cloud-local: no model transform, no global_scale); every gaussian
 *     takes part, whatever its current visibility;
 *   - count_i = #{j : d2 < r2}, j == i included, d2 = ((dx*dx + dy*dy) + dz*dz), dx = x_j - x_i (likewise y, z),
 *     r2 = radius*radius rounded to f32, every operation f32 round-to-nearest-even without FMA (the order of
 *     `distance += diff * diff` from zero);
 *   - gaussian i is selected iff count_i < neighbor_threshold.
 *   So a non-finite position has a NaN d2 against everything, itself included: its count is 0.  radius == 0 counts
 *   nothing (every gaussian is selected when neighbor_threshold > 0); neighbor_threshold == 0 selects nothing.
 *   The reference delegates the comparison to the kd-tree 0.6.2 crate, absent here: `<` against `<=` and the
 *   accumulation order are **unpinned**.
 *   radius NaN, infinite or negative -> BGS_EINVAL.
 *   Cost: a hashed uniform grid (cells just over `radius`), one radix sort, and a scan of the 27 neighbour cells that
 *   stops once a count reaches neighbor_threshold.  A radius that puts most of the cloud into one cell (also: a radius
 *   below max|coordinate| * 2^-40, where cell coordinates saturate) with a large threshold costs O(N x threshold).
 *   It reuses the context's scratch (sort buffers and records): bgs_debug_* hooks, bgs_frame_stats_get and
 *   bgs_stage_times_us return BGS_NOT_READY, and bgs_frame_device_ptr NULL, until the next render.  The next frame's
 *   plan does not change (the hints it is planned from are kept).
 * bgs_cloud_visibility_get / _set: the visibility lane of every gaussian, n floats to / from host memory (_set writes
 *   the values as given: a 0/1 array built on the host covers Select, its inversion and any host-side labelling).
 * The writers (select_sparse, select_in_mesh, visibility_set) first complete this context's queued (BGS_FLAG_ASYNC) frames, as a
 * synchronous render does, returning their failure if there is one; and they wait for the queued frames of every
 * other context on the cloud's GPU (which may read this cloud), as bgs_cloud_destroy does.
 * A null cloud or array, or a cloud on another device than the context's -> BGS_EINVAL. */
bgs_status bgs_cloud_select_sparse(bgs_context* ctx, bgs_cloud* cloud, float radius, uint32_t neighbor_threshold,
                                   uint32_t* out_selected /* may be NULL */);
bgs_status bgs_cloud_visibility_get(bgs_context* ctx, const bgs_cloud* cloud, float* out_vis);
bgs_status bgs_cloud_visibility_set(bgs_context* ctx, bgs_cloud* cloud, const float* vis);

/* bgs_cloud_select_in_mesh: point-in-mesh selection (src/query/raycast.rs:54-124, RaycastSelectionPlugin).  A
 * gaussian is inside a triangle mesh iff the ray from its position along +x hits an odd number of its triangles.
 * mode BGS_SELECT_REPLACE: visibility := inside ? 1.0 : 0.0.  BGS_SELECT_ADD: visibility := 1.0 where inside, left
 * untouched elsewhere (the reference's sticky InsideMesh marker across several meshes; subtract is invert, ADD,
 * invert).  *out_inside (may be NULL) = how many gaussians are inside.  The rule, exactly:
 *   - q = mesh_from_cloud * (x, y, z, 1), (x, y, z) the plane's position as uploaded (cloud-local), mesh_from_cloud a
 *     column-major 4x4 (NULL: identity; the reference's transform.to_matrix().inverse() is the caller's), each row
 *     ((m_r0 x + m_r1 y) + m_r2 z) + m_r3; every gaussian takes part, whatever its current visibility;
 *   - triangle k is (v[i[3k]], v[i[3k + 1]], v[i[3k + 2]]), vertices (nv, 3) f32, indices (nt, 3) u32;
 *   - ray_intersects_triangle(q, dir = (1, 0, 0), tri) literally (raycast.rs:92-124): eps = 1e-6f; edge1 = v1 - v0,
 *     edge2 = v2 - v0, h = dir x edge2, a = edge1 . h, miss if a > -eps && a < eps; f = 1 / a, s = q - v0,
 *     u = f * (s . h), miss unless 0 <= u <= 1; q' = s x edge1, v = f * (dir . q'), miss if v < 0 || u + v > 1;
 *     t = f * (edge2 . q'), hit iff t > eps.  dot = (x x' + y y') + z z', cross = (y z' - y' z, z x' - z' x,
 *     x y' - x' y), the products with dir evaluated as written (0 * inf = NaN); every operation f32
 *     round-to-nearest-even without FMA.  glam's operation order is assumed, not pinned: the glam crate is absent
 *     here, so the order of its scalar Vec3 dot / cross / Mat4 transform is **unpinned**;
 *   - inside iff the hit count is odd.
 *   Consequences the rule keeps: a point on an edge shared by two triangles hits both (a ray through a shared edge
 *   or vertex may flip parity); a triangle with |a| < 1e-6 (e.g. any whose yz extent is below ~1e-3: eps is
 *   absolute) is never hit; an open or self-intersecting mesh gives whatever parity the rule gives; a non-finite
 *   point or triangle is never hit.  nt == 0: nothing is inside.
 *   Cost: a uniform grid over (y, z) binning the triangles, one radix sort of the (cell, triangle) pairs, and the
 *   literal test of each gaussian against the triangles of its cell.  Slivers (edge^2 / |a| > 2^16), triangles with a
 *   coordinate beyond 2^62 and gaussians with a coordinate of q beyond 2^62 are tested against everything instead.
 *   Synchronous; the quiesce rules of the writers above.  It uses its own scratch, not the frame's: the bgs_debug_*
 *   hooks, bgs_frame_stats_get and bgs_stage_times_us keep reporting the last frame, and the next frame's plan does
 *   not change.
 *   A null cloud, null vertices or indices with nt > 0, an index >= nv, an unknown mode, or a cloud on another device
 *   -> BGS_EINVAL; a refused call changes nothing.  nt >= 2^26 -> BGS_ENOMEM. */
enum { BGS_SELECT_REPLACE = 0u, BGS_SELECT_ADD = 1u };
bgs_status bgs_cloud_select_in_mesh(bgs_context* ctx, bgs_cloud* cloud, const float* vertices /* nv * 3 */, uint32_t nv,
                                    const uint32_t* indices /* nt * 3 */, uint32_t nt,
                                    const float* mesh_from_cloud /* 16, column-major, may be NULL */, uint32_t mode,
                                    uint32_t* out_inside /* may be NULL */);

/* bgs_cloud_select_in_view: selection through a screen-space mask -- rectangle, lasso and brush selection "through" the
 * volume, whatever is occluded (the host rasterises the shape into the mask).  mode as bgs_cloud_select_in_mesh's:
 * BGS_SELECT_REPLACE: visibility := inside ? 1.0 : 0.0; BGS_SELECT_ADD: 1.0 where inside, left untouched elsewhere.
 * *out_inside (may be NULL) = how many gaussians are inside.  The rule, exactly:
 *   - gaussian i is inside iff the projection, with this uniform's transform and this view, finds it in the frustum
 *     (key-gen's in_frustum decision); its record centre (cx, cy) -- bit for bit what bgs_debug_projected reports for it --
 *     satisfies 0 <= cx < w and 0 <= cy < h; and mask[floor(cy) * w + floor(cx)] != 0, with w = (int)viewport[2] and
 *     h = (int)viewport[3].  A NaN centre is never inside;
 *   - every gaussian takes part, whatever its visibility lane, draw mode or opacity; only the uniform's transform is read.
 *   mask: h * w bytes, row-major, in host memory or (mask_is_device_ptr) device memory of the context's GPU.
 *   Cost: one streaming pass over the position plane.  Synchronous; the quiesce rules of the writers above.  It uses its
 *   own scratch, not the frame's: the bgs_debug_* hooks, bgs_frame_stats_get and bgs_stage_times_us keep reporting the
 *   last frame, and the next frame's plan does not change.
 *   A Gaussian4d cloud (its drawn position depends on time; bgs_render_entities_pick covers 4D); a NULL ctx, cloud,
 *   uniform, view or mask; a viewport outside 1..65535; an unknown mode; a device mask that is not device memory of the
 *   context's GPU; or a cloud on another device -> BGS_EINVAL.  A refused call changes nothing. */
bgs_status bgs_cloud_select_in_view(bgs_context* ctx, bgs_cloud* cloud, const bgs_cloud_uniform* uniform, const bgs_view* view,
                                    const uint8_t* mask /* h * w, row-major */, int mask_is_device_ptr, uint32_t mode,
                                    uint32_t* out_inside /* may be NULL */);

/* Keeping a selection as its own cloud, and reading a cloud back (the reference's save_selection,
 * src/query/select.rs:156-176: cloud.subset(indices), then write_to_file).
 *
 * bgs_cloud_subset: a new resident cloud holding some of `cloud`'s gaussians, on the same device and in the same layout
 * (f32 / f16 / f16 precomputed covariance).  The rule, exactly:
 *   - selection mode (indices == NULL; k must be 0): gaussian i is kept iff !(w_i < 0.5f), w_i its visibility lane as
 *     it is now (after every selection edit, and every particle step enqueued on any context, before the call).  That is
 *     the set DrawMode::Selected draws: 0.5 is kept, nextafterf(0.5f, 0) is not; NaN and +inf are kept; -0, +0, -inf and
 *     subnormals are dropped.  (The hosts' selection() helpers use w >= 0.5, which drops NaN; they are unchanged.)  The
 *     kept gaussians stay in ascending index order.  Nothing kept: BGS_OK with *out = NULL and *out_n = 0 (a cloud
 *     still holds at least one gaussian, as at upload).
 *   - index mode (indices != NULL): the reference's subset(indices) literally: gaussian j of the result is gaussian
 *     indices[j] of the source; order is kept, repeats are allowed.  k must be in [1, 2^30); an index >= the cloud's n
 *     -> BGS_EINVAL, checked on the host before anything is allocated.
 *   - every byte of both device copies is copied unchanged (the position plane and the gaussian-major block), and the
 *     covariance flag is carried over.  The new cloud is registered with ctx like an uploaded one and released with
 *     bgs_cloud_destroy; it outlives its source and ctx.  It has never been stepped: its frames add no wait.
 *   Selection mode reads one number back (the kept count, which sizes the new planes).  Device memory beyond the new
 *   cloud: one mask word per 32 gaussians and one count per 256 (selection mode), or the k indices (index mode).
 * bgs_cloud_download_f32 / _f16: the planes exactly as the matching upload call takes them.  pos_vis comes from the
 *   position plane, the other planes from the blocks; a cloud that was never edited gives back the upload's arrays bit
 *   for bit.  For f16 clouds second_plane is the packed rotation-scale-opacity words, or the Covariance3dOpacityPacked128
 *   words of a precomputed-covariance cloud.  The planes go in chunks of 2^17 gaussians through device staging
 *   and two pinned host buffers the context keeps (2 x 30 MB, from its first download on).  The call of the other
 *   layout, or of a cloud of SH degree < 3 (bgs_cloud_download_f32_sh / _f16_sh read those) -> BGS_EINVAL.
 * Ordering: both calls only read the source and are synchronous.  They wait on the device for the particle steps
 * queued on the cloud (as bgs_cloud_visibility_get does) and do not drain other contexts' queued frames.  Their
 * scratch is their own: the bgs_debug_* hooks, bgs_frame_stats_get and bgs_stage_times_us keep reporting the last
 * frame, and the next frame's plan does not change.
 * A null ctx, cloud, out or plane pointer, a cloud on another device, or indices == NULL with k != 0 -> BGS_EINVAL;
 * an allocation failure -> BGS_ENOMEM.  A refused call creates and changes nothing (*out stays NULL). */
bgs_status bgs_cloud_subset(bgs_context* ctx, const bgs_cloud* cloud, const uint32_t* indices /* k, may be NULL */, uint32_t k,
                            bgs_cloud** out, uint32_t* out_n /* may be NULL */);
bgs_status bgs_cloud_download_f32(bgs_context* ctx, const bgs_cloud* cloud, float* pos_vis /* n*4 */, float* sh /* n*48 */,
                                  float* rot_wxyz /* n*4 */, float* scale_opacity /* n*4 */);
bgs_status bgs_cloud_download_f16(bgs_context* ctx, const bgs_cloud* cloud, float* pos_vis /* n*4 */,
                                  uint32_t* sh_packed /* n*24 */, uint32_t* second_plane /* n*4 */);

/* Gaussian4d clouds (planar_4d.rs:38-51, f32.rs:110-123,195-205; f32 only, as in the reference).  Per gaussian:
 *   pos_vis n*4 (x, y, z, visibility); sh n*144 (the SH-3 colour times time degree 2: coefficients 0..47 as
 *   bgs_cloud_upload_f32's, 48..95 the cos(2 pi theta) set, 96..143 the cos(4 pi theta) set, each interleaved RGB x 16);
 *   rotations n*8 (rotation then rotation_r, each (w, x, y, z) in storage order, used exactly as given: not normalised);
 *   scale_opacity n*4 (linear scale xyz, linear opacity); timestamp_timescale n*4 (timestamp, timescale, pad, pad).
 * The cloud is stored as 768 B gaussian-major blocks beside the position plane.  bgs_cloud_download_4d returns the
 * planes as uploaded, bit for bit for a cloud that was never edited (pads included).  bgs_cloud_subset,
 * bgs_cloud_select_sparse, bgs_cloud_select_in_mesh, bgs_cloud_visibility_get / _set, bgs_cloud_positions_get and
 * bgs_cloud_particles_step work on a 4D cloud as on a 3D one: they read and write the base position and visibility only.
 * The download call of another layout, bgs_cloud_interpolate of 4D clouds, bgs_render, bgs_render_ex,
 * bgs_render_depth_test and bgs_render_aux of a 4D cloud -> BGS_EINVAL. */
bgs_status bgs_cloud_upload_4d(bgs_context* ctx, uint32_t n, const float* pos_vis, const float* sh, const float* rotations,
                               const float* scale_opacity, const float* timestamp_timescale, bgs_cloud** out);
bgs_status bgs_cloud_download_4d(bgs_context* ctx, const bgs_cloud* cloud, float* pos_vis /* n*4 */, float* sh /* n*144 */,
                                 float* rotations /* n*8 */, float* scale_opacity /* n*4 */,
                                 float* timestamp_timescale /* n*4 */);

/* Particle behaviours (src/morph/particle.rs, particle.wgsl; the reference's `morph_particles` feature): a
 * ParticleBehaviors asset moves the gaussians it names every frame, in place, without a re-upload.
 *
 * bgs_particle_behavior is ParticleBehavior (particle.rs:349-358), 64 B.  indices[0] = the gaussian's index; a value
 * >= 2^31 (negative read as i32, as the shader reads it) marks the behaviour inactive; indices[1..3] are carried and
 * unused.
 * bgs_particles_create: uploads `count` behaviours (count in [1, 2^30)); two active behaviours naming the same gaussian
 *   -> BGS_EINVAL.  bgs_particles_get copies the current records back (count of them); bgs_particles_destroy releases
 *   them (steps still queued on any context complete first).
 * bgs_cloud_particles_step: one step of every behaviour over delta_time dt (particle.wgsl:36-52).  The rule, exactly:
 *   for each active behaviour, with p = pos_vis[indices[0]] (all four lanes: the visibility lane .w moves too),
 *   C6 = (float)(1.0 / 6.0) and every operation f32 round-to-nearest-even without FMA, per lane:
 *     dp = ((v*dt) + (((0.5f*a)*dt)*dt)) + ((((C6*j)*dt)*dt)*dt)
 *     dv = (a*dt) + (((0.5f*j)*dt)*dt)
 *     da = j*dt
 *   pos_vis[indices[0]] := p + dp, velocity := v + dv, acceleration := a + da; jerk and indices are never written.
 *   Inactive behaviours write nothing; gaussians no active behaviour names are untouched; non-finite values propagate
 *   as the arithmetic gives them.  Both device copies of the position (the plane key-gen streams, the block the
 *   projection reads) get the same four floats.  dt may be negative or zero.
 *   dt NaN or infinite, a behaviour naming a gaussian >= the cloud's n, a null argument, or a cloud or behaviours on
 *   another device than the context's -> BGS_EINVAL; a refused call changes nothing.
 * Ordering.  The step is ENQUEUED on the context's render stream (one kernel) and returns: no host synchronisation.
 *   Over every context on the cloud's GPU: a frame (or any call) enqueued before the step, on any context, reads the
 *   positions from before it; every call after it, on any context, observes it -- bgs_render, bgs_render_aux, the
 *   selection calls, bgs_cloud_visibility_get / _set, bgs_cloud_positions_get and further steps.  Steps of one
 *   bgs_particles, or of one cloud, run in call order whatever context queued them.  bgs_cloud_destroy and
 *   bgs_particles_destroy wait for steps queued on any context.  bgs_sync(ctx) completes ctx's queued steps; a fault
 *   of a step is reported by the next synchronising call on that context.  Frames of a cloud that was never stepped
 *   run exactly as before (no added wait, no added launch).
 * bgs_cloud_positions_get: the position plane, n * 4 floats (x, y, z, visibility), after every step queued on the cloud.
 * Where this port deliberately differs from the reference:
 *   1. Out-of-bounds dispatch: the shader indexes gid.x * 32 + gid.y with @workgroup_size(32, 32) over ceil(count / 32)
 *      workgroups, ~32x more invocations than behaviours; the extra ones read past the array, and under robust-access
 *      clamping the last behaviour is applied many times in one frame, racing with itself.  Here each behaviour is
 *      applied exactly once per step.
 *   2. Indices past the cloud and duplicate indices (particle_count may exceed the cloud, viewer.rs:407-438; two
 *      behaviours on one gaussian race) are refused with BGS_EINVAL.
 *   3. The reference runs the pass once per camera view (particle.rs:272-323: two cameras move the particles twice a
 *      frame), unordered against the sort (sort/radix.rs:97-118).  Here the caller steps explicitly, and a frame sees
 *      exactly the steps enqueued before it.
 *   4. The entity's Aabb is not updated, as in the reference (gaussian/cloud.rs:43): RasterizeMode::Position keeps
 *      the uniform's aabb_min / aabb_max as the caller passes them. */
typedef struct bgs_particles bgs_particles; /* opaque, library-owned: a ParticleBehaviors asset resident on one GPU */
typedef struct {
    uint32_t indices[4]; /* [0] = gaussian index; >= 2^31 (i32 < 0) = inactive; [1..3] carried, unused */
    float velocity[4];
    float acceleration[4];
    float jerk[4];
} bgs_particle_behavior;
bgs_status bgs_particles_create(bgs_context* ctx, const bgs_particle_behavior* behaviors, uint32_t count, bgs_particles** out);
bgs_status bgs_particles_get(bgs_context* ctx, const bgs_particles* particles, bgs_particle_behavior* out /* count */);
void bgs_particles_destroy(bgs_particles* particles);
bgs_status bgs_cloud_particles_step(bgs_context* ctx, bgs_cloud* cloud, bgs_particles* particles, float delta_time);
bgs_status bgs_cloud_positions_get(bgs_context* ctx, const bgs_cloud* cloud, float* out_pos_vis /* n * 4 */);

/* Interpolation (src/morph/interpolate.rs, interpolate.wgsl:51-119; the reference's GaussianInterpolate { lhs, rhs }):
 * `out` := the blend of two clouds at a time between time_start and time_stop (CloudSettings.time / time_start /
 * time_stop of the output entity, defaults 0 / 0 / 1), without a re-upload.  The output cloud is made once, e.g. as
 * bgs_cloud_subset(lhs, [0, n)), the device form of the reference's "clone lhs".
 * bgs_cloud_interpolate.  The rule, exactly:
 *   - the factor t (interpolate.wgsl:51-57), computed once on the host in f32: d = time_stop - time_start; if
 *     |d| < 1e-6f, t = (time >= time_stop) ? 1 : 0; otherwise t = min(max((time - time_start) / d, 0), 1), where a
 *     quotient of -0 stays -0 (time == time_start with d < 0; WGSL does not pin the sign of a zero max);
 *   - every lane of gaussian i is mix(a, b, t) = a*(1-t) + b*t, a from lhs, b from rhs, 1-t rounded once; every
 *     operation f32 round-to-nearest-even without FMA, subnormals kept.  The lanes: position xyz and visibility (both
 *     device copies: the position plane and the block), the S_d SH lanes (48 at degree 3), scale xyz and opacity, or for the
 *     precomputed-covariance layout the six covariance entries and opacity;
 *   - the rotation is normalize_quaternion(mix(q_l, q_r, t)) (:59-65): l2 = ((q0*q0 + q1*q1) + q2*q2) + q3*q3 in
 *     storage lane order (w, x, y, z); if l2 <= 0 the lanes are (0, 0, 0, 1), i.e. w = 0, z = 1 (a half-turn about z:
 *     it renders like the identity, and is what a download returns), which also covers q and -q at t = 0.5 and
 *     components whose squares underflow; otherwise each lane is q_k / sqrt(l2), IEEE division and square root.  NaN
 *     and overflow propagate as that arithmetic gives them;
 *   - f16 layouts: each half is widened exactly, blended as above in f32 and narrowed with round-to-nearest-even
 *     (past the f16 range: +-inf), in the lane map of the upload (planar.wgsl:264-331 against :116-176), except that
 *     the covariance record's fourth word is pack2x16float(vec2(0.0, opacity)): its low half is +0 whatever the inputs
 *     held.  The reference's f16 path is never compiled and the rounding of its pack2x16float is the implementation's:
 *     both are **unpinned**, as for the rest of f16.
 *   Note that mix(a, a, t) need not equal a; lhs == rhs is allowed.
 * Ordering.  The call is ENQUEUED on the context's render stream (one kernel) and returns: no host synchronisation.
 *   `out` is written as a particle step writes a cloud: after every frame queued on any context of the GPU and every
 *   earlier queued write of `out`; frames and reads of `out` on any context see exactly the interpolations enqueued
 *   before them.  lhs and rhs are read after every queued write of them enqueued before the call (particle steps,
 *   interpolations into them), on any context.  A later write of lhs or rhs -- a particle step, an interpolation into
 *   them, bgs_cloud_visibility_set, the selection calls -- or bgs_cloud_destroy waits for the interpolation.  bgs_sync(ctx)
 *   completes ctx's queued interpolations; a fault is reported by the next synchronising call on that context.  A
 *   context that never interpolates issues the same launches and waits as before.
 * Where this port deliberately differs from the reference:
 *   1. lhs, rhs and out must hold the same n in the same layout (f32 / f16 / f16 precomputed covariance) and SH
 *      degree.  The reference sizes the output as a clone of lhs and indexes rhs unguarded.
 *   2. out may not be lhs or rhs (in the reference it is always a separate asset).
 *   3. The caller interpolates explicitly, once; the reference runs the pass once per camera view
 *      (interpolate.rs:388-475), with the same inputs and so the same result.
 *   4. The entity's Aabb is not updated, as for the particle step: RasterizeMode::Position reads the caller's.
 * A null argument, a cloud on another device than the context's, a mismatch of n, layout or SH degree, out == lhs or rhs, a
 * time, time_start or time_stop that is not finite, or a NaN factor (e.g. (3e38 - -3e38) / inf) -> BGS_EINVAL; a
 * refused call changes and enqueues nothing. */
bgs_status bgs_cloud_interpolate(bgs_context* ctx, bgs_cloud* out, const bgs_cloud* lhs, const bgs_cloud* rhs, float time,
                                 float time_start, float time_stop);

/* Transforms and bounds: move, rotate or scale a resident cloud or its selection in place (an editor's gizmo drag, the
 * alignment of one scan to another, a node transform baked in before saving), and measure its positions' bounds.
 * bgs_cloud_transform bakes a similarity transform M -- a rotation R, a uniform scale s > 0 and a translation, given
 * column-major in the cloud's own frame (a world-space delta W becomes model^-1 W model) -- into the stored gaussians.
 * The rule, exactly:
 *   - which gaussians: BGS_TRANSFORM_ALL every one; BGS_TRANSFORM_SELECTED those whose visibility v has !(v < 0.5f)
 *     (DrawMode::Selected's and bgs_cloud_subset's predicate: NaN and +inf are selected, -0 and -inf are not), read as
 *     the visibility lane is when the transform runs.  Every byte of a gaussian it leaves alone stays as it was, in both
 *     device copies;
 *   - the matrix, checked on the host in f64: every entry finite; the bottom row exactly (0, 0, 0, 1); with c_i the
 *     columns of the 3x3 block A, |c|^2 = (x*x + y*y) + z*z and s^2 = ((|c0|^2 + |c1|^2) + |c2|^2) / 3 > 0;
 *     |c_i . c_j - s^2 delta_ij| <= 1e-5 s^2 for every i, j; det A > 0 (a reflection has no quaternion with positive
 *     scales).  s = sqrt(s^2), R = A / s, and q_R is R's quaternion by Shepperd's method (the largest of trace, R00, R11,
 *     R22 picks the root, the first on a tie), normalised in f64, taken with w >= 0 and rounded to f32; s is rounded
 *     to f32 likewise;
 *   - position: p' = M (x, y, z, 1), each row ((m_r0 x + m_r1 y) + m_r2 z) + m_r3 -- the projection's model multiply,
 *     so the baked position is, bit for bit, the world position a frame with uniform.transform = M computes.  Both
 *     copies are written; the visibility lane keeps its bits;
 *   - rotation: q' = q_R (x) q, the Hamilton product in storage order (w, x, y, z), not normalised:
 *       w' = ((aw bw - ax bx) - ay by) - az bz        x' = ((aw bx + ax bw) + ay bz) - az by
 *       y' = ((aw by - ax bz) + ay bw) + az bx        z' = ((aw bz + ax by) - ay bx) + az bw    (a = q_R, b = q).
 *     The renderer's rotation rows are R_std(q)^T, so a splat's covariance is R_std S^2 R_std^T and R_std(q') =
 *     R R_std(q).  That identity holds for unit quaternions only, as the renderer's formula is one for unit ones;
 *   - scale: scale' = s * scale per axis; opacity keeps its bits;
 *   - precomputed-covariance layout: Sigma' = A Sigma A^T (= s^2 R Sigma R^T), with X = A Sigma then X A^T, each entry
 *     (a0 b0 + a1 b1) + a2 b2 -- the projection's T Sigma T^t order; the opacity word keeps its bits;
 *   - SH: for each channel and band l in 1..3 up to the cloud's degree, c'_l = D_l^T c_l, where D_l is defined by
 *     Y_l(R^T d) = D_l Y_l(d) with Y_l the renderer's own band-l basis (its polynomials times its constants), so the
 *     baked colour seen along a direction equals the original's seen along the rotated one.  D_l is computed once per
 *     call on the host in f64, from q_R's rotation before rounding (least squares over 64 fixed directions; entries
 *     below 2^-40 are 0), and rounded to f32.  (D_l^T composes as the rotations do: D(R1 R2)^T = D(R1)^T D(R2)^T.)  The
 *     kernel sums c'_i = E_i0 c_0 + E_i1 c_1 + ... over j ascending, E = D_l^T.  Band 0 and the padding lanes are never
 *     touched: a degree-0 cloud's SH stays bit for bit;
 *   - every operation f32 round-to-nearest-even without FMA, subnormals kept; non-finite values propagate as that
 *     arithmetic gives them.  f16 layouts: each half is widened exactly, transformed in f32 and narrowed
 *     round-to-nearest-even (past 65504: +-inf), in the upload's lane map; the opacity half, and the zero words of the
 *     last SH chunk, keep their stored bits.
 * Ordering: a queued write of the cloud, exactly as bgs_cloud_particles_step: one kernel enqueued on the context's render
 *   stream, no host synchronisation.  Frames and calls enqueued before it, on any context, see the old cloud; every
 *   call after it the new one.  bgs_sync(ctx) completes it, bgs_cloud_destroy waits for it.  A context that never
 *   transforms issues the same launches as before.  The entity's Aabb is not updated, as after a particle step:
 *   bgs_cloud_bounds is how the caller refreshes it.
 * A null argument, a cloud on another device than the context's, an unknown mode, a matrix that fails the check, or a
 * Gaussian4d cloud (its two rotations and spherindrical coefficients are not rotated here) -> BGS_EINVAL; a refused call
 * changes and enqueues nothing.
 * bgs_cloud_bounds: per axis, the min and max of the position plane (cloud-local, after every write queued on the
 * cloud) over the gaussians `mode` selects (the transform's predicate) whose x, y and z are all finite; *out_count (may
 * be NULL) is how many took part.  With none: min = +inf, max = -inf, count 0.  -0 and +0 compare equal: which zero
 * comes back when both occur on an axis is unpinned.  Synchronous: it waits on the device only for the writes queued on
 * this cloud, never for other contexts' frames; one streaming pass over the position plane (16 B per gaussian) into the
 * call's own words, then one read-back, so the debug hooks and the next frame's plan are untouched.  A Gaussian4d
 * cloud's base positions are measured.  A null argument, a cloud on another device or an unknown mode -> BGS_EINVAL.
 * An entity's Aabb (positions -+ 0.1) follows from the bounds as the host's compute_aabb computes it. */
enum { BGS_TRANSFORM_ALL = 0u, BGS_TRANSFORM_SELECTED = 1u };
bgs_status bgs_cloud_transform(bgs_context* ctx, bgs_cloud* cloud, const float* local_from_local /* 16, column-major */,
                               uint32_t mode);
bgs_status bgs_cloud_bounds(bgs_context* ctx, const bgs_cloud* cloud, uint32_t mode /* BGS_TRANSFORM_* */, float out_min[3],
                            float out_max[3], uint32_t* out_count /* may be NULL */);

/* One view of one cloud: key-gen -> depth radix sort -> projection + SH colour -> tile
 * binning -> per-tile front-to-back blend.  out_rgba is caller-owned (host pointer, or a
 * device pointer when out_is_device_ptr != 0); may be NULL to keep the frame on the device.
 * A device target must be aligned to one pixel: 4 bytes for RGBA8, 8 for RGBA16F, 16 for RGBA32F
 * (bgs_render_aux: each of its three targets); else BGS_EINVAL, nothing enqueued or written. */
bgs_status bgs_render(bgs_context* ctx, const bgs_cloud* cloud, const bgs_view* view,
                      const bgs_cloud_uniform* uniform, const bgs_settings* settings, void* out_rgba,
                      uint32_t out_format, int out_is_device_ptr);

/* Colour + depth + normal frames of one view in ONE pass (BASELINE.json config 4: "2M-surfel 2dgs cloud with depth+normal
 * outputs").  out_rgba gets the frame bgs_render would produce with `settings` as given; out_depth / out_normal get, bit
 * for bit, the frames bgs_render would produce with rasterize_mode = Depth / Normal (gaussian.wgsl:329-368,
 * material/depth.wgsl:3-11): the splats' geometry, order and alpha do not depend on the colour source, so the extra
 * colours ride along (two more float3 per projected record, six more FMAs per blend).  All three frames share
 * out_format and the host/device kind of the pointers.  Synchronous only. */
bgs_status bgs_render_aux(bgs_context* ctx, const bgs_cloud* cloud, const bgs_view* view,
                          const bgs_cloud_uniform* uniform, const bgs_settings* settings, void* out_rgba,
                          void* out_depth, void* out_normal, uint32_t out_format, int out_is_device_ptr);

/* What a frame needs beyond bgs_render's arguments for RasterizeMode::Classification and OpticalFlow. */
typedef struct {
    float previous_clip_from_world[16]; /* OpticalFlow: this view's clip_from_world of the previous frame
                                           (PreviousViewUniforms.clip_from_world), column-major */
    float delta_time;                   /* OpticalFlow: seconds since that frame (Bevy's globals.delta_time) */
    uint32_t num_classes;               /* Classification: CloudSettings.num_classes (CloudUniform.num_classes) */
} bgs_render_extras;

/* bgs_render with extras: the one call that renders RasterizeMode::Classification and OpticalFlow.  bgs_render is this
 * call with extras == NULL, which means num_classes = 1 and no previous view; the four other modes ignore extras.
 * Both modes change only the colour a splat gets in the vertex stage (gaussian.wgsl:312-421): geometry, opacity,
 * coverage, sort order and blending are those of Color mode, and so are every geometry, layout, draw mode, output format
 * and flag they accept.
 *
 * The rule, exactly (f32, every step rounded, in the order written):
 *   Classification (gaussian.wgsl:315-328, material/classification.wgsl:9-27): sh = the Color-mode colour (the SH-3
 *     evaluation along the camera ray, sRGB -> linear decoded when color_space == 0: the decode is part of get_color,
 *     planar.wgsl:92-96, so it applies to sh and not to the hue); vis = the gaussian's visibility lane.  vis < 2: sh.
 *     Else hue = ((vis - 2) / f32(num_classes)) * 6.283185307 and the colour is mix(sh, hsv_to_rgb(hue, 1, 1), 0.5) =
 *     sh * (1 - 0.5) + rgb * 0.5.  vis is not floored (fractional labels give in-between hues) and a NaN vis takes the
 *     hue path, as in the reference.  An app labels gaussian i with class k by writing 2 + k into its visibility lane
 *     (bgs_cloud_visibility_set).
 *   OpticalFlow (gaussian.wgsl:201,369-375, material/optical_flow.wgsl:16-53): p = the transformed position (model * pos);
 *     the reference's previous position is the same p, so the colour shows camera motion only (particles and
 *     interpolation do not show).  c = clip_from_world (p, 1), c' = previous_clip_from_world (p, 1);
 *     mv = (c.xy / c.w - c'.xy / c'.w) * (0.5, -0.5); flow = mv / delta_time; radius = sqrt(flow.x^2 + flow.y^2);
 *     angle = atan2(flow.y, flow.x), + PI_2 when angle < 0; rgb = hsv_to_rgb(angle, clamp(radius, 0, 1), 1).
 *   hsv_to_rgb(h, s, v) (bevy_render::color_operations): k = (vec3(5, 3, 1) + h / FRAC_PI_3) % 6 with WGSL's f32
 *     remainder x - 6 * trunc(x / 6) (not fmodf); rgb = v - v * s * max(0, min(k, min(4 - k, 1))).  FRAC_PI_3 =
 *     1.0471975512 and PI_2 = 6.28318530718 (bevy_render::maths) rounded to f32.  The formula and the constants are
 *     restated from Bevy's source and its cited formula (Wikipedia, "HSV to RGB alternative"): parity unpinned, as f16
 *     rounding is.
 *   FP policy: min / max / clamp ignore a NaN operand (fminf / fmaxf); atan2 is a fixed f64 series rounded to f32
 *     (IEEE atan2's values at zeros and infinities: atan2(+-0, +0) = +-0, atan2(+-0, -0) = +-pi), so OpticalFlow colours
 *     are bit-exact against the oracle; Classification keeps Color mode's tolerance on sh, halved by the mix.
 *   DrawMode::HighlightSelected still paints every gaussian with vis > 0.5 green, labelled ones included
 *     (gaussian.wgsl:423-427); DrawMode::Selected still drops vis < 0.5.
 * Where this port deliberately differs from the reference (each BGS_EINVAL; a refused call changes and enqueues nothing):
 *   1. Classification with num_classes == 0 (the reference divides by zero).
 *   2. OpticalFlow without extras, with a delta_time that is not finite and > 0, or with a non-finite entry of
 *      previous_clip_from_world.
 *   3. Either mode through bgs_render_aux, which takes no extras. */
bgs_status bgs_render_ex(bgs_context* ctx, const bgs_cloud* cloud, const bgs_view* view,
                         const bgs_cloud_uniform* uniform, const bgs_settings* settings,
                         const bgs_render_extras* extras, void* out_rgba, uint32_t out_format, int out_is_device_ptr);

/* The scene's depth buffer a frame is depth-tested against (the view's Depth32Float depth texture, reverse-Z). */
typedef struct {
    const float* depth;    /* device memory on the context's GPU: the viewport's w x h Depth32Float values,
                              row-major, pixel (0, 0) at the viewport's top-left */
    uint64_t pitch_bytes;  /* bytes from one row to the next: a multiple of 4, >= 4 w (wgpu's copy_texture_to_buffer
                              pads rows to 256 bytes) */
} bgs_scene_depth;

/* bgs_render_ex with the reference's depth test: splats are drawn in the transparent pass against the view's depth
 * buffer with depth_compare GreaterEqual and depth writes off (render/mod.rs:959-974), so opaque geometry drawn earlier
 * hides the splats behind it.  depth == NULL makes the call exactly bgs_render_ex.  Every geometry, layout, RasterizeMode,
 * draw mode, format, output mode and flag bgs_render_ex accepts is accepted here.
 *
 * The rule, exactly (f32, round to nearest even, IEEE division, no contraction):
 *   Splat depth.  Each splat has one depth d = pz / pw, where p = model * pos as the projection computes it,
 *     h = clip_from_world * (p, 1), pz = h.z / (h.w + 1e-9) and pw = h.w / (h.w + 1e-9): the z and w lanes of
 *     world_to_clip (transform.wgsl:5-8).  The reference emits (projected.xy + bb.xy, projected.zw) for all four quad
 *     vertices (gaussian.wgsl:429-433), so its fragment depth is constant over the quad; 2DGS surfels use the same d.
 *     Fixed-function depth interpolation may differ from this d in the last ulp: parity unpinned, as f16 rounding is.
 *   The test.  A (pixel, splat) pair blends iff the coverage decision of bgs_render_ex holds and d >= scene[pixel].  The
 *     compare is IEEE: a NaN scene depth or +inf hides every splat, and -0 == +0.  A hidden pair leaves T and the colour
 *     unchanged, and later splats at that pixel continue.  A cleared reverse-Z buffer (0.0) hides nothing drawn with
 *     h.w >= 0 (every drawn splat has pz > 0); a splat drawn with h.w in (-1e-9, 0) -- possible only when the frustum
 *     test passes with |h.x|, |h.y|, h.z all below 1.1e-9, e.g. a clip matrix scaled to tiny values -- has pw < 0 and
 *     d < 0, and a zero buffer hides it.
 *   Unchanged stages.  Key-gen, the depth sort, the projection records, binning, the pair list, the tile ranges and
 *     entries and bgs_frame_stats are those of the same frame without a depth buffer; only pixels change.
 *   The buffer.  Only read, never written (the reference does not write depth either).  A queued frame
 *     (BGS_FLAG_ASYNC) reads it in its blend kernel, so it must stay unchanged until that frame completes, the same
 *     contract a device target has.
 * Known difference, left as it is: a splat with h.w below about 0.03 can have pz / pw > 1.  The reference's clipper
 *   (unclipped_depth: false) drops it; this port draws it, with or without a depth buffer.
 * Refused with BGS_EINVAL, nothing enqueued or written: a NULL depth->depth; a pitch that is not a multiple of 4 or is
 *   below 4 w; a pointer that is not 4-byte aligned; a pointer that is not device memory of the context's GPU.
 * bgs_render_aux takes no depth buffer. */
bgs_status bgs_render_depth_test(bgs_context* ctx, const bgs_cloud* cloud, const bgs_view* view,
                                 const bgs_cloud_uniform* uniform, const bgs_settings* settings,
                                 const bgs_render_extras* extras, const bgs_scene_depth* depth, void* out_rgba,
                                 uint32_t out_format, int out_is_device_ptr);

/* A Gaussian4d cloud (bgs_cloud_upload_4d) at time uniform->time: the reference's GaussianMode::Gaussian4d
 * (gaussian.wgsl:191-311, gaussian_4d.wgsl:37-130, spherindrical_harmonics.wgsl:11-126).  Arguments as
 * bgs_render_depth_test's (extras and depth may be NULL), plus the playback window time_start / time_stop
 * (CloudSettings.time_start / time_stop).  settings->gaussian_mode must be BGS_GAUSSIAN_4D; rasterize_mode Color, Depth,
 * Position, Classification, OpticalFlow or Velocity; every draw mode, format, output mode and flag of
 * bgs_render_depth_test is accepted.  Key-gen and the depth sort are those of a 3D cloud of the same base positions (the
 * key does not depend on time); binning, the blend and the depth test are unchanged; records have the 3D format.
 *
 * The rule, exactly (f32, round to nearest even, IEEE division and sqrt, no contraction, in the order written; matrices
 * [col][row] as WGSL indexes them, mat4x4(a, b, c, d, ...) filling columns):
 *   1. Drawn only if the base position p0 = model * (pos, 1) passes the frustum test (every depth width: difference 1
 *      below) and not (DrawMode::Selected and vis < 0.5).
 *   2. cutoff from the stored opacity (gaussian.wgsl:229-235), before the time modifier.
 *   3. S = diag(gs*sx, gs*sy, gs*sz, timescale), gs = global_scale.  With (w, x, y, z) = rotation and (wr, xr, yr, zr) =
 *      rotation_r as stored (lane 0 is w; not normalised): M_l = mat4x4(w,-x,-y,-z, x,w,-z,y, y,z,w,-x, z,-y,x,w),
 *      M_r = mat4x4(wr,-xr,-yr,-zr, xr,wr,zr,-yr, yr,-zr,wr,xr, zr,yr,-xr,wr).  R = M_r * M_l: R[c][r] =
 *      ((M_r[0][r] M_l[c][0] + M_r[1][r] M_l[c][1]) + M_r[2][r] M_l[c][2]) + M_r[3][r] M_l[c][3].  M = R * S:
 *      M[c][r] = R[c][r] * S[c][c] (the zero products of the diagonal are not added).  Sigma = transpose(M) * M:
 *      Sigma[c][r] = ((M[r][0] M[c][0] + M[r][1] M[c][1]) + M[r][2] M[c][2]) + M[r][3] M[c][3].
 *   4. dt = time - timestamp; cov_t = Sigma[3][3]; marginal_t = exp(((-0.5 * dt) * dt) / cov_t), exp the fixed f64
 *      series of csrc/project_math.cuh (det_exp: range reduction by ln 2, Taylor to degree 16, rounded to f32; 0 below
 *      -110, +inf above 89).  Not drawn unless marginal_t > 0.05 (a NaN, e.g. from cov_t == 0 with dt == 0, is not).
 *   5. c12 = (Sigma[0][3], Sigma[1][3], Sigma[2][3]); cov3d[c][r] = Sigma[c][r] - (c12[c] * c12[r]) / cov_t, passed to
 *      cov2d as (cov3d[0][0], [0][1], [0][2], [1][1], [1][2], [2][2]); delta_mean[i] = (c12[i] / cov_t) * dt.
 *   6. p = model * (pos + delta_mean, 1); not drawn unless p passes the frustum test; opacity = stored opacity *
 *      marginal_t.  The record is that of bgs_render's projection at p with cov3d (OBB or AABB; the model 3x3 does not
 *      touch cov3d, global_scale enters through S only), opacity * global_opacity, centre from p.
 *   7. Colour: Color = spherindrical_harmonics_lookup(dir, dt, sh): the SH-3 colour of bgs_render along the camera ray
 *      to p in the model frame, + cos(2 pi theta) * (sum_k basis_k sh[48 + 3k + c]) + cos(4 pi theta) * (sum_k basis_k
 *      sh[96 + 3k + c]), theta = dt / (time_stop - time_start), 2 pi and 4 pi the f32 multiples of radians(180.0), cos the
 *      fixed f64 series det_cos (reduction by 2 pi, Taylor to degree 36, rounded to f32); then the sRGB decode when
 *      color_space == 0.  Classification = that colour, then bgs_render_ex's class hue.  Depth = bgs_render's depth
 *      colour of |p - cam| between the distances of sorted entries 1 and count - 1, which hold base positions.
 *      Position = from p.  OpticalFlow = bgs_render_ex's rule with the current clip of p and the previous clip of the
 *      unmoved p0 (gaussian.wgsl:201).  Velocity (gaussian.wgsl:378-405): f = the conditioning at time + 1e-3 (its
 *      delta_mean 0 when its mask fails); v = (f.delta_mean - delta_mean) / 1e-3 in the local frame;
 *      scaled = clamp((|v| - 1) / (2 - 1), 0, 1), |v| = sqrt((vx*vx + vy*vy) + vz*vz); scaled < 1e-2: opacity 0 and rgb
 *      0 (difference 2); else rgb = (0.5 * (v / |v| + 1)) * scaled.
 *   8. DrawMode::HighlightSelected overrides colour and opacity of vis > 0.5 splats, as in bgs_render.
 *   9. The depth-test depth d is bgs_render_depth_test's of p.
 *   An undrawn record keeps the base position's centre and the stored opacity, with an empty bbox and no colour.
 *   FP policy: geometry, bbox, the draw decision, opacity, Velocity, OpticalFlow, Depth and Position colours are
 *   bit-exact against the oracle (temporal_oracle/); the SH-based colours are compared under a bound (FMA sums,
 *   approximate rsqrt and pow).
 * Where this port deliberately differs from the reference (BGS_EINVAL items: nothing enqueued or written):
 *   1. The reference drops base-culled gaussians by their key only at 32 depth bits; at 16 and 24 bits it skips the base
 *      frustum test for 4D and draws a base-culled gaussian whose moved position is in view, sorted as the farthest.
 *      Here every depth width culls on the base position, as the reference does at 32 bits.
 *   2. When Velocity sets opacity to 0, rgb is 0 too; the reference blends normalize(0) * 0 = NaN whenever v == 0.
 *   3. time_start == time_stop, time_stop - time_start not finite, or any of time, time_start, time_stop not finite
 *      -> BGS_EINVAL (the reference divides by zero).
 *   4. RasterizeMode::Normal (the reference calls get_rotation, which its 4D layout does not define), a cloud that is not
 *      4D, gaussian_mode != BGS_GAUSSIAN_4D -> BGS_EINVAL; bgs_render_aux and bgs_cloud_interpolate take no 4D cloud. */
bgs_status bgs_render_4d(bgs_context* ctx, const bgs_cloud* cloud, const bgs_view* view, const bgs_cloud_uniform* uniform,
                         const bgs_settings* settings, const bgs_render_extras* extras, const bgs_scene_depth* depth,
                         void* out_rgba, uint32_t out_format, int out_is_device_ptr, float time_start, float time_stop);

/* Several resident clouds in one view, rendered as one depth-sorted set: the k clouds clouds[0..k), cloud j with its own
 * uniforms[j], into one frame as if their gaussians were one cloud.  Arguments otherwise as bgs_render_depth_test's
 * (extras and depth may be NULL).  The reference draws each cloud entity as its own transparent item, sorted by entity
 * distance (render/mod.rs:398-452), so one cloud is painted wholly over another even where they interpenetrate; here
 * the clouds' splats share one depth sort, one binning and one blend.
 *
 * The rule, exactly:
 *   Index space.  Cloud j contributes its n_j gaussians at global indices o_j + i, o_j = n_0 + ... + n_{j-1};
 *     N = n_0 + ... + n_{k-1}.  The same cloud may be listed more than once (instancing): each listing is its own segment.
 *   Per-cloud values.  Everything a bgs_cloud_uniform carries (transform, global_opacity, global_scale, color_space,
 *     aabb_min / max) and the cloud's layout and SH degree come from the gaussian's own cloud j.  gaussian_mode,
 *     rasterize_mode, aabb, opacity_adaptive_radius, draw_mode, radix_sort_depth_bits, flags, num_classes and the depth
 *     buffer are the frame's.
 *   Key.  The key of global index g = o_j + i is the key bgs_render computes for gaussian i of cloud j with uniforms[j].
 *     The depth sort is stable and ascending over (key, g).
 *   Projected record.  The record of g is, bit for bit, the record bgs_render_depth_test with cloud j and uniforms[j]
 *     writes for i; so are its splat depth under a depth buffer, its OpticalFlow colour (p = M_j * pos) and its Position
 *     colour (cloud j's aabb).
 *   Depth mode.  The range is the sorted[1] / sorted[N-1] rule applied to the joint sorted entry list of N entries
 *     (culled tail in ascending global index); each entry's distance is taken from its own cloud's transformed position.
 *   Everything else is unchanged.  Binning, tile ranges and slices, chunked rounds, the blend, the depth test,
 *     PREMULTIPLIED_OUT, BLEND_OVER_TARGET, ASYNC and the pair-overflow re-render work on the joint record set exactly as
 *     for one cloud.  So k == 1 is exactly bgs_render_depth_test, and a cloud split into contiguous subsets (bgs_cloud_subset
 *     in index mode), each listed with the uniform of the whole, renders bit-identically to the whole cloud: pixels,
 *     sorted entries, tile ranges and slices, records, frame stats and launch count.  Clouds whose depth intervals do not
 *     overlap match the reference's far-first blend-over composite up to the rounding of the reassociated "over".
 *   Ordering.  Each listed cloud is read after every write queued on it before the call (particle steps, interpolations),
 *     on any context.  A queued frame's targets and depth buffer follow bgs_render_depth_test's contract.
 *   Debug hooks.  bgs_debug_sorted_entries, _tile_ranges, _tile_entries, _projected, _splat_depths, bgs_frame_stats_get
 *     (n = N) and bgs_stage_times_us report the frame in the global index space.
 * Launches: one key-gen over the whole scene, and one projection per distinct projection kernel among the clouds (f32
 *   or f16 storage, SH degree; the f16 and f16-covariance layouts share one), so a scene of clouds of one layout and
 *   degree costs the launches of one cloud.
 * Refused with BGS_EINVAL, nothing enqueued or written: k == 0 or k > BGS_SCENE_MAX_CLOUDS; a NULL entry in clouds; a
 *   Gaussian4d cloud; a cloud on another device; N >= 2^30; BGS_FLAG_SORT_ALL (the reference-literal order belongs to
 *   one draw, and a scene is several); any refusal bgs_render_depth_test makes for one of the clouds with its uniform.
 *   NULL clouds, uniforms, view or settings -> BGS_NOT_READY, as for bgs_render. */
#define BGS_SCENE_MAX_CLOUDS 64
bgs_status bgs_render_scene(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms, uint32_t k,
                            const bgs_view* view, const bgs_settings* settings, const bgs_render_extras* extras,
                            const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format, int out_is_device_ptr);

/* bgs_render_scene with Gaussian4d clouds among the k: a dynamic 4D capture inside a static 3D scan, or one 4D capture
 * shown several times at staggered times, rendered as one depth-sorted set.  windows[j] is entity j's
 * CloudSettings.time_start / time_stop; it is read for Gaussian4d clouds only.  The reference draws each entity as its
 * own transparent item, so a performer is painted wholly over or under the room around it.
 *
 * The rule, exactly:
 *   Index space, keys, sort, binning, blend, depth test, flags, debug hooks, ordering: bgs_render_scene's.  A 4D cloud's
 *     key is bgs_render_4d's, the 3D key of its base position; every depth width culls on the base position.
 *   Per-cloud time.  A Gaussian4d cloud j is conditioned at uniforms[j].time in windows[j] (time_future = time + 1e-3f,
 *     duration = time_stop - time_start).  The same 4D cloud may be listed more than once, at different times.
 *   Record of a 4D gaussian: bit for bit the record bgs_render_4d writes for it with cloud j, uniforms[j] and windows[j];
 *     so are its splat depth under a depth buffer (from the moved position), its Position, OpticalFlow, Classification
 *     and Velocity colours, its Depth colour (the range from the joint sorted list, as in bgs_render_scene) and its
 *     undrawn record (masked by time, or moved out of the frustum).
 *   Record of any other gaussian: bgs_render_scene's.  In a Velocity frame it is keyed, sorted and counted in n_visible
 *     but undrawn (empty bbox, no colour): the reference's Velocity source conditions a 4D covariance, so a 3D entity
 *     has no pipeline in that mode and draws nothing.
 *   gaussian_mode.  4D clouds render as Gaussian4d; settings->gaussian_mode is the other clouds' (2D or 3D), and may be
 *     BGS_GAUSSIAN_4D only when every listed cloud is a Gaussian4d one.
 *   So with no 4D cloud listed the call is exactly bgs_render_scene (windows is not read and may be NULL), and a 4D cloud
 *   split into contiguous subsets, each listed with the uniform and window of the whole, renders exactly like
 *   bgs_render_4d of the whole: pixels, sorted entries, tile ranges and slices, records, splat depths, frame stats and
 *   launch count.
 * Launches: bgs_render_scene's for the non-4D clouds, plus one projection covering every 4D cloud.  The splat-depth
 *   launch runs only when a non-4D cloud is listed (the 4D projection writes its own), so an all-4D scene costs what
 *   bgs_render_4d costs.
 * Refused with BGS_EINVAL, nothing enqueued or written: every refusal of bgs_render_scene but the 4D one; every refusal
 *   of bgs_render_4d for a 4D cloud with its uniform and window (non-finite time or window, time_stop == time_start, an
 *   overflowing window, RasterizeMode::Normal, ...); windows == NULL with a 4D cloud listed; BGS_GAUSSIAN_4D with a
 *   non-4D cloud; BGS_GAUSSIAN_2D with aabb = 1 and a 4D cloud (that blend reads a surfel record for every splat; under
 *   OBB 2D and 4D records share one blend).  NULL clouds, uniforms, view or settings -> BGS_NOT_READY. */
typedef struct {
    float time_start, time_stop;   /* CloudSettings.time_start / time_stop of one entity */
} bgs_time_window;
bgs_status bgs_render_scene_4d(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                               const bgs_time_window* windows /* k; read for Gaussian4d clouds only */, uint32_t k,
                               const bgs_view* view, const bgs_settings* settings, const bgs_render_extras* extras,
                               const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format, int out_is_device_ptr);

/* bgs_render_scene_4d with each entity's own CloudSettings: an editor highlights one object's selection inside a room
 * drawn in full, a labelled object is drawn in Classification inside a scan drawn in Color, a 3DGS object or a 4D
 * performer stands on a 2DGS surface drawn with aabb -- all in one depth-sorted frame.
 *
 * The rule, exactly:
 *   Everything that is not below stays bgs_render_scene_4d's: index space, keys, the stable sort over (key, g), binning,
 *     the depth test, output modes, ASYNC, the pair-overflow re-render, ordering against queued writes, debug hooks.
 *   Frame-wide values.  frame->radix_sort_depth_bits and frame->flags (BGS_FLAG_SORT_ALL refused, as in scenes); the
 *     OpticalFlow previous view and delta_time of `extras` (its num_classes is not read); the depth buffer and the output.
 *   Per-entity values.  entities[j] carries entity j's gaussian_mode, rasterize_mode, aabb, opacity_adaptive_radius,
 *     draw_mode, num_classes and (Gaussian4d clouds only) time window; uniforms[j] its uniform.
 *   Records.  The record of g = o_j + i is, bit for bit, the record the single-cloud call (bgs_render_depth_test, or
 *     bgs_render_4d for a 4D cloud) writes for gaussian i with cloud j, uniforms[j] and entity j's settings as the frame's;
 *     so are the 2DGS aabb surfel record and the splat depth under a depth buffer.  A non-4D entity in Velocity gives an
 *     undrawn record, as bgs_render_scene_4d rules.
 *   Depth colour range.  bgs_render_scene's: sorted[1] / sorted[N-1] of the joint list over every entry, computed when
 *     some entity is in Depth mode.  (A deliberate difference: the reference takes each entity's range from its own sort.)
 *   Coverage.  Each (pixel, splat) decision is the one that splat's own blend makes -- quad-uv (OBB: 3DGS, 2DGS and 4D),
 *     conic (3DGS and 4D with aabb) or surfel (2DGS with aabb) -- bit for bit, and the splats blend in joint order.
 *     Frames whose entities use more than one of the three run one blend that tests each splat by its own kind; like
 *     aabb frames, they are never split into chunked rounds (BGS_FLAG_CHUNKS is ignored).
 *   Identity.  When all k entities agree (every setting above, num_classes in Classification, and the non-4D entities'
 *     gaussian_mode), the call is bgs_render_scene_4d with those settings, byte for byte: pixels, sorted entries, tile
 *     ranges and slices, records, stats and launch count.
 * Launches: one projection per (layout and SH degree, plain or Classification / OpticalFlow / Velocity colour kernel)
 *   among the non-4D entities and one for the 4D ones; a frame of mixed blend kinds adds one launch that tags each
 *   visible splat with its kind.
 * Refused with BGS_EINVAL, nothing enqueued or written: every refusal of bgs_render_scene_4d that still applies; any
 *   refusal of the single-cloud call for an entity with its settings (num_classes == 0 in Classification, a 4D cloud
 *   whose entity is not BGS_GAUSSIAN_4D, BGS_GAUSSIAN_4D on a 3D cloud, Normal on a 4D entity, an invalid window, ...);
 *   entities == NULL.  BGS_GAUSSIAN_2D with aabb beside a 4D cloud is accepted.  NULL clouds, uniforms, entities, view
 *   or frame -> BGS_NOT_READY. */
typedef struct {
    uint32_t gaussian_mode, rasterize_mode, aabb, opacity_adaptive_radius, draw_mode;   /* bgs_settings' */
    uint32_t num_classes;        /* Classification entities: > 0 */
    bgs_time_window window;      /* Gaussian4d entities only */
} bgs_entity_settings;
bgs_status bgs_render_entities(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                               const bgs_entity_settings* entities, uint32_t k, const bgs_view* view,
                               const bgs_settings* frame /* radix_sort_depth_bits and flags only */,
                               const bgs_render_extras* extras /* previous view and delta_time; num_classes unused */,
                               const bgs_scene_depth* depth, void* out_rgba, uint32_t out_format, int out_is_device_ptr);

/* bgs_render_entities with each entity's own flags (the reference's per-entity pipeline key): entity_flags[j] (k words;
 * NULL = none) is a set of BGS_ENTITY_* bits.  BGS_ENTITY_VISUALIZE_BOUNDING_BOX draws entity j's bounding boxes
 * (BGS_FLAG_VISUALIZE_BOUNDING_BOX's rule, for its splats only); the frame's BGS_FLAG_VISUALIZE_BOUNDING_BOX draws every
 * entity's.  Entities agree only when their overlays also agree; entities that differ in nothing else still blend in the
 * mixed blend.  bgs_render_entities is this call with entity_flags = NULL.  Refused with BGS_EINVAL, nothing enqueued or
 * written: an unknown bit in some entity_flags[j], and every refusal of bgs_render_entities. */
enum { BGS_ENTITY_VISUALIZE_BOUNDING_BOX = 1u };
bgs_status bgs_render_entities_ex(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                                  const bgs_entity_settings* entities, const uint32_t* entity_flags /* k, or NULL */,
                                  uint32_t k, const bgs_view* view, const bgs_settings* frame,
                                  const bgs_render_extras* extras, const bgs_scene_depth* depth, void* out_rgba,
                                  uint32_t out_format, int out_is_device_ptr);

/* bgs_render_entities_ex's frame and its depth and normal frames in ONE pass: bgs_render_aux for a scene, with or without
 * a depth buffer.  A 2DGS room scan with a 3DGS object in it gets the G-buffer an app needs for relighting, SSAO or
 * mesh compositing from one key-gen, sort, projection, binning and blend, with the splats of both clouds in joint order.
 *
 * The rule, exactly:
 *   out_rgba.  Byte for byte the frame bgs_render_entities_ex produces with the same arguments; every colour mode a
 *     non-4D entity takes, Classification and OpticalFlow included (extras as there).
 *   out_depth / out_normal.  Byte for byte the frames bgs_render_entities_ex produces when every entity's rasterize_mode is
 *     replaced by Depth / by Normal and everything else is kept: draw modes, each entity's bounding-box overlay (its edges
 *     in all three frames, as bgs_render_aux draws them), the depth test, BGS_FLAG_PREMULTIPLIED_OUT and
 *     BGS_FLAG_BLEND_OVER_TARGET.  The Depth colour range is the scenes' joint sorted[1] / sorted[N-1] rule.
 *   Targets.  All three share out_format and the host/device kind of the pointers.  Blend-over: a device target is blended
 *     over what it holds, each of the three over its own pixels.  Host targets: out_rgba over the context's last frame
 *     (as bgs_render_entities_ex), out_depth / out_normal over the depth / normal frames of the last aux frame
 *     (bgs_render_aux or this call) this context delivered to host memory -- transparent black before the first, and
 *     whenever this frame is larger than every aux frame before it (the library's aux buffers grow, zeroed).
 *   k == 1.  With depth == NULL and a Color, Depth, Position or Normal entity the call is bgs_render_aux with that
 *     entity's settings as the frame's, byte for byte in all three frames; with a depth buffer it is that frame with the
 *     depth test.  (bgs_render_aux itself takes no depth buffer.)
 *   Hooks and stats.  Sorted entries, tile ranges and slices, records (bgs_debug_projected: the rgba frame's colours; the
 *     aux colours are not part of the records), splat depths and bgs_frame_stats are those of the rgba frame's
 *     bgs_render_entities_ex call rendered in one round: like bgs_render_aux, the call is never split into chunked rounds
 *     (BGS_FLAG_CHUNKS is ignored).
 *   Synchronous only.
 * Launches: bgs_render_entities_ex's, plus the Depth range's when no entity is in Depth mode.
 * Refused with BGS_EINVAL, nothing enqueued or written and the previous frame's debug hooks kept: every refusal of
 *   bgs_render_entities_ex; a NULL target (any of the three); a device target not aligned to its pixel (each of the
 *   three); BGS_FLAG_ASYNC; a Gaussian4d cloud (its layout has no Normal colour); a precomputed-covariance cloud (no
 *   rotation); an entity in Velocity mode (it changes opacity and which splats draw, so the three frames would no
 *   longer share their alphas).  NULL clouds, uniforms, entities, view or frame -> BGS_NOT_READY. */
bgs_status bgs_render_entities_aux(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                                   const bgs_entity_settings* entities, const uint32_t* entity_flags /* k, or NULL */,
                                   uint32_t k, const bgs_view* view, const bgs_settings* frame,
                                   const bgs_render_extras* extras, const bgs_scene_depth* depth /* may be NULL */,
                                   void* out_rgba, void* out_depth, void* out_normal, uint32_t out_format,
                                   int out_is_device_ptr);

/* bgs_render_entities_ex's frame and, from the same pass, a pick frame: which gaussian the viewer sees at each pixel, for
 * click-to-select, brush and rectangle tools, hover highlights, and "place at cursor" or "measure" (the depth under the
 * cursor).  Per pixel, one 16 B bgs_pick record.
 *
 * The rule, exactly:
 *   out_rgba.  Byte for byte the frame bgs_render_entities_ex produces with the same arguments: in all three formats, with
 *     BGS_FLAG_PREMULTIPLIED_OUT and BGS_FLAG_BLEND_OVER_TARGET, per-entity and frame-wide bounding-box overlays, and under
 *     a depth buffer.
 *   Pairs.  The pairs a pixel's pick considers are exactly those that blend into its colour: each passes its splat's own
 *     coverage decision (quad-uv, conic or surfel), the depth test when a buffer is given, and arrives while the pixel is
 *     still alive (T >= T_STOP).
 *   Weight.  A pair's weight is w = a * T, the f32 product the blend multiplies the splat's colour by (an overlay edge
 *     pair has a = 1: w = T).
 *   Pick.  The pair with the largest w.  On a tie the pair earlier in blend order wins: a later pair replaces the current
 *     pick only when its w is strictly greater (a NaN w is never picked).
 *   Record.  entity: the entity j of the picked splat.  index: its gaussian index i within cloud j, as uploaded (the
 *     instances of one cloud differ in entity only).  weight: w.  depth: the splat depth d bgs_render_depth_test compares,
 *     clip z / w of the splat's world position (a 4D entity's moved position).
 *   Empty pixels.  A pixel where nothing blends gets {BGS_PICK_NONE, BGS_PICK_NONE, 0.0f, 0.0f} (0 is the reverse-Z far
 *     value, a Depth32Float clear).
 *   Targets.  out_pick (w * h records, row-major) shares out_is_device_ptr with out_rgba.  Every pixel of out_pick is
 *     written: blend-over applies to out_rgba only.
 *   Hooks and stats.  Sorted entries, tile ranges and slices, records and bgs_frame_stats are those of the same
 *     bgs_render_entities_ex frame rendered in one round: a pick frame is never chunked (BGS_FLAG_CHUNKS is ignored).
 *     After a pick frame bgs_debug_splat_depths reports every rank's d, whether or not a depth buffer was given.
 *   Synchronous only.
 * Launches: bgs_render_entities_ex's, plus the splat depths' when no depth buffer is given and a non-4D cloud is listed
 *   (the blend itself writes the pick records).
 * Refused with BGS_EINVAL, nothing enqueued or written and the previous frame's debug hooks kept: every refusal of
 *   bgs_render_entities_ex; a NULL out_pick; a device out_pick not aligned to 16 B; BGS_FLAG_ASYNC.  NULL clouds,
 *   uniforms, entities, view or frame -> BGS_NOT_READY. */
typedef struct {
    uint32_t entity;   /* entity j, or BGS_PICK_NONE */
    uint32_t index;    /* gaussian index within cloud j, or BGS_PICK_NONE */
    float weight;      /* w = a * T of the picked pair; 0 where nothing blends */
    float depth;       /* its splat depth d; 0 where nothing blends */
} bgs_pick;            /* 16 B */
#define BGS_PICK_NONE 0xFFFFFFFFu   /* (a macro: C99 enumerators are ints) */
bgs_status bgs_render_entities_pick(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                                    const bgs_entity_settings* entities, const uint32_t* entity_flags /* k, or NULL */,
                                    uint32_t k, const bgs_view* view, const bgs_settings* frame,
                                    const bgs_render_extras* extras, const bgs_scene_depth* depth /* may be NULL */,
                                    void* out_rgba, uint32_t out_format, int out_is_device_ptr,
                                    void* out_pick /* w * h bgs_pick */);

/* bgs_render_entities_ex of several views of one scene in ONE frame: stereo eyes, the six faces of a cube map, split-screen
 * and picture-in-picture cameras, or many cameras of a dataset share one key-gen, depth sort, projection, binning,
 * tile-id sort and blend launch instead of one set of launches per view (the reference renders every GaussianCamera).
 *
 * The rule, exactly:
 *   Per-view identity.  out_rgba[i] is byte for byte the frame bgs_render_entities_ex(clouds, uniforms, entities,
 *     entity_flags, k, &views[i], frame, NULL, depths ? &depths[i] : NULL, out_rgba[i], out_format, out_is_device_ptr)
 *     produces: in all three formats, with BGS_FLAG_PREMULTIPLIED_OUT, per-entity and frame-wide bounding-box overlays,
 *     and under each view's own depth buffer.  With BGS_FLAG_BLEND_OVER_TARGET each device target is blended over its own
 *     pixels.  Views may differ in size, and a view's size need not be a multiple of the tile size.
 *   Index space.  Segment i k + j is cloud j with uniforms[j] and entities[j], seen from view i; global indices run view
 *     after view (view i's are [i n, (i + 1) n), n = sum of the clouds' counts).  N = v n must be below 2^30, and
 *     v k <= BGS_SCENE_MAX_CLOUDS.
 *   Sort.  One stable depth sort over (key, g) of every view's entries; restricted to view i it is view i's own order.
 *   Tiles.  View i's tiles are the global tile ids [T_i, T_i + tiles_x(i) tiles_y(i)), T_i the sum over the earlier
 *     views, each view's in row-major order.  The tile-id sort runs over the global id, with pair_passes(total tiles)
 *     digit places.
 *   One round.  A views frame is never split into chunked rounds (BGS_FLAG_CHUNKS is ignored; chunked pixels are
 *     bit-identical anyway).
 *   Hooks and stats.  Sorted entries, records (bgs_debug_projected), splat depths and tile entries are in the global index
 *     and rank space; bgs_debug_tile_ranges writes every view's ranges, view after view.  bgs_frame_stats: n = N, n_visible
 *     and n_pairs over the whole frame, rounds = 1, tiles_x = every view's tiles and tiles_y = 1 (so a hook buffer sized
 *     tiles_x x tiles_y holds the ranges), width and height view 0's.
 *   BGS_FLAG_ASYNC is allowed, with bgs_render_entities_ex's pair-overflow rule.  Host targets: the library's frames hold
 *     all v frames, and each view is copied out to its out_rgba[i].
 *   v == 1.  The call is bgs_render_entities_ex: pixels, hooks, stats and launch count.
 * Launches: those of one bgs_render_entities_ex frame of the same entities, whatever v is.
 * Refused with BGS_EINVAL, nothing enqueued or written and the previous frame's debug hooks kept: every refusal
 *   bgs_render_entities_ex makes for some view; v == 0, v k > BGS_SCENE_MAX_CLOUDS or N >= 2^30; a NULL out_rgba or
 *   out_rgba[i]; a device target not aligned to its pixel; an entity in Depth mode (its colour range would be per
 *   view); an entity in OpticalFlow mode (one previous view per frame); BGS_FLAG_BLEND_OVER_TARGET with host targets
 *   (the context's last frame is not v frames).  NULL clouds, uniforms, entities, views or frame -> BGS_NOT_READY. */
bgs_status bgs_render_views(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                            const bgs_entity_settings* entities, const uint32_t* entity_flags /* k, or NULL */, uint32_t k,
                            const bgs_view* views, uint32_t v, const bgs_settings* frame,
                            const bgs_scene_depth* depths /* v, or NULL */, void* const* out_rgba /* v */,
                            uint32_t out_format, int out_is_device_ptr);

/* bgs_render_entities_aux of several views of one scene in ONE frame: the colour, depth and normal frames of every view --
 * a stereo headset's eyes for reprojection, the six faces of a cube map for relighting, a glTF scene's cameras, or a 2DGS
 * surfel scene seen from many dataset cameras -- from one key-gen, depth sort, projection, binning, tile-id sort and
 * blend launch instead of one set of launches per view.  Entities in Depth mode are drawn, each view over its own range.
 *
 * The rule, exactly:
 *   Per-view identity.  out_rgba[i], out_depth[i] and out_normal[i] are byte for byte the three frames
 *     bgs_render_entities_aux(clouds, uniforms, entities, entity_flags, k, &views[i], frame, NULL,
 *     depths ? &depths[i] : NULL, out_rgba[i], out_depth[i], out_normal[i], out_format, out_is_device_ptr) produces: in
 *     all three formats, with BGS_FLAG_PREMULTIPLIED_OUT, per-entity and frame-wide bounding-box overlays, and under each
 *     view's own depth buffer.  With BGS_FLAG_BLEND_OVER_TARGET each device target is blended over its own pixels.
 *   Per-view Depth range.  View i's list is its visible entries in sort order, then its culled entries in ascending
 *     index; its Depth colours (a Depth entity's rgba, every entity's out_depth) are over the distances of that list's
 *     sorted[n-1] / sorted[1], n the entity list's count -- bgs_render_entities_aux's rule for view i alone, including a
 *     view with 0 or 1 visible gaussians, a view with none culled, and black Depth colours when n < 2.
 *   Index space, sort, tiles, one round, hooks and stats: bgs_render_views' (segment i k + j, view i's global indices
 *     [i n, (i + 1) n), N = v n below 2^30, one stable sort, view after view of tiles, BGS_FLAG_CHUNKS ignored).  Host
 *     targets: the library's frames hold all v frames of each kind, and each view's three are copied out to its targets.
 *   v == 1.  The call is bgs_render_entities_aux: all three frames, hooks, stats and launch count.
 *   Synchronous only.
 * Launches: those of one bgs_render_entities_aux frame of the same entities, whatever v is (v >= 2: the per-view Depth
 *   range in place of the frame's, as one launch).
 * Refused with BGS_EINVAL, nothing enqueued or written and the previous frame's debug hooks kept: every refusal
 *   bgs_render_entities_aux makes for some view; v == 0, v k > BGS_SCENE_MAX_CLOUDS or N >= 2^30; a NULL out_rgba,
 *   out_depth or out_normal, or a NULL entry of one; a device target not aligned to its pixel (each of the 3 v);
 *   BGS_FLAG_ASYNC; a Gaussian4d cloud, a precomputed-covariance cloud, an entity in Velocity mode (as
 *   bgs_render_entities_aux); an entity in OpticalFlow mode (one previous view per frame); BGS_FLAG_BLEND_OVER_TARGET with
 *   host targets.  NULL clouds, uniforms, entities, views or frame -> BGS_NOT_READY. */
bgs_status bgs_render_views_aux(bgs_context* ctx, const bgs_cloud* const* clouds, const bgs_cloud_uniform* uniforms,
                                const bgs_entity_settings* entities, const uint32_t* entity_flags /* k, or NULL */,
                                uint32_t k, const bgs_view* views, uint32_t v, const bgs_settings* frame,
                                const bgs_scene_depth* depths /* v, or NULL */, void* const* out_rgba /* v */,
                                void* const* out_depth /* v */, void* const* out_normal /* v */,
                                uint32_t out_format, int out_is_device_ptr);

/* Wait for every frame enqueued with BGS_FLAG_ASYNC.  BGS_OK: the last frame is complete and valid.
 * BGS_NOT_READY: a frame's (splat, tile) pair list outgrew its buffer (scene/camera changed a
 * lot); the buffer has been grown -- render that frame again.  An overflowed frame leaves its target
 * as it was (see BGS_FLAG_BLEND_OVER_TARGET).  A no-op after a synchronous render. */
bgs_status bgs_sync(bgs_context* ctx);

/* Parity / debug hooks (valid after a completed bgs_render on this context). */
/* n*2 words (key, index): the reference's sorted_entry_buffer (sort/mod.rs:323-329). */
bgs_status bgs_debug_sorted_entries(bgs_context* ctx, uint32_t* key_index_pairs);
/* tiles*2 words (start, end) into the per-tile entry list.  The two tile hooks need a one-round frame
 * (BGS_NOT_READY after a multi-round one: render with BGS_FLAG_NO_CHUNKS). */
bgs_status bgs_debug_tile_ranges(bgs_context* ctx, uint32_t* start_end);
/* n_pairs words: front-to-back rank of each (tile, splat) pair, tile-major. */
bgs_status bgs_debug_tile_entries(bgs_context* ctx, uint32_t* ranks, uint64_t capacity);
/* n_visible records of 12 floats: cx, cy, ux, uy, vx, vy, bbox(2 words), r, g, b, opacity;
 * and n_visible gaussian indices (front-to-back rank -> index). */
bgs_status bgs_debug_projected(bgs_context* ctx, float* records, uint32_t* rank_to_index);
/* n_visible floats: each splat's depth d (bgs_render_depth_test's rule) in front-to-back rank order, the order of
 * bgs_debug_projected.  Valid after a completed depth-tested frame (else BGS_NOT_READY). */
bgs_status bgs_debug_splat_depths(bgs_context* ctx, float* out);
bgs_status bgs_frame_stats_get(bgs_context* ctx, bgs_frame_stats* out);

/* Last frame's stage times (CUDA events on the context stream), microseconds:
 * [0] key-gen, [1] depth sort, [2] projection, [3] binning + tile sort + ranges,
 * [4] raster, [5] whole frame.  (Multi-round frames: [3] also holds the earlier rounds' blends,
 * [4] the last round's.) */
bgs_status bgs_stage_times_us(bgs_context* ctx, float out[6]);
const char* bgs_last_error(const bgs_context* ctx);
/* The CUDA stream (cudaStream_t) all of this context's work is launched on. */
void* bgs_context_stream(bgs_context* ctx);
/* The copy/comm stream (cudaStream_t): async frames delivered to host memory or gathered over NCCL are consumed here,
 * so device-side timing of a multi-frame window must cover this stream as well as the render stream. */
void* bgs_context_copy_stream(bgs_context* ctx);
/* Device pointer of the last frame in `out_format` layout (valid until the next render). */
const void* bgs_frame_device_ptr(bgs_context* ctx);
/* Kernel launches issued by the last bgs_render. */
uint32_t bgs_last_launch_count(const bgs_context* ctx);

/* Frame hand-back without a copy (SURVEY.md §8 f4).  bgs_frame_export_create allocates a frame target in memory that is
 * exportable as a POSIX file descriptor: pass *out_device_ptr to bgs_render as out_rgba with out_is_device_ptr = 1, and
 * hand *out_fd (+ *out_alloc_bytes) to the graphics API -- Vulkan / wgpu-hal import it with VK_KHR_external_memory_fd
 * (VkImportMemoryFdInfoKHR, handle type OPAQUE_FD) as the memory behind the view-target image or a staging buffer
 * (INTEGRATION.md §6).  The fd is owned by the caller (importing into Vulkan transfers that ownership).
 * bgs_frame_export_import is the consumer side in CUDA terms (another process / library maps the same allocation); the
 * tests use it to prove the exported handle carries the rendered frame.  bgs_frame_export_destroy unmaps and releases a
 * pointer returned by either call. */
bgs_status bgs_frame_export_create(int cuda_device, size_t bytes, void** out_device_ptr, int* out_fd, size_t* out_alloc_bytes);
bgs_status bgs_frame_export_import(int cuda_device, int fd, size_t alloc_bytes, void** out_device_ptr);
void bgs_frame_export_destroy(void* device_ptr);

/* Multi-GPU (one view per GPU, replicated cloud): gather every rank's frame to `root`.
 * nccl_comm is an ncclComm_t.  Enqueued on the context's streams (a frame produced by an async
 * bgs_render is gathered on the copy/comm stream so the next frame overlaps the transfer);
 * bgs_sync() completes it. */
bgs_status bgs_nccl_unique_id(void* out_id128 /* 128 bytes */);
bgs_status bgs_nccl_comm_init(bgs_context* ctx, int nranks, int rank, const void* id128, void** out_comm);
void bgs_nccl_comm_destroy(void* nccl_comm);
bgs_status bgs_gather_frames(bgs_context* ctx, void* nccl_comm, int root, const void* local_frame,
                             void* all_frames, size_t bytes);

/* Copy-engine alternative to bgs_gather_frames (same contract: rank r's frame lands at all_frames + r * bytes on the
 * root), reported beside the NCCL gather by bench.py (`gather_ce`).  The root creates its frame array exportable
 * (bgs_peer_buffer_create -> 64-byte CUDA IPC handle, shipped to the other ranks by the host's own channel); every other
 * rank -- a separate process -- opens it (bgs_peer_buffer_open) and pushes each finished frame with bgs_push_frame: a
 * peer-to-peer copy over NVLink on the sender's copy/comm stream, no SM on either side.  The root itself pushes into its
 * own array (index = its rank).  Completion on the root is the host's to establish (the bench: sync + barrier).
 * bgs_peer_buffer_release(ptr, opened): opened != 0 for pointers from bgs_peer_buffer_open. */
bgs_status bgs_peer_buffer_create(int cuda_device, size_t bytes, void** out_ptr, void* out_handle64);
bgs_status bgs_peer_buffer_open(int cuda_device, const void* handle64, void** out_ptr);
void bgs_peer_buffer_release(void* ptr, int opened);
bgs_status bgs_push_frame(bgs_context* ctx, const void* local_frame, void* remote_frames, int index, size_t bytes);

/* Device-side completion for the copy-engine gather.  bgs_push_frame_signal = bgs_push_frame, then the 32-bit word
 * remote_flags[index] is set to `sequence` by the same stream (ordered after the copy; the words live in the peer buffer,
 * e.g. behind the frames, and start at 0 -- bgs_peer_buffer_create clears the allocation).  bgs_wait_frames makes
 * `cuda_stream` (a CUstream / cudaStream_t of the consumer, NULL = the legacy default stream) wait until
 * flags[0..count) have all reached `sequence` (cyclic >=, so sequences may wrap): work queued behind it sees every
 * frame of that step.  Senders use increasing sequences (frame number + 1).  When local_frame IS the slot
 * (remote_frames + index * bytes) -- the frame was rendered straight into the peer buffer by passing that address to
 * bgs_render as a device target, so the blend kernel's own stores crossed NVLink -- no copy is queued, only the word.  No host round-trip and no cross-process
 * event is involved; the caller must make sure every awaited push is eventually queued, or the stream never resumes.
 * Replaces: the queue-submission order that makes a finished view target visible to its consumer in the reference
 * (src/render/mod.rs:1501-1569 draws inside the view's render pass; here the producer is another process / GPU). */
bgs_status bgs_push_frame_signal(bgs_context* ctx, const void* local_frame, void* remote_frames, int index, size_t bytes,
                                 void* remote_flags, uint32_t sequence);
bgs_status bgs_wait_frames(void* cuda_stream, const void* flags, int count, uint32_t sequence);

#ifdef __cplusplus
}
#endif
#endif
