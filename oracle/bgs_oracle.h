/*
 * bgs_oracle.h -- CPU ORACLE for the forward splat path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library.  The product (libbgs.so) never links, loads or calls it.
 *
 * PARITY STATUS (SURVEY.md §8c): the reference (Rust + WGSL over wgpu) cannot be built or run
 * in this image, so this oracle is a CPU *restatement* of the cited WGSL.  It is pinned by
 * the reference's own pure tests for the sort key / pass plan (tests/radix.rs:10-106,
 * restated in tests/test_oracle_radix.py) and by the coarse scene statistics of
 * tests/visibility_render.rs:199-274.  Everything past the sort key (projection, SH colour,
 * coverage, blending) is "parity unpinned": the reference holds no golden vector for it.
 *
 * Fixed FP policy (WGSL leaves evaluation order / contraction to the driver, so "bit-exact"
 * is defined against THIS policy): IEEE-754 binary32, round-to-nearest-even, no FMA
 * contraction (build with -ffp-contract=off), the evaluation orders written in
 * bgs_oracle.cpp; ln() for the adaptive cutoff is a fixed double-precision series;
 * exp()/pow() come from libm and are compared under tolerance only.
 */
#ifndef BGS_ORACLE_H
#define BGS_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Same field layout as bgs_view / bgs_cloud_uniform / bgs_settings in include/bgs.h. */
typedef struct {
    float view_from_world[16], clip_from_view[16], clip_from_world[16]; /* column-major */
    float world_position[3];
    float viewport[4]; /* x, y, w, h in px */
} orc_view;
typedef struct {
    float transform[16];
    float global_opacity, global_scale;
    uint32_t color_space; /* 0 = SrgbRec709Display (decode sRGB->linear), 1 = LinRec709Display */
    float time;
    float aabb_min[4], aabb_max[4]; /* CloudUniform.min / .max (render/mod.rs:1070-1071) */
} orc_uniform;
typedef struct {
    uint32_t gaussian_mode;           /* 0 = Gaussian2d, 1 = Gaussian3d */
    uint32_t rasterize_mode;          /* 0 = Color, 1 = Depth, 2 = Normal, 3 = Position */
    uint32_t aabb;                    /* 0 = USE_OBB, 1 = USE_AABB */
    uint32_t opacity_adaptive_radius; /* bool */
    uint32_t draw_mode;               /* 0 = All, 1 = Selected, 2 = HighlightSelected */
    uint32_t radix_sort_depth_bits;   /* 16 | 24 | 32 */
    uint32_t flags;
    uint32_t reserved;
} orc_settings;

/* Projected splat record (one per visible gaussian), the unit both raster modes consume. */
typedef struct {
    float cx, cy;         /* centre, pixel coordinates (x right, y down) */
    float ux, uy, vx, vy; /* OBB: rows of the pixel-offset -> quad-uv map.  AABB/2DGS: see .cpp */
    float r, g, b, op;    /* linear rgb (unclamped), opacity * global_opacity */
    int32_t xlo, xhi, ylo, yhi; /* conservative pixel bbox (inclusive); xlo > xhi = empty */
    float extra[16];      /* mode-specific (AABB conic+R; 2DGS R, mean, aspect, T0..T2) */
} orc_splat;

/* a2: key-gen, src/sort/radix.wgsl:86-101 + src/render/transform.wgsl:5-14 */
int orc_keygen(uint32_t n, const float* pos_vis, const orc_view* view, const orc_uniform* u,
               uint32_t depth_bits, uint32_t* keys_out);
/* a3: the literal LSD pass structure (src/sort/radix.rs:672-754, src/render/mod.rs:715-745) */
int orc_radix_sort(uint32_t n, const uint32_t* keys, uint32_t depth_bits,
                   uint32_t* sorted_keys, uint32_t* sorted_index);
/* a3 cross-check: std::stable_sort ascending by key */
int orc_stable_sort(uint32_t n, const uint32_t* keys, uint32_t* sorted_index);
/* pass plan (digit places, key shift, initial parity) -- src/render/mod.rs:715-760 */
void orc_pass_plan(uint32_t depth_bits, uint32_t* places, uint32_t* shift, uint32_t* parity);

/* a1/A.9: f16 planar pack / decode -- src/gaussian/f16.rs:38-56,244-263, planar.wgsl:117-176 */
void orc_pack_f16(uint32_t n, const float* sh, const float* rot, const float* scale_opacity,
                  uint32_t* sh_packed /*n*24*/, uint32_t* rso_packed /*n*4*/);
void orc_decode_f16(uint32_t n, const uint32_t* sh_packed, const uint32_t* rso_packed,
                    float* sh, float* rot, float* scale_opacity);

/* f3: src/gaussian/covariance.rs:4-41 -- the f32 upper triangle that Covariance3dOpacityPacked128 stores as f16
 * (f16.rs:131-170).  With orc_settings.reserved bit 0 set, projection / rendering read the decoded record from the
 * plane slots it occupies (rotation = c0..c3, scale_opacity = c4, c5, opacity, opacity) and skip Sigma = M^T M,
 * global_scale and the model 3x3, as PRECOMPUTE_COVARIANCE_3D does (gaussian_3d.wgsl:78-79). */
void orc_covariance_3d(uint32_t n, const float* rot, const float* scale_opacity, float* cov6);

/* a4+a5: per-gaussian projection + colour for the listed ids (gaussian.wgsl:185-436) */
int orc_project(uint32_t n, const float* pos_vis, const float* sh, const float* rot,
                const float* scale_opacity, const orc_view* view, const orc_uniform* u,
                const orc_settings* s, uint32_t count, const uint32_t* ids, orc_splat* out);

/* a6 ref_mode: back-to-front over the sorted quads, no tiles, no early-out.
 * out_rgba = W*H*4 f32 premultiplied linear.  threads<=0 -> all cores. */
int orc_render_ref(uint32_t n, const float* pos_vis, const float* sh, const float* rot,
                   const float* scale_opacity, const orc_view* view, const orc_uniform* u,
                   const orc_settings* s, float* out_rgba, int threads);

/* a6 ref_mode over an initial target (premultiplied linear RGBA, W*H*4; NULL = opaque black clear): the
 * reference's PREMULTIPLIED_ALPHA_BLENDING onto the view target, render/mod.rs:944-948. */
int orc_render_ref_over(uint32_t n, const float* pos_vis, const float* sh, const float* rot,
                        const float* scale_opacity, const orc_view* view, const orc_uniform* u,
                        const orc_settings* s, const float* dst_init, float* out_rgba, int threads);

/* a6+a7 tile_mode: 16x16 tile ranges over the global order, front-to-back, pixel stops at
 * T < 1e-4.  tile_ranges = tiles*2 (start,end into tile_entries); tile_entries holds the
 * front-to-back rank r (0 = nearest visible splat) of each (tile,splat) pair, capacity cap.
 * rank_to_id (n_vis entries, optional) maps rank -> gaussian index. */
int orc_render_tiles(uint32_t n, const float* pos_vis, const float* sh, const float* rot,
                     const float* scale_opacity, const orc_view* view, const orc_uniform* u,
                     const orc_settings* s, float* out_rgba, uint32_t* tile_ranges,
                     uint32_t* tile_entries, uint64_t cap, uint64_t* n_pairs, uint32_t* n_vis,
                     uint32_t* rank_to_id, int threads);

/* Coverage probe: for each pair j, splat record splats[j] at the pixel centre (pixel_xy[2j], pixel_xy[2j+1]), the
 * quantities fs_main's coverage decision turns on, exactly as render_tiles computes them.  u, v: USE_OBB quad uv
 * (|u| <= 1 && |v| <= 1); mx, my, Rq: USE_AABB quad offset and half-side (|mx| <= Rq && |my| <= Rq); power: the
 * exponent (covered pixels; USE_AABB also sets it when only power > 0 rejects).  covered_if_unfused: the decision with
 * u, v from a separately rounded multiply and add instead of the fma. */
typedef struct {
    float u, v, mx, my, Rq, power, alpha;
    uint32_t covered, covered_if_unfused;
} orc_probe;
int orc_coverage_probe(uint32_t count, const orc_splat* splats, const orc_settings* s, const float* pixel_xy,
                       orc_probe* out);

/* Blend trace: the tile_mode walk of render_tiles (same slices, same f32 coverage decisions, same f32 stop index),
 * per pixel (row-major, W*H):
 *   c64, T64: the colour and transmittance of that walk accumulated in float64, alpha = min(exp(power) * op, 0.999)
 *             with exp taken in double of the f32 power -- the exact value of the blend the f32 walk performs;
 *   T:        the f32 transmittance where the walk stopped; n_blended, rank0 / rank1 (first two blended ranks, -1 none);
 *   max_c:    max |r|, |g|, |b| of the blended records; max_power: max |power| of the blended splats;
 *   t_sens:   sum of a / (1 - a) over the blended alphas below the clamp: |dT / T| <= t_sens * (relative alpha error);
 *   w_power, t_sens_power: sum of w64 |power| over the blended splats, sum of a / (1 - a) |power| over the unclamped
 *             ones (for alpha errors that grow with |power|);
 *   stop_margin: min over the T < T_STOP tests of |T / T_STOP - 1|;
 *   flags:    NEAR_STOP (stop_margin <= 1e-5: a kernel computing T another way may stop one splat apart),
 *             NEAR_CLAMP (a blended exp * op within 1e-5 relative of 0.999), UNCLAMPED (a blended exp * op < 0.999). */
#define ORC_TRACE_NEAR_STOP 1u
#define ORC_TRACE_NEAR_CLAMP 2u
#define ORC_TRACE_UNCLAMPED 4u
typedef struct {
    double c64[3], T64, t_sens, stop_margin, w_power, t_sens_power;
    float T;
    uint32_t n_blended;
    int32_t rank0, rank1;
    uint32_t flags;
    float max_c, max_power;
    uint32_t pad;
} orc_trace;
int orc_blend_trace(uint32_t n, const float* pos_vis, const float* sh, const float* rot,
                    const float* scale_opacity, const orc_view* view, const orc_uniform* u,
                    const orc_settings* s, orc_trace* out, int threads);

/* CPU-baseline model of the reference's native CPU sort (src/sort/rayon.rs:86-104):
 * key = bits(|p - cam|^2), parallel unstable sort, descending.  Returns seconds. */
double orc_cpu_sort_model(uint32_t n, const float* pos_vis, const float* cam, int threads,
                          uint32_t* sorted_index);

/* the fixed-series ln() used for the adaptive cutoff (exposed for unit tests) */
float orc_ln(float x);
int orc_num_threads(void);

#ifdef __cplusplus
}
#endif
#endif
