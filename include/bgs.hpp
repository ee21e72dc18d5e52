// bgs.hpp -- C++ host mirror of the reference's plugin surface for the forward splat path, header-only,
// layered strictly above the C ABI of bgs.h.  (The reference host is Rust; no Rust toolchain exists in the
// build image, so the compiled-language host side is C++.  INTEGRATION.md has the Rust binding.)
//
// Names and defaults follow mosure/bevy_gaussian_splatting:
//   CloudSettings + enums            src/gaussian/settings.rs:6-133
//   PlanarGaussian3d                 src/gaussian/formats/planar_3d.rs:28-54 (struct of four planes)
//   random_gaussians_3d_seeded       src/gaussian/formats/planar_3d.rs:120-191 (distributions + field order)
//   GaussianCamera                   src/camera.rs:6-9
//   ParticleBehaviors                src/morph/particle.rs:349-410 (random_particle_behaviors: distributions)
//   GaussianSplattingPlugin          src/lib.rs:48-80 -- here: owns the bgs_context of one GPU; render_view() is
//                                    run_radix_sort (src/sort/radix.rs:616-756) + DrawGaussians
//                                    (src/render/mod.rs:986-992) for one view
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "bgs.h"

namespace bgs {

enum class DrawMode : uint32_t { All = 0, Selected = 1, HighlightSelected = 2 };
enum class GaussianMode : uint32_t { Gaussian2d = 0, Gaussian3d = 1, Gaussian4d = 2 };
enum class RasterizeMode : uint32_t {
    Color = 0, Depth = 1, Normal = 2, Position = 3, Classification = 4, OpticalFlow = 5, Velocity = 6 /* Gaussian4d only */
};
enum class RadixSortDepthBits : uint32_t { Bits16 = 16, Bits24 = 24, Bits32 = 32 };
enum class GaussianColorSpace : uint32_t { SrgbRec709Display = 0, LinRec709Display = 1 };

struct CloudSettings {   // src/gaussian/settings.rs:110-133 (defaults)
    bool aabb = false;
    float global_opacity = 1.0f;
    float global_scale = 1.0f;
    bool opacity_adaptive_radius = true;
    bool visualize_bounding_box = false;   // the band around each splat's quad (BGS_FLAG_VISUALIZE_BOUNDING_BOX)
    RadixSortDepthBits radix_sort_depth_bits = RadixSortDepthBits::Bits32;
    DrawMode draw_mode = DrawMode::All;
    GaussianMode gaussian_mode = GaussianMode::Gaussian3d;
    RasterizeMode rasterize_mode = RasterizeMode::Color;
    GaussianColorSpace color_space = GaussianColorSpace::SrgbRec709Display;
    uint32_t num_classes = 1;   // RasterizeMode::Classification's hue count (CloudUniform.num_classes)
    float time = 0.0f;
    float time_start = 0.0f;   // the interpolation window (GaussianSplattingPlugin::interpolate), a 4D cloud's playback window
    float time_stop = 1.0f;
    // this repo's extension: front-to-back binning rounds (BGS_FLAG_CHUNKS): -1 = the library's choice from the last
    // frame's footprint statistics, 1 = always, 0 = never (the tile debug hooks need a one-round frame)
    int binning_rounds = -1;

    bgs_settings to_abi(uint32_t flags = 0) const {
        if (binning_rounds >= 0) flags |= binning_rounds ? BGS_FLAG_CHUNKS : BGS_FLAG_NO_CHUNKS;
        if (visualize_bounding_box) flags |= BGS_FLAG_VISUALIZE_BOUNDING_BOX;
        bgs_settings s{};
        s.gaussian_mode = (uint32_t)gaussian_mode; s.rasterize_mode = (uint32_t)rasterize_mode;
        s.aabb = aabb; s.opacity_adaptive_radius = opacity_adaptive_radius; s.draw_mode = (uint32_t)draw_mode;
        s.radix_sort_depth_bits = (uint32_t)radix_sort_depth_bits; s.flags = flags;
        return s;
    }
};

struct SparseSelect {   // src/query/sparse.rs:24-38 (defaults): the floater filter
    float radius = 0.05f;
    uint32_t neighbor_threshold = 3;
};

struct ShaderDefines {   // src/render/mod.rs:698-760: the radix pass plan
    uint32_t radix_bits_per_digit, radix_digit_places, radix_key_shift, radix_base;
    static ShaderDefines for_radix_depth_bits(RadixSortDepthBits b) {
        const uint32_t bits = (uint32_t)b;
        return {8u, bits / 8u, 32u - bits, 256u};
    }
    uint32_t radix_initial_parity() const { return radix_digit_places % 2u; }
};

struct PlanarGaussian4d {   // five planes, binding order (planar_4d.rs:38-51); bgs_cloud_upload_4d's
    std::vector<float> position_visibility;     // n*4
    std::vector<float> spherindrical_harmonic;  // n*144: SH-3 colour, cos(2 pi t) set, cos(4 pi t) set
    std::vector<float> isotropic_rotations;     // n*8: rotation (w, x, y, z), rotation_r (w, x, y, z)
    std::vector<float> scale_opacity;           // n*4
    std::vector<float> timestamp_timescale;     // n*4: timestamp, timescale, pad, pad
    size_t len() const { return position_visibility.size() / 4; }
};

// SH degree d (bgs.h): S_d floats per gaussian in the SH plane
inline size_t sh_width(uint32_t sh_degree) { return sh_degree == 0 ? 4 : sh_degree == 1 ? 12 : sh_degree == 2 ? 28 : 48; }

struct PlanarGaussian3d {   // four planes, binding order (planar_3d.rs:45-54)
    std::vector<float> position_visibility;   // n*4
    std::vector<float> spherical_harmonic;    // n*S_d, sh[3k + c] (S_d = sh_width(sh_degree))
    std::vector<float> rotation;              // n*4, (w, x, y, z)
    std::vector<float> scale_opacity;         // n*4
    uint32_t sh_degree = 3;                   // 0..3
    size_t len() const { return position_visibility.size() / 4; }
    // the entity Aabb's min()/max(): compute_aabb (interface.rs:22-66, positions +- 0.1) -> Aabb {center, half_extents}
    // (cloud.rs:45-62) -> center -+ half_extents (render/mod.rs:1070-1071), all in f32
    void compute_aabb(float mn[3], float mx[3]) const {
        for (int k = 0; k < 3; ++k) {
            float lo = INFINITY, hi = -INFINITY;
            for (size_t i = 0; i < len(); ++i) {
                const float p = position_visibility[4 * i + k];
                lo = std::fmin(lo, p - 0.1f); hi = std::fmax(hi, p + 0.1f);
            }
            const float center = (lo + hi) / 2.0f, half = (hi - lo) / 2.0f;
            mn[k] = center - half; mx[k] = center + half;
        }
    }
};

// splitmix64-based counter PRNG: this repo's generator for the C++ host (the reference's ChaCha stream is not
// reproduced; SURVEY.md §8c).  Same distributions and field order as planar_3d.rs:120-168.
inline PlanarGaussian3d random_gaussians_3d_seeded(size_t n, uint64_t seed) {
    PlanarGaussian3d c;
    c.position_visibility.resize(n * 4); c.spherical_harmonic.resize(n * 48); c.rotation.resize(n * 4); c.scale_opacity.resize(n * 4);
    uint64_t ctr = seed * 0x9E3779B97F4A7C15ull + 0x1234567ull;
    auto uni = [&ctr]() {
        uint64_t z = (ctr += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
        return (float)(z >> 40) * (1.0f / 16777216.0f);   // [0, 1)
    };
    for (size_t i = 0; i < n; ++i) {
        for (int k = 0; k < 4; ++k) c.rotation[4 * i + k] = uni() * 2.0f - 1.0f;
        for (int k = 0; k < 3; ++k) c.position_visibility[4 * i + k] = uni() * 40.0f - 20.0f;
        c.position_visibility[4 * i + 3] = 1.0f;
        for (int k = 0; k < 3; ++k) c.scale_opacity[4 * i + k] = uni();
        c.scale_opacity[4 * i + 3] = uni() * 0.8f;
        for (int k = 0; k < 48; ++k) c.spherical_harmonic[48 * i + k] = uni() * 2.0f - 1.0f;
    }
    return c;
}

// random_particle_behaviors (particle.rs:374-410): behaviour i moves gaussian i; velocity U(-1, 1), acceleration
// U(-0.01, 0.01), jerk U(-1e-4, 1e-4) in all four lanes.  The same splitmix64 stream as above, seeded.
using ParticleBehaviors = std::vector<bgs_particle_behavior>;
// one pixel of a pick frame (bgs_render_entities_pick): entity, gaussian index, blend weight, splat depth
using Pick = bgs_pick;
inline ParticleBehaviors random_particle_behaviors(size_t n, uint64_t seed) {
    ParticleBehaviors b(n);
    uint64_t ctr = seed * 0x9E3779B97F4A7C15ull + 0x7654321ull;
    auto uni = [&ctr]() {
        uint64_t z = (ctr += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
        return (float)(z >> 40) * (1.0f / 16777216.0f);   // [0, 1)
    };
    for (size_t i = 0; i < n; ++i) {
        b[i].indices[0] = (uint32_t)i;
        b[i].indices[1] = b[i].indices[2] = b[i].indices[3] = 0;
        for (int k = 0; k < 4; ++k) b[i].acceleration[k] = (uni() * 2.0f - 1.0f) * 0.01f;
        for (int k = 0; k < 4; ++k) b[i].jerk[k] = (uni() * 2.0f - 1.0f) * 1e-4f;
        for (int k = 0; k < 4; ++k) b[i].velocity[k] = uni() * 2.0f - 1.0f;
    }
    return b;
}

struct GaussianCamera { bool warmup = false; };   // src/camera.rs:6-9

// Column-major 4x4 helpers (Bevy/glam conventions).
struct Mat4 {
    float m[16];
    static Mat4 identity() { Mat4 r{}; r.m[0] = r.m[5] = r.m[10] = r.m[15] = 1.0f; return r; }
    Mat4 operator*(const Mat4& b) const {   // f32 arithmetic like glam
        Mat4 r{};
        for (int c = 0; c < 4; ++c) for (int rr = 0; rr < 4; ++rr) {
            float s = 0.0f;
            for (int k = 0; k < 4; ++k) s += m[k * 4 + rr] * b.m[c * 4 + k];
            r.m[c * 4 + rr] = s;
        }
        return r;
    }
};
inline Mat4 perspective_infinite_reverse_rh(float fov_y, float aspect, float z_near) {
    const float f = 1.0f / std::tan(0.5f * fov_y);
    Mat4 r{};
    r.m[0] = f / aspect; r.m[5] = f; r.m[11] = -1.0f; r.m[14] = z_near;
    return r;
}
inline Mat4 view_from_translation(float x, float y, float z) {   // camera with identity rotation at (x, y, z)
    Mat4 r = Mat4::identity();
    r.m[12] = -x; r.m[13] = -y; r.m[14] = -z;
    return r;
}
inline bgs_view make_view(const Mat4& view_from_world, const Mat4& clip_from_view, const float eye[3], int w, int h) {
    bgs_view v{};
    std::memcpy(v.view_from_world, view_from_world.m, 64);
    std::memcpy(v.clip_from_view, clip_from_view.m, 64);
    const Mat4 cw = clip_from_view * view_from_world;
    std::memcpy(v.clip_from_world, cw.m, 64);
    std::memcpy(v.world_position, eye, 12);
    v.viewport[0] = 0; v.viewport[1] = 0; v.viewport[2] = (float)w; v.viewport[3] = (float)h;
    return v;
}
// examples/headless.rs:177-184: Camera3d at (0, 1.5, 5), identity rotation, default perspective
inline bgs_view headless_view(int w = 1920, int h = 1080) {
    const float eye[3] = {0.0f, 1.5f, 5.0f};
    return make_view(view_from_translation(eye[0], eye[1], eye[2]),
                     perspective_infinite_reverse_rh(3.14159265358979323846f / 4.0f, (float)w / (float)h, 0.1f), eye, w, h);
}

class Error : public std::runtime_error {
public:
    Error(bgs_status st, const std::string& msg) : std::runtime_error(msg), status(st) {}
    bgs_status status;
};

class GaussianSplattingPlugin;

class PlanarGaussian3dHandle {   // a cloud resident in HBM
public:
    PlanarGaussian3dHandle() = default;
    PlanarGaussian3dHandle(const PlanarGaussian3dHandle&) = delete;
    PlanarGaussian3dHandle& operator=(const PlanarGaussian3dHandle&) = delete;
    PlanarGaussian3dHandle(PlanarGaussian3dHandle&& o) noexcept : h_(o.h_), n_(o.n_), temporal_(o.temporal_) {
        std::memcpy(aabb_min_, o.aabb_min_, 12); std::memcpy(aabb_max_, o.aabb_max_, 12); o.h_ = nullptr;
    }
    const float* aabb_min() const { return aabb_min_; }
    const float* aabb_max() const { return aabb_max_; }
    ~PlanarGaussian3dHandle() { if (h_) bgs_cloud_destroy(h_); }
    bgs_cloud* get() const { return h_; }
    uint32_t len() const { return n_; }
    bool temporal() const { return temporal_; }   // a Gaussian4d cloud (PlanarGaussian4dHandle)
private:
    friend class GaussianSplattingPlugin;
    bgs_cloud* h_ = nullptr;
    uint32_t n_ = 0;
    bool temporal_ = false;
    float aabb_min_[3] = {0, 0, 0}, aabb_max_[3] = {1, 1, 1};
};

// a Gaussian4d cloud resident in HBM (bgs_cloud_upload_4d): rendered by render_view_4d, or by render_scene among other
// entities.  The calls on a cloud's positions and visibility take it through get() as they take a 3D one
class PlanarGaussian4dHandle : public PlanarGaussian3dHandle {};

class ParticleBehaviorsHandle {   // a ParticleBehaviors asset resident in HBM (bgs_particles)
public:
    ParticleBehaviorsHandle() = default;
    ParticleBehaviorsHandle(const ParticleBehaviorsHandle&) = delete;
    ParticleBehaviorsHandle& operator=(const ParticleBehaviorsHandle&) = delete;
    ParticleBehaviorsHandle(ParticleBehaviorsHandle&& o) noexcept : h_(o.h_), count_(o.count_) { o.h_ = nullptr; }
    ~ParticleBehaviorsHandle() { if (h_) bgs_particles_destroy(h_); }
    bgs_particles* get() const { return h_; }
    uint32_t len() const { return count_; }
private:
    friend class GaussianSplattingPlugin;
    bgs_particles* h_ = nullptr;
    uint32_t count_ = 0;
};

class GaussianSplattingPlugin {
public:
    explicit GaussianSplattingPlugin(int cuda_device = 0) {
        const bgs_status st = bgs_context_create(cuda_device, &ctx_);
        if (st != BGS_OK) throw Error(st, "bgs_context_create failed: no usable CUDA device (there is no CPU fallback)");
    }
    GaussianSplattingPlugin(const GaussianSplattingPlugin&) = delete;
    GaussianSplattingPlugin& operator=(const GaussianSplattingPlugin&) = delete;
    ~GaussianSplattingPlugin() { bgs_context_destroy(ctx_); }

    PlanarGaussian3dHandle add_cloud(const PlanarGaussian3d& c) {   // asset prepare, at the cloud's SH degree
        if (c.sh_degree > 3 || c.spherical_harmonic.size() != c.len() * sh_width(c.sh_degree))
            throw Error(BGS_EINVAL, "add_cloud: spherical_harmonic must hold sh_width(sh_degree) floats per gaussian");
        PlanarGaussian3dHandle h;
        h.n_ = (uint32_t)c.len();
        c.compute_aabb(h.aabb_min_, h.aabb_max_);
        check(bgs_cloud_upload_f32_sh(ctx_, h.n_, c.sh_degree, c.position_visibility.data(), c.spherical_harmonic.data(),
                                      c.rotation.data(), c.scale_opacity.data(), &h.h_));
        return h;
    }
    PlanarGaussian4dHandle add_cloud(const PlanarGaussian4d& c) {
        PlanarGaussian4dHandle h;
        h.n_ = (uint32_t)c.len();
        h.temporal_ = true;
        for (int k = 0; k < 3; ++k) {   // the Aabb as PlanarGaussian3d::compute_aabb makes it, from the positions
            float lo = INFINITY, hi = -INFINITY;
            for (size_t i = 0; i < c.len(); ++i) {
                lo = std::fmin(lo, c.position_visibility[4 * i + k]); hi = std::fmax(hi, c.position_visibility[4 * i + k]);
            }
            lo -= 0.1f; hi += 0.1f;
            const float center = (lo + hi) / 2.0f, half = (hi - lo) / 2.0f;
            h.aabb_min_[k] = center - half; h.aabb_max_[k] = center + half;
        }
        check(bgs_cloud_upload_4d(ctx_, h.n_, c.position_visibility.data(), c.spherindrical_harmonic.data(),
                                  c.isotropic_rotations.data(), c.scale_opacity.data(), c.timestamp_timescale.data(), &h.h_));
        return h;
    }
    static bgs_cloud_uniform cloud_uniform(const CloudSettings& s, const Mat4& transform = Mat4::identity()) {
        bgs_cloud_uniform u{};
        std::memcpy(u.transform, transform.m, 64);
        u.global_opacity = s.global_opacity; u.global_scale = s.global_scale;
        u.color_space = (uint32_t)s.color_space; u.time = s.time;
        u.aabb_min[3] = u.aabb_max[3] = 1.0f;
        for (int k = 0; k < 3; ++k) u.aabb_max[k] = 1.0f;
        return u;
    }
    // One view of one cloud.  Returns false when the frame is skipped (warm-up camera / not ready), like the
    // reference's silent skip (src/render/mod.rs:361-371, src/sort/radix.rs:645-658).
    // `extra_flags`: BGS_FLAG_BLEND_OVER_TARGET (blend over what the target holds: one call per cloud, far cloud first, as
    // the reference's Transparent3d items do, render/mod.rs:398-452, :944-948), BGS_FLAG_PREMULTIPLIED_OUT (the layer alone).
    bool render_view(const PlanarGaussian3dHandle& cloud, const CloudSettings& settings, const bgs_view& view, void* out_rgba,
                     uint32_t format = BGS_FORMAT_RGBA8_SRGB, const GaussianCamera& camera = {}, bool out_is_device = false,
                     uint32_t extra_flags = 0) {
        if (camera.warmup) return false;
        bgs_cloud_uniform u = cloud_uniform(settings);
        std::memcpy(u.aabb_min, cloud.aabb_min(), 12); std::memcpy(u.aabb_max, cloud.aabb_max(), 12);
        const bgs_settings s = settings.to_abi(extra_flags);
        bgs_render_extras ex{};   // Classification's num_classes; no previous view (OpticalFlow takes the overload below)
        ex.num_classes = settings.num_classes;
        const bgs_status st = bgs_render_ex(ctx_, cloud.get(), &view, &u, &s,
                                            settings.rasterize_mode == RasterizeMode::OpticalFlow ? nullptr : &ex, out_rgba,
                                            format, out_is_device ? 1 : 0);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    // RasterizeMode::OpticalFlow needs the view's previous frame: its clip_from_world and the seconds since
    // (bgs_render_ex); RasterizeMode::Classification reads settings.num_classes.
    bool render_view(const PlanarGaussian3dHandle& cloud, const CloudSettings& settings, const bgs_view& view,
                     const bgs_view& previous_view, float delta_time, void* out_rgba, uint32_t format = BGS_FORMAT_RGBA8_SRGB,
                     bool out_is_device = false, uint32_t extra_flags = 0) {
        bgs_cloud_uniform u = cloud_uniform(settings);
        std::memcpy(u.aabb_min, cloud.aabb_min(), 12); std::memcpy(u.aabb_max, cloud.aabb_max(), 12);
        const bgs_settings s = settings.to_abi(extra_flags);
        bgs_render_extras ex{};
        std::memcpy(ex.previous_clip_from_world, previous_view.clip_from_world, 64);
        ex.delta_time = delta_time;
        ex.num_classes = settings.num_classes;
        const bgs_status st = bgs_render_ex(ctx_, cloud.get(), &view, &u, &s, &ex, out_rgba, format, out_is_device ? 1 : 0);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    // A Gaussian4d cloud at settings.time in [settings.time_start, settings.time_stop] (bgs_render_4d; settings.gaussian_mode
    // must be Gaussian4d).  `previous_view` / `delta_time`: OpticalFlow's (nullptr otherwise); `depth` / `pitch_bytes`: the
    // scene's depth buffer as render_view_depth_test takes it (nullptr: no depth test).
    bool render_view_4d(const PlanarGaussian4dHandle& cloud, const CloudSettings& settings, const bgs_view& view, void* out_rgba,
                        uint32_t format = BGS_FORMAT_RGBA8_SRGB, const bgs_view* previous_view = nullptr, float delta_time = 0.0f,
                        const float* depth = nullptr, uint64_t pitch_bytes = 0, bool out_is_device = false,
                        uint32_t extra_flags = 0) {
        bgs_cloud_uniform u = cloud_uniform(settings);
        std::memcpy(u.aabb_min, cloud.aabb_min(), 12); std::memcpy(u.aabb_max, cloud.aabb_max(), 12);
        const bgs_settings s = settings.to_abi(extra_flags);
        bgs_render_extras ex{};
        ex.num_classes = settings.num_classes;
        if (previous_view) {
            std::memcpy(ex.previous_clip_from_world, previous_view->clip_from_world, 64);
            ex.delta_time = delta_time;
        }
        bgs_scene_depth zd{depth, pitch_bytes};
        const bgs_status st = bgs_render_4d(ctx_, cloud.get(), &view, &u, &s,
                                            settings.rasterize_mode == RasterizeMode::OpticalFlow && !previous_view ? nullptr : &ex,
                                            depth ? &zd : nullptr, out_rgba, format, out_is_device ? 1 : 0, settings.time_start,
                                            settings.time_stop);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    // render_view depth-tested against the scene's depth buffer (bgs_render_depth_test: the reference's GreaterEqual test,
    // no depth writes): `depth` is the view's w x h Depth32Float buffer in device memory of this context's GPU, rows
    // `pitch_bytes` apart.  A queued frame reads it until it completes.
    bool render_view_depth_test(const PlanarGaussian3dHandle& cloud, const CloudSettings& settings, const bgs_view& view,
                                const float* depth, uint64_t pitch_bytes, void* out_rgba,
                                uint32_t format = BGS_FORMAT_RGBA8_SRGB, const GaussianCamera& camera = {},
                                bool out_is_device = false, uint32_t extra_flags = 0) {
        if (camera.warmup) return false;
        bgs_cloud_uniform u = cloud_uniform(settings);
        std::memcpy(u.aabb_min, cloud.aabb_min(), 12); std::memcpy(u.aabb_max, cloud.aabb_max(), 12);
        const bgs_settings s = settings.to_abi(extra_flags);
        bgs_render_extras ex{};
        ex.num_classes = settings.num_classes;
        const bgs_scene_depth zd{depth, pitch_bytes};
        const bgs_status st = bgs_render_depth_test(ctx_, cloud.get(), &view, &u, &s,
                                                    settings.rasterize_mode == RasterizeMode::OpticalFlow ? nullptr : &ex,
                                                    &zd, out_rgba, format, out_is_device ? 1 : 0);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    // One cloud entity of a scene frame: its resident cloud, settings and transform
    struct SceneEntity {
        const PlanarGaussian3dHandle* cloud;
        CloudSettings settings;
        Mat4 transform = Mat4::identity();
    };
    // Every cloud entity of one view in one frame (bgs_render_scene): their splats share one depth sort, so clouds that
    // interpenetrate blend splat by splat.  Each entity's global_opacity, global_scale, color_space, transform and aabb
    // go to its own uniform; the other settings are the frame's, taken from entities[0].  `depth` / `pitch_bytes` as render_view_depth_test's (nullptr: no depth test).
    // With a Gaussian4d entity (a PlanarGaussian4dHandle) the frame is bgs_render_scene_4d's: each entity's time and
    // [time_start, time_stop] are its own too, a 4D entity's gaussian_mode is Gaussian4d, and the frame's gaussian_mode is
    // the first non-4D entity's (Gaussian4d when every entity is 4D).
    bool render_scene(const std::vector<SceneEntity>& entities, const bgs_view& view, void* out_rgba,
                      uint32_t format = BGS_FORMAT_RGBA8_SRGB, const bgs_view* previous_view = nullptr, float delta_time = 0.0f,
                      const float* depth = nullptr, uint64_t pitch_bytes = 0, bool out_is_device = false,
                      uint32_t extra_flags = 0) {
        if (entities.empty()) check(BGS_EINVAL);
        std::vector<const bgs_cloud*> clouds;
        std::vector<bgs_cloud_uniform> unis;
        std::vector<bgs_time_window> windows;
        bool temporal = false;
        CloudSettings settings = entities[0].settings;
        settings.gaussian_mode = GaussianMode::Gaussian4d;
        for (const SceneEntity& e : entities) {
            bgs_cloud_uniform u = cloud_uniform(e.settings, e.transform);
            std::memcpy(u.aabb_min, e.cloud->aabb_min(), 12); std::memcpy(u.aabb_max, e.cloud->aabb_max(), 12);
            clouds.push_back(e.cloud->get());
            unis.push_back(u);
            windows.push_back({e.settings.time_start, e.settings.time_stop});
            temporal = temporal || e.cloud->temporal();
        }
        for (auto it = entities.rbegin(); it != entities.rend(); ++it)   // (the first non-4D entity's mode)
            if (!it->cloud->temporal()) settings.gaussian_mode = it->settings.gaussian_mode;
        if (!temporal) settings = entities[0].settings;
        const bgs_settings s = settings.to_abi(extra_flags);
        bgs_render_extras ex{};
        ex.num_classes = settings.num_classes;
        if (previous_view) {
            std::memcpy(ex.previous_clip_from_world, previous_view->clip_from_world, 64);
            ex.delta_time = delta_time;
        }
        const bgs_scene_depth zd{depth, pitch_bytes};
        const bgs_render_extras* exp = settings.rasterize_mode == RasterizeMode::OpticalFlow && !previous_view ? nullptr : &ex;
        const bgs_status st =
            temporal ? bgs_render_scene_4d(ctx_, clouds.data(), unis.data(), windows.data(), (uint32_t)clouds.size(), &view, &s, exp,
                                           depth ? &zd : nullptr, out_rgba, format, out_is_device ? 1 : 0)
                     : bgs_render_scene(ctx_, clouds.data(), unis.data(), (uint32_t)clouds.size(), &view, &s, exp,
                                        depth ? &zd : nullptr, out_rgba, format, out_is_device ? 1 : 0);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    // render_scene with each entity drawn with its own settings (bgs_render_entities_ex): gaussian_mode, rasterize_mode, aabb,
    // opacity_adaptive_radius, draw_mode, num_classes, visualize_bounding_box and [time_start, time_stop] are the entity's;
    // the sort settings and `extra_flags` are the frame's, taken from entities[0].  The arguments are render_scene's.
    bool render_entities(const std::vector<SceneEntity>& entities, const bgs_view& view, void* out_rgba,
                         uint32_t format = BGS_FORMAT_RGBA8_SRGB, const bgs_view* previous_view = nullptr, float delta_time = 0.0f,
                         const float* depth = nullptr, uint64_t pitch_bytes = 0, bool out_is_device = false,
                         uint32_t extra_flags = 0) {
        return entities_call(entities, previous_view, delta_time, extra_flags, [&](const EntitiesArgs& a) {
            const bgs_scene_depth zd{depth, pitch_bytes};
            return bgs_render_entities_ex(ctx_, a.clouds.data(), a.unis.data(), a.ents.data(), a.eflags.data(),
                                          (uint32_t)a.clouds.size(), &view, &a.s, a.ex, depth ? &zd : nullptr, out_rgba, format,
                                          out_is_device ? 1 : 0);
        });
    }
    // render_entities' frame and, from the same pass, its pick frame (bgs_render_entities_pick): out_pick receives w x h
    // Pick records -- per pixel the entity and gaussian index of the pair with the largest blend weight, that weight and
    // the splat's depth, or BGS_PICK_NONE.  out_pick shares out_is_device with out_rgba (a device one 16 B aligned).
    // Synchronous only; the other arguments are render_entities'.
    void render_entities_pick(const std::vector<SceneEntity>& entities, const bgs_view& view, void* out_rgba, void* out_pick,
                              uint32_t format = BGS_FORMAT_RGBA8_SRGB, const bgs_view* previous_view = nullptr,
                              float delta_time = 0.0f, const float* depth = nullptr, uint64_t pitch_bytes = 0,
                              bool out_is_device = false, uint32_t extra_flags = 0) {
        entities_call(entities, previous_view, delta_time, extra_flags, [&](const EntitiesArgs& a) {
            const bgs_scene_depth zd{depth, pitch_bytes};
            return bgs_render_entities_pick(ctx_, a.clouds.data(), a.unis.data(), a.ents.data(), a.eflags.data(),
                                            (uint32_t)a.clouds.size(), &view, &a.s, a.ex, depth ? &zd : nullptr, out_rgba, format,
                                            out_is_device ? 1 : 0, out_pick);
        });
    }
    // render_entities of each of `views` in one frame (bgs_render_views): out_rgba[i] receives views[i]'s frame, byte for
    // byte render_entities' frame of that view.  depths: one buffer per view (pitches[i] its row pitch), or empty.  No
    // extras: Depth and OpticalFlow entities are refused.
    bool render_views(const std::vector<SceneEntity>& entities, const std::vector<bgs_view>& views,
                      const std::vector<void*>& out_rgba, uint32_t format = BGS_FORMAT_RGBA8_SRGB,
                      const std::vector<const float*>& depths = {}, const std::vector<uint64_t>& pitches = {},
                      bool out_is_device = false, uint32_t extra_flags = 0) {
        if (out_rgba.size() != views.size()) check(BGS_EINVAL);
        return views_call(entities, views, depths, pitches, extra_flags, [&](const ViewsArgs& a) {
            return bgs_render_views(ctx_, a.clouds.data(), a.unis.data(), a.ents.data(), a.eflags.data(), (uint32_t)a.clouds.size(),
                                    views.data(), (uint32_t)views.size(), &a.s, a.zd.empty() ? nullptr : a.zd.data(),
                                    out_rgba.data(), format, out_is_device ? 1 : 0);
        });
    }
    // render_views' frames and each view's depth and normal frames in one pass (bgs_render_views_aux): out_rgba[i],
    // out_depth[i] and out_normal[i] receive views[i]'s three frames, byte for byte bgs_render_entities_aux's of that view.
    // Depth entities are drawn over each view's own range; OpticalFlow entities are refused.  Synchronous only.
    bool render_views_aux(const std::vector<SceneEntity>& entities, const std::vector<bgs_view>& views,
                          const std::vector<void*>& out_rgba, const std::vector<void*>& out_depth,
                          const std::vector<void*>& out_normal, uint32_t format = BGS_FORMAT_RGBA8_SRGB,
                          const std::vector<const float*>& depths = {}, const std::vector<uint64_t>& pitches = {},
                          bool out_is_device = false, uint32_t extra_flags = 0) {
        if (out_rgba.size() != views.size() || out_depth.size() != views.size() || out_normal.size() != views.size())
            check(BGS_EINVAL);
        return views_call(entities, views, depths, pitches, extra_flags, [&](const ViewsArgs& a) {
            return bgs_render_views_aux(ctx_, a.clouds.data(), a.unis.data(), a.ents.data(), a.eflags.data(),
                                        (uint32_t)a.clouds.size(), views.data(), (uint32_t)views.size(), &a.s,
                                        a.zd.empty() ? nullptr : a.zd.data(), out_rgba.data(), out_depth.data(),
                                        out_normal.data(), format, out_is_device ? 1 : 0);
        });
    }
    // Colour + depth + normal frames of one view in one pass (BASELINE.json config 4; bgs_render_aux).
    bool render_view_aux(const PlanarGaussian3dHandle& cloud, const CloudSettings& settings, const bgs_view& view, void* out_rgba,
                         void* out_depth, void* out_normal, uint32_t format = BGS_FORMAT_RGBA8_SRGB, bool out_is_device = false) {
        bgs_cloud_uniform u = cloud_uniform(settings);
        std::memcpy(u.aabb_min, cloud.aabb_min(), 12); std::memcpy(u.aabb_max, cloud.aabb_max(), 12);
        const bgs_settings s = settings.to_abi();
        const bgs_status st = bgs_render_aux(ctx_, cloud.get(), &view, &u, &s, out_rgba, out_depth, out_normal, format, out_is_device ? 1 : 0);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    // Selection edits of a resident cloud: the visibility lane DrawMode::Selected / HighlightSelected read (bgs.h).
    // select_sparse: SparseSelect (src/query/sparse.rs:24-54) on the GPU; returns how many were selected.
    uint32_t select_sparse(PlanarGaussian3dHandle& cloud, const SparseSelect& query = {}) {
        uint32_t selected = 0;
        check(bgs_cloud_select_sparse(ctx_, cloud.get(), query.radius, query.neighbor_threshold, &selected));
        return selected;
    }
    // select_in_mesh: point-in-mesh selection (src/query/raycast.rs:54-124) on the GPU; vertices nv x 3, indices nt x 3,
    // mesh_from_cloud column-major (nullptr = identity), mode BGS_SELECT_REPLACE / BGS_SELECT_ADD; returns how many are inside.
    uint32_t select_in_mesh(PlanarGaussian3dHandle& cloud, const std::vector<float>& vertices, const std::vector<uint32_t>& indices,
                            const float* mesh_from_cloud = nullptr, uint32_t mode = BGS_SELECT_REPLACE) {
        if (vertices.size() % 3 || indices.size() % 3) throw Error(BGS_EINVAL, "select_in_mesh: vertices and indices come in threes");
        uint32_t inside = 0;
        check(bgs_cloud_select_in_mesh(ctx_, cloud.get(), vertices.data(), (uint32_t)(vertices.size() / 3), indices.data(),
                                       (uint32_t)(indices.size() / 3), mesh_from_cloud, mode, &inside));
        return inside;
    }
    // select_in_view: rectangle, lasso and brush selection through the volume (bgs_cloud_select_in_view): a gaussian is
    // inside when the projection with `transform` and `view` finds it in the frustum and mask[floor(cy) w + floor(cx)] is
    // set; mask h x w bytes, host or (mask_is_device) device memory; mode as select_in_mesh's; returns how many are inside.
    uint32_t select_in_view(PlanarGaussian3dHandle& cloud, const bgs_view& view, const uint8_t* mask, bool mask_is_device = false,
                            const Mat4& transform = Mat4::identity(), uint32_t mode = BGS_SELECT_REPLACE) {
        const bgs_cloud_uniform u = cloud_uniform(CloudSettings{}, transform);
        uint32_t inside = 0;
        check(bgs_cloud_select_in_view(ctx_, cloud.get(), &u, &view, mask, mask_is_device ? 1 : 0, mode, &inside));
        return inside;
    }
    std::vector<float> visibility(const PlanarGaussian3dHandle& cloud) {
        std::vector<float> v(cloud.len());
        check(bgs_cloud_visibility_get(ctx_, cloud.get(), v.data()));
        return v;
    }
    void set_visibility(PlanarGaussian3dHandle& cloud, const std::vector<float>& vis) {
        if (vis.size() != cloud.len()) throw Error(BGS_EINVAL, "set_visibility: one value per gaussian");
        check(bgs_cloud_visibility_set(ctx_, cloud.get(), vis.data()));
    }
    // src/query/select.rs:81-110: visibility 0 everywhere, 1 at `indices`
    void apply_selection(PlanarGaussian3dHandle& cloud, const std::vector<uint32_t>& indices) {
        std::vector<float> v(cloud.len(), 0.0f);
        for (uint32_t i : indices) {
            if (i >= cloud.len()) throw Error(BGS_EINVAL, "apply_selection: index out of range");
            v[i] = 1.0f;
        }
        set_visibility(cloud, v);
    }
    // src/query/select.rs:116-150 on a 0/1 lane: visibility == 0 becomes 1, everything else 0
    void invert_selection(PlanarGaussian3dHandle& cloud) {
        std::vector<float> v = visibility(cloud);
        for (float& x : v) x = x == 0.0f ? 1.0f : 0.0f;
        set_visibility(cloud, v);
    }
    // indices with visibility >= 0.5: the gaussians DrawMode::Selected draws
    std::vector<uint32_t> selection(const PlanarGaussian3dHandle& cloud) {
        const std::vector<float> v = visibility(cloud);
        std::vector<uint32_t> idx;
        for (uint32_t i = 0; i < (uint32_t)v.size(); ++i)
            if (v[i] >= 0.5f) idx.push_back(i);
        return idx;
    }
    // Keeping a selection as its own cloud (src/query/select.rs:156-176; the rule: bgs.h).  indices nullptr: the gaussians
    // DrawMode::Selected draws (visibility !(w < 0.5), NaN included), in index order -- an empty handle (get() == nullptr,
    // len() == 0) when none is; else gaussian j of the result is gaussian (*indices)[j].  The Aabb is the new cloud's own.
    PlanarGaussian3dHandle subset(const PlanarGaussian3dHandle& cloud, const std::vector<uint32_t>* indices = nullptr) {
        PlanarGaussian3dHandle h;
        if (indices) check(bgs_cloud_subset(ctx_, cloud.get(), indices->data(), (uint32_t)indices->size(), &h.h_, &h.n_));
        else check(bgs_cloud_subset(ctx_, cloud.get(), nullptr, 0, &h.h_, &h.n_));
        if (h.h_) {
            PlanarGaussian3d p;
            p.position_visibility = positions(h);
            p.compute_aabb(h.aabb_min_, h.aabb_max_);
        }
        return h;
    }
    // A KHR_gaussian_splatting primitive whose accessors the caller has described (bgs_cloud_upload_khr; this header parses
    // no glTF), as an f32 cloud.  *zero_quats (optional): how many zero-length rotations became the identity.
    PlanarGaussian3dHandle upload_khr(const bgs_khr_primitive& primitive, uint32_t* zero_quats = nullptr) {
        PlanarGaussian3dHandle h;
        check(bgs_cloud_upload_khr(ctx_, &primitive, 0, zero_quats, &h.h_));
        h.n_ = primitive.n;
        PlanarGaussian3d p;
        p.position_visibility = positions(h);
        p.compute_aabb(h.aabb_min_, h.aabb_max_);
        return h;
    }
    // The cloud's four planes at its SH degree (bgs_cloud_download_f32_sh: this host uploads f32 clouds only).
    PlanarGaussian3d download(const PlanarGaussian3dHandle& cloud) {
        const size_t n = cloud.len();
        PlanarGaussian3d c;
        check(bgs_cloud_sh_degree(cloud.get(), &c.sh_degree));
        c.position_visibility.resize(n * 4); c.spherical_harmonic.resize(n * sh_width(c.sh_degree)); c.rotation.resize(n * 4);
        c.scale_opacity.resize(n * 4);
        check(bgs_cloud_download_f32_sh(ctx_, cloud.get(), c.position_visibility.data(), c.spherical_harmonic.data(),
                                        c.rotation.data(), c.scale_opacity.data()));
        return c;
    }
    // The reference's save_selection: the selected gaussians written to `path` as .gcloud (bgs::io::encode_gcloud, defined
    // in bgs_io.hpp).  Returns how many were written; nothing selected throws Error(BGS_EINVAL) and writes nothing.
    uint32_t save_selection(const PlanarGaussian3dHandle& cloud, const std::string& path);
    // Particle behaviours (src/morph/particle.rs; the rule and its ordering: bgs.h).  step_particles only enqueues the
    // step: frames rendered before it (on any context) see the old positions, everything after it the new ones.
    ParticleBehaviorsHandle add_particles(const ParticleBehaviors& behaviors) {
        ParticleBehaviorsHandle h;
        h.count_ = (uint32_t)behaviors.size();
        check(bgs_particles_create(ctx_, behaviors.data(), h.count_, &h.h_));
        return h;
    }
    ParticleBehaviors particles(const ParticleBehaviorsHandle& p) {
        ParticleBehaviors b(p.len());
        check(bgs_particles_get(ctx_, p.get(), b.data()));
        return b;
    }
    void step_particles(PlanarGaussian3dHandle& cloud, ParticleBehaviorsHandle& p, float delta_time) {
        check(bgs_cloud_particles_step(ctx_, cloud.get(), p.get(), delta_time));
    }
    // Interpolation (src/morph/interpolate.rs; the rule and its ordering: bgs.h): out := the blend of lhs and rhs at
    // settings.time between settings.time_start and time_stop, enqueued like a particle step.  The three clouds hold the
    // same number of gaussians in one layout; make `out` once as subset(lhs, &indices 0 .. n-1).
    void interpolate(PlanarGaussian3dHandle& out, const PlanarGaussian3dHandle& lhs, const PlanarGaussian3dHandle& rhs,
                     const CloudSettings& settings) {
        check(bgs_cloud_interpolate(ctx_, out.get(), lhs.get(), rhs.get(), settings.time, settings.time_start, settings.time_stop));
    }
    // Transforms (the rule and its ordering: bgs.h): bake the similarity transform m (column-major, in the cloud's own
    // frame: a world-space delta W of an entity with model matrix `model` is model^-1 W model) into every gaussian, or
    // with selected_only into the selected ones, enqueued like a particle step.  The entity's Aabb is not updated:
    // refresh it from bounds().
    void transform(PlanarGaussian3dHandle& cloud, const Mat4& m, bool selected_only = false) {
        check(bgs_cloud_transform(ctx_, cloud.get(), m.m, selected_only ? BGS_TRANSFORM_SELECTED : BGS_TRANSFORM_ALL));
    }
    // bounds: per axis, the min and max of the finite positions of every (or every selected) gaussian, after every write
    // queued on the cloud; count 0 (min +inf, max -inf) when there are none.
    struct Bounds {
        float min[3], max[3];
        uint32_t count;
    };
    Bounds bounds(const PlanarGaussian3dHandle& cloud, bool selected_only = false) {
        Bounds b{};
        check(bgs_cloud_bounds(ctx_, cloud.get(), selected_only ? BGS_TRANSFORM_SELECTED : BGS_TRANSFORM_ALL, b.min, b.max,
                               &b.count));
        return b;
    }
    // update_aabb: the handle's Aabb from the GPU bounds, through compute_aabb's f32 steps (+-0.1, centre, half extents)
    void update_aabb(PlanarGaussian3dHandle& cloud) {
        const Bounds b = bounds(cloud);
        for (int k = 0; k < 3; ++k) {
            const float lo = b.min[k] - 0.1f, hi = b.max[k] + 0.1f;
            const float center = (lo + hi) / 2.0f, half = (hi - lo) / 2.0f;
            cloud.aabb_min_[k] = center - half; cloud.aabb_max_[k] = center + half;
        }
    }
    std::vector<float> positions(const PlanarGaussian3dHandle& cloud) {   // n * 4: x, y, z, visibility
        std::vector<float> v((size_t)cloud.len() * 4);
        check(bgs_cloud_positions_get(ctx_, cloud.get(), v.data()));
        return v;
    }
    bool sync() {   // complete the queued frames and steps; false: the last queued frame must be rendered again
        const bgs_status st = bgs_sync(ctx_);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    bgs_frame_stats frame_stats() { bgs_frame_stats fs{}; check(bgs_frame_stats_get(ctx_, &fs)); return fs; }
    bgs_context* context() const { return ctx_; }

private:
    void check(bgs_status st) { if (st != BGS_OK) throw Error(st, bgs_last_error(ctx_)); }
    // the entity arrays of a render_views / render_views_aux call, and the call made with them (false: BGS_NOT_READY)
    // the arguments of a bgs_render_entities_ex / _pick call of `entities`
    struct EntitiesArgs {
        std::vector<const bgs_cloud*> clouds;
        std::vector<bgs_cloud_uniform> unis;
        std::vector<bgs_entity_settings> ents;
        std::vector<uint32_t> eflags;
        bgs_settings s;
        bgs_render_extras extras;
        const bgs_render_extras* ex;
    };
    template <class Call>
    bool entities_call(const std::vector<SceneEntity>& entities, const bgs_view* previous_view, float delta_time,
                       uint32_t extra_flags, Call call) {
        if (entities.empty()) check(BGS_EINVAL);
        EntitiesArgs a;
        for (const SceneEntity& e : entities) {
            bgs_cloud_uniform u = cloud_uniform(e.settings, e.transform);
            std::memcpy(u.aabb_min, e.cloud->aabb_min(), 12); std::memcpy(u.aabb_max, e.cloud->aabb_max(), 12);
            a.clouds.push_back(e.cloud->get());
            a.unis.push_back(u);
            const bgs_settings s = e.settings.to_abi();
            a.ents.push_back({s.gaussian_mode, s.rasterize_mode, s.aabb, s.opacity_adaptive_radius, s.draw_mode,
                              e.settings.num_classes, {e.settings.time_start, e.settings.time_stop}});
            a.eflags.push_back(e.settings.visualize_bounding_box ? (uint32_t)BGS_ENTITY_VISUALIZE_BOUNDING_BOX : 0u);
        }
        a.s = entities[0].settings.to_abi(extra_flags);
        if (!(extra_flags & BGS_FLAG_VISUALIZE_BOUNDING_BOX)) a.s.flags &= ~(uint32_t)BGS_FLAG_VISUALIZE_BOUNDING_BOX;   // (per entity)
        a.extras = bgs_render_extras{};
        a.extras.num_classes = 1;
        if (previous_view) {
            std::memcpy(a.extras.previous_clip_from_world, previous_view->clip_from_world, 64);
            a.extras.delta_time = delta_time;
        }
        a.ex = previous_view ? &a.extras : nullptr;
        const bgs_status st = call(a);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    struct ViewsArgs {
        std::vector<const bgs_cloud*> clouds;
        std::vector<bgs_cloud_uniform> unis;
        std::vector<bgs_entity_settings> ents;
        std::vector<uint32_t> eflags;
        bgs_settings s;
        std::vector<bgs_scene_depth> zd;
    };
    template <class Call>
    bool views_call(const std::vector<SceneEntity>& entities, const std::vector<bgs_view>& views,
                    const std::vector<const float*>& depths, const std::vector<uint64_t>& pitches, uint32_t extra_flags,
                    Call call) {
        if (entities.empty() || views.empty()) check(BGS_EINVAL);
        if (!depths.empty() && (depths.size() != views.size() || pitches.size() != views.size())) check(BGS_EINVAL);
        ViewsArgs a;
        for (const SceneEntity& e : entities) {
            bgs_cloud_uniform u = cloud_uniform(e.settings, e.transform);
            std::memcpy(u.aabb_min, e.cloud->aabb_min(), 12); std::memcpy(u.aabb_max, e.cloud->aabb_max(), 12);
            a.clouds.push_back(e.cloud->get());
            a.unis.push_back(u);
            const bgs_settings s = e.settings.to_abi();
            a.ents.push_back({s.gaussian_mode, s.rasterize_mode, s.aabb, s.opacity_adaptive_radius, s.draw_mode,
                              e.settings.num_classes, {e.settings.time_start, e.settings.time_stop}});
            a.eflags.push_back(e.settings.visualize_bounding_box ? (uint32_t)BGS_ENTITY_VISUALIZE_BOUNDING_BOX : 0u);
        }
        a.s = entities[0].settings.to_abi(extra_flags);
        if (!(extra_flags & BGS_FLAG_VISUALIZE_BOUNDING_BOX)) a.s.flags &= ~(uint32_t)BGS_FLAG_VISUALIZE_BOUNDING_BOX;   // (per entity)
        for (size_t i = 0; i < depths.size(); ++i) a.zd.push_back({depths[i], pitches[i]});
        const bgs_status st = call(a);
        if (st == BGS_NOT_READY) return false;
        check(st);
        return true;
    }
    bgs_context* ctx_ = nullptr;
};

}  // namespace bgs

#include "bgs_io.hpp"   // GaussianSplattingPlugin::save_selection
