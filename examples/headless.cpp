// headless.cpp -- C++ host example over include/bgs.hpp, the counterpart of the reference's
// examples/headless.rs (offscreen target, camera at (0, 1.5, 5), random cloud, one frame written to disk).
//
//   headless [count=100000] [width=1920] [height=1080] [global_scale=1.0] [out=headless_output/0.ppm]
//            [--dump-cloud file] [--raw file] [--remove-floaters radius]
//            [--particles N --steps K --dt S [--dump-particles file]] [--interpolate SEED --time T]
//            [--rasterize classification|optical-flow] [--num-classes K] [--prev-view dx,dy,dz] [--instances N]
//            [--shutter S]
// --dump-cloud writes the four f32 planes (n, then pos_vis, sh, rot, scale_opacity) so another host can
// render the identical cloud; --raw writes the RGBA8 frame bytes.  --remove-floaters selects the sparse gaussians
// (SparseSelect with that radius), inverts the selection and draws only the rest (DrawMode::Selected), the
// reference converter's floater filter (tools/ply_to_gcloud.rs:54-66) applied to the resident cloud.
// --particles attaches random_particle_behaviors(N, 0) to the cloud and enqueues K steps of S seconds before the frames
// (the reference's morph_particles feature, stepped once per frame); --dump-particles writes N (u64), the behaviours
// before and after the steps (N * 64 B each) and the position plane after them (count * 16 B).
// --interpolate blends the cloud (lhs) with random_gaussians_3d_seeded(count, SEED) (rhs) at time T of the window
// [0, 1] into a third cloud, made as the subset of every gaussian of lhs, and draws that one (the reference's
// GaussianInterpolate { lhs, rhs }); --dump-cloud then writes rhs's four planes after lhs's.
// --instances N draws the cloud instanced N times on a grid through a resident entity list (bgs_entity_list), the
// instances then moved by one set_transforms from a row-major host array.
// --shutter S draws the cloud as one motion-blurred frame of S samples (bgs_render_shutter), sample i moved by 0.25 i in x.
// --rasterize picks RasterizeMode::Classification (labels: gaussian i gets visibility 2 + i % K, --num-classes K, default
// 3) or OpticalFlow (the previous frame's camera is the headless camera moved by --prev-view, default 0.05,0,0, at
// 1/60 s); the previous view's clip_from_world is printed as 16 hex words ("prev_clip: ...").
#include <memory>
#include <numeric>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <string>
#include <sys/stat.h>
#include <dlfcn.h>

#include "../include/bgs.hpp"

int main(int argc, char** argv) {
    size_t count = 100000; int W = 1920, H = 1080; float scale = 1.0f;
    std::string out = "headless_output/0.ppm", dump, raw;
    float floater_radius = 0.0f;
    size_t n_particles = 0; int steps = 0; float dt = 1.0f / 60.0f;
    std::string dump_particles;
    long interp_seed = -1; float interp_time = 0.0f;
    std::string rasterize = "color"; uint32_t num_classes = 3; float prev_off[3] = {0.05f, 0.0f, 0.0f};
    uint32_t instances = 0;      // --instances N: the cloud instanced N times on a grid through an entity list
    uint32_t shutter = 0;        // --shutter S: a motion-blurred frame of S samples
    float depth_plane = -1.0f;   // --depth-plane Z: render depth-tested against a half-frame plane at reverse-Z depth Z
    int pos = 0;
    for (int i = 1; i < argc; ++i) {
        const std::string a = argv[i];
        if (a == "--dump-cloud" && i + 1 < argc) { dump = argv[++i]; continue; }
        if (a == "--raw" && i + 1 < argc) { raw = argv[++i]; continue; }
        if (a == "--remove-floaters" && i + 1 < argc) { floater_radius = (float)std::atof(argv[++i]); continue; }
        if (a == "--particles" && i + 1 < argc) { n_particles = std::strtoull(argv[++i], nullptr, 10); continue; }
        if (a == "--steps" && i + 1 < argc) { steps = std::atoi(argv[++i]); continue; }
        if (a == "--dt" && i + 1 < argc) { dt = (float)std::atof(argv[++i]); continue; }
        if (a == "--dump-particles" && i + 1 < argc) { dump_particles = argv[++i]; continue; }
        if (a == "--interpolate" && i + 1 < argc) { interp_seed = std::atol(argv[++i]); continue; }
        if (a == "--time" && i + 1 < argc) { interp_time = (float)std::atof(argv[++i]); continue; }
        if (a == "--rasterize" && i + 1 < argc) { rasterize = argv[++i]; continue; }
        if (a == "--depth-plane" && i + 1 < argc) { depth_plane = (float)std::atof(argv[++i]); continue; }
        if (a == "--instances" && i + 1 < argc) { instances = (uint32_t)std::strtoul(argv[++i], nullptr, 10); continue; }
        if (a == "--shutter" && i + 1 < argc) { shutter = (uint32_t)std::strtoul(argv[++i], nullptr, 10); continue; }
        if (a == "--num-classes" && i + 1 < argc) { num_classes = (uint32_t)std::strtoul(argv[++i], nullptr, 10); continue; }
        if (a == "--prev-view" && i + 1 < argc) {
            if (std::sscanf(argv[++i], "%f,%f,%f", &prev_off[0], &prev_off[1], &prev_off[2]) != 3) return 1;
            continue;
        }
        switch (pos++) {
            case 0: count = std::strtoull(a.c_str(), nullptr, 10); break;
            case 1: W = std::atoi(a.c_str()); break;
            case 2: H = std::atoi(a.c_str()); break;
            case 3: scale = (float)std::atof(a.c_str()); break;
            case 4: out = a; break;
        }
    }
    try {
        bgs::GaussianSplattingPlugin plugin(0);
        const bgs::PlanarGaussian3d cloud = bgs::random_gaussians_3d_seeded(count, 0);
        bgs::PlanarGaussian3dHandle handle = plugin.add_cloud(cloud);
        bgs::CloudSettings settings;
        settings.global_scale = scale;
        if (floater_radius > 0.0f) {
            bgs::SparseSelect query;
            query.radius = floater_radius;
            const uint32_t sparse = plugin.select_sparse(handle, query);
            plugin.invert_selection(handle);
            settings.draw_mode = bgs::DrawMode::Selected;
            std::printf("floaters: %u of %zu gaussians hidden\n", sparse, count);
        }
        if (n_particles > 0) {
            const bgs::ParticleBehaviors behaviors = bgs::random_particle_behaviors(n_particles, 0);
            bgs::ParticleBehaviorsHandle particles = plugin.add_particles(behaviors);
            for (int k = 0; k < steps; ++k) plugin.step_particles(handle, particles, dt);
            const bgs::ParticleBehaviors after = plugin.particles(particles);
            const std::vector<float> moved = plugin.positions(handle);
            std::printf("particles: %zu behaviours, %d steps of %g s\n", n_particles, steps, (double)dt);
            if (!dump_particles.empty()) {
                std::ofstream f(dump_particles, std::ios::binary);
                const uint64_t n = n_particles;
                f.write((const char*)&n, 8);
                f.write((const char*)behaviors.data(), n * 64);
                f.write((const char*)after.data(), n * 64);
                f.write((const char*)moved.data(), moved.size() * 4);
            }
        }
        bgs::PlanarGaussian3d rhs_cloud;
        std::unique_ptr<bgs::PlanarGaussian3dHandle> blended;
        if (interp_seed >= 0) {
            rhs_cloud = bgs::random_gaussians_3d_seeded(count, (uint64_t)interp_seed);
            bgs::PlanarGaussian3dHandle rhs = plugin.add_cloud(rhs_cloud);
            std::vector<uint32_t> all(count);
            std::iota(all.begin(), all.end(), 0u);
            blended.reset(new bgs::PlanarGaussian3dHandle(plugin.subset(handle, &all)));
            bgs::CloudSettings window = settings;
            window.time = interp_time; window.time_start = 0.0f; window.time_stop = 1.0f;
            plugin.interpolate(*blended, handle, rhs, window);
            std::printf("interpolated: seed %ld at time %g\n", interp_seed, (double)interp_time);
        }
        const bgs::PlanarGaussian3dHandle& drawn_cloud = blended ? *blended : handle;
        const bgs_view view = bgs::headless_view(W, H);
        const float prev_eye[3] = {prev_off[0], 1.5f + prev_off[1], 5.0f + prev_off[2]};
        const bgs_view prev_view = bgs::make_view(bgs::view_from_translation(prev_eye[0], prev_eye[1], prev_eye[2]),
                                                  bgs::perspective_infinite_reverse_rh(3.14159265358979323846f / 4.0f,
                                                                                       (float)W / (float)H, 0.1f),
                                                  prev_eye, W, H);
        if (rasterize == "classification") {
            settings.rasterize_mode = bgs::RasterizeMode::Classification;
            settings.num_classes = num_classes;
            std::vector<float> labels(count);
            for (size_t i = 0; i < count; ++i) labels[i] = 2.0f + (float)(i % num_classes);
            bgs_cloud_visibility_set(plugin.context(), drawn_cloud.get(), labels.data());
        } else if (rasterize == "optical-flow") {
            settings.rasterize_mode = bgs::RasterizeMode::OpticalFlow;
            std::printf("prev_clip:");
            for (int k = 0; k < 16; ++k) {
                uint32_t w;
                std::memcpy(&w, &prev_view.clip_from_world[k], 4);
                std::printf(" %08x", w);
            }
            std::printf("\n");
        } else if (rasterize != "color") {
            std::fprintf(stderr, "headless: --rasterize %s (color, classification or optical-flow)\n", rasterize.c_str());
            return 1;
        }
        std::vector<unsigned char> frame((size_t)W * H * 4);
        bool drawn = false;
        if (depth_plane >= 0.0f) {
            // the scene's depth buffer: the left half of the frame at depth_plane, the rest cleared (reverse-Z 0), rows
            // padded to 256 bytes as wgpu's copy_texture_to_buffer pads them; device memory through the CUDA driver
            // (libbgs's context is current on this thread)
            using Alloc = int (*)(unsigned long long*, size_t);
            using HtoD = int (*)(unsigned long long, const void*, size_t);
            using Free = int (*)(unsigned long long);
            void* cu = dlopen("libcuda.so.1", RTLD_NOW);
            if (!cu) { std::fprintf(stderr, "headless: libcuda.so.1 not found\n"); return 1; }
            const Alloc mem_alloc = (Alloc)dlsym(cu, "cuMemAlloc_v2");
            const HtoD htod = (HtoD)dlsym(cu, "cuMemcpyHtoD_v2");
            const Free mem_free = (Free)dlsym(cu, "cuMemFree_v2");
            const size_t pitch = ((size_t)W * 4 + 255) / 256 * 256;
            std::vector<float> z(pitch / 4 * H, 0.0f);
            for (int y = 0; y < H; ++y)
                for (int x = 0; x < W / 2; ++x) z[(size_t)y * (pitch / 4) + x] = depth_plane;
            unsigned long long d = 0;
            if (mem_alloc(&d, pitch * H) != 0 || htod(d, z.data(), pitch * H) != 0) {
                std::fprintf(stderr, "headless: could not place the depth buffer\n");
                return 1;
            }
            for (int f = 0; f < 3; ++f)
                drawn = plugin.render_view_depth_test(drawn_cloud, settings, view, reinterpret_cast<const float*>(d), pitch,
                                                      frame.data(), BGS_FORMAT_RGBA8_SRGB);
            mem_free(d);
        }
        std::unique_ptr<bgs::EntityList> list;   // (kept to the end: destroying it drops the frame the stats describe)
        if (instances > 0) {
            // instance j at ((j % 32) / 4 - 4, 1.5 + (j / 32 % 32) / 8 - 2, -2 - (j / 1024) / 2) (exact in f32), listed once;
            // then every instance moved by +0.5 in x through one row-major set_transforms, and three frames of the list
            std::vector<bgs::GaussianSplattingPlugin::SceneEntity> ents(instances);
            std::vector<float> rows((size_t)instances * 16, 0.0f);
            for (uint32_t j = 0; j < instances; ++j) {
                const float t[3] = {(float)(j % 32) * 0.25f - 4.0f, 1.5f + (float)(j / 32 % 32) * 0.125f - 2.0f,
                                    -2.0f - (float)(j / 1024) * 0.5f};
                ents[j].cloud = &drawn_cloud;
                ents[j].settings = settings;
                for (int k = 0; k < 3; ++k) ents[j].transform.m[12 + k] = t[k];
                float* r = &rows[(size_t)j * 16];
                r[0] = r[5] = r[10] = r[15] = 1.0f;
                r[3] = t[0] + 0.5f; r[7] = t[1]; r[11] = t[2];
            }
            list.reset(new bgs::EntityList(plugin.entity_list(ents)));
            list->set_transforms(0, instances, rows.data(), true);
            for (int f = 0; f < 3; ++f) drawn = plugin.render_entity_list(*list, view, frame.data(), BGS_FORMAT_RGBA8_SRGB);
            std::printf("instances: %u through an entity list\n", list->size());
        }
        if (shutter > 0) {
            std::vector<std::vector<bgs::GaussianSplattingPlugin::SceneEntity>> samples(shutter);
            for (uint32_t i = 0; i < shutter; ++i) {
                bgs::GaussianSplattingPlugin::SceneEntity e;
                e.cloud = &drawn_cloud;
                e.settings = settings;
                e.transform.m[12] = 0.25f * (float)i;
                samples[i].push_back(e);
            }
            const std::vector<bgs_view> views(shutter, view);
            for (int f = 0; f < 3; ++f) drawn = plugin.render_shutter(samples, views, frame.data(), BGS_FORMAT_RGBA8_SRGB);
            std::printf("shutter: %u samples\n", shutter);
        }
        for (int f = 0; f < 3 && depth_plane < 0.0f && instances == 0 && shutter == 0; ++f)
            drawn = settings.rasterize_mode == bgs::RasterizeMode::OpticalFlow
                        ? plugin.render_view(drawn_cloud, settings, view, prev_view, 1.0f / 60.0f, frame.data(), BGS_FORMAT_RGBA8_SRGB)
                        : plugin.render_view(drawn_cloud, settings, view, frame.data(), BGS_FORMAT_RGBA8_SRGB);
        const bgs_frame_stats fs = plugin.frame_stats();
        float us[6];
        bgs_stage_times_us(plugin.context(), us);
        std::printf("rendered=%d n=%u visible=%u pairs=%llu frame=%.1f us\n", (int)drawn, fs.n, fs.n_visible,
                    (unsigned long long)fs.n_pairs, us[5]);
        if (!dump.empty()) {
            std::ofstream f(dump, std::ios::binary);
            const uint64_t n = cloud.len();
            f.write((const char*)&n, 8);
            f.write((const char*)cloud.position_visibility.data(), n * 16);
            f.write((const char*)cloud.spherical_harmonic.data(), n * 192);
            f.write((const char*)cloud.rotation.data(), n * 16);
            f.write((const char*)cloud.scale_opacity.data(), n * 16);
            if (interp_seed >= 0) {
                f.write((const char*)rhs_cloud.position_visibility.data(), n * 16);
                f.write((const char*)rhs_cloud.spherical_harmonic.data(), n * 192);
                f.write((const char*)rhs_cloud.rotation.data(), n * 16);
                f.write((const char*)rhs_cloud.scale_opacity.data(), n * 16);
            }
        }
        if (!raw.empty()) { std::ofstream f(raw, std::ios::binary); f.write((const char*)frame.data(), frame.size()); }
        const size_t slash = out.find_last_of('/');
        if (slash != std::string::npos) mkdir(out.substr(0, slash).c_str(), 0755);
        std::ofstream f(out, std::ios::binary);
        f << "P6\n" << W << " " << H << "\n255\n";
        for (size_t i = 0; i < (size_t)W * H; ++i) f.write((const char*)&frame[4 * i], 3);
        std::printf("wrote %s\n", out.c_str());
    } catch (const bgs::Error& e) {
        std::fprintf(stderr, "headless: %s (status %d)\n", e.what(), (int)e.status);
        return 2;
    }
    return 0;
}
