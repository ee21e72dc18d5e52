// cloud_tool.cpp -- CPU-only helper over include/bgs_io.hpp: load a cloud file the way the reference's asset loader
// does (src/io/loader.rs:38-66: `.ply` and `.gcloud`) and dump the four f32 planes in the format headless.cpp's
// --dump-cloud uses (u64 n, then pos_vis n*4, sh n*48, rot n*4, scale_opacity n*4), so another host (or a test) can
// check the planes or render the identical cloud.  A cloud of SH degree d < 3 dumps its sh plane at S_d floats per
// gaussian (4, 12, 28).  --sh-degree D parses a .ply as the reference's sh_D build does (default 3); a .gcloud carries
// its own degree.
//
//   cloud_tool <in.ply|in.gcloud> <out.bin> [--sh-degree D]
//   cloud_tool <in.ply|in.gcloud> <out.gcloud> --gcloud [--sh-degree D]
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>

#include "../include/bgs_io.hpp"

int main(int argc, char** argv) {
    bool gcloud = false, ok = argc >= 3;
    uint32_t sh_degree = 3;
    for (int a = 3; a < argc && ok; ++a) {
        const std::string arg = argv[a];
        if (arg == "--gcloud") gcloud = true;
        else if (arg == "--sh-degree" && a + 1 < argc) sh_degree = (uint32_t)std::strtoul(argv[++a], nullptr, 10);
        else ok = false;
    }
    if (!ok) {
        std::fprintf(stderr, "usage: cloud_tool <in.ply|in.gcloud> <out.bin> [--sh-degree D]            (dump the four f32 planes)\n"
                             "       cloud_tool <in.ply|in.gcloud> <out.gcloud> --gcloud [--sh-degree D]  (re-encode as .gcloud)\n");
        return 1;
    }
    try {
        const std::string in = argv[1];
        const bool ply = in.size() >= 4 && in.compare(in.size() - 4, 4, ".ply") == 0;
        std::ifstream ply_in;
        if (ply) ply_in.open(in, std::ios::binary);
        if (ply && !ply_in) throw std::runtime_error("cannot open " + in);
        const bgs::PlanarGaussian3d cloud = ply ? bgs::io::parse_ply_3d(ply_in, sh_degree)
                                                : bgs::io::load_cloud(in);      // src/io/loader.rs:38-66
        std::ofstream f(argv[2], std::ios::binary);
        const uint64_t n = cloud.len();
        if (gcloud) {
            const std::vector<unsigned char> bytes = bgs::io::encode_gcloud(cloud);
            f.write((const char*)bytes.data(), (std::streamsize)bytes.size());
        } else {
            f.write((const char*)&n, 8);
            f.write((const char*)cloud.position_visibility.data(), n * 16);
            f.write((const char*)cloud.spherical_harmonic.data(), n * 4 * bgs::sh_width(cloud.sh_degree));
            f.write((const char*)cloud.rotation.data(), n * 16);
            f.write((const char*)cloud.scale_opacity.data(), n * 16);
        }
        std::printf("%llu gaussians\n", (unsigned long long)n);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "cloud_tool: %s\n", e.what());
        return 2;
    }
    return 0;
}
