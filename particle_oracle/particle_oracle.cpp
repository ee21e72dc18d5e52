// particle_oracle.cpp -- see particle_oracle.h.  A plain scalar restatement of src/morph/particle.wgsl:36-52; the
// compile flags (-ffp-contract=off, no fast-math) keep every operation an IEEE f32 round-to-nearest-even one.
#include "particle_oracle.h"

#include <cstring>
#include <vector>

namespace {

// WGSL's abstract-float 1.0 / 6.0, converted to f32 once where it meets the f32 jerk (particle.wgsl:36)
const float C6 = (float)(1.0 / 6.0);

struct Behavior {
    uint32_t indices[4];
    float velocity[4], acceleration[4], jerk[4];
};
static_assert(sizeof(Behavior) == 64, "ParticleBehavior is 64 B");

}  // namespace

extern "C" {

float orc_particle_c6(void) { return C6; }

int orc_particle_step(float* pos_vis, uint32_t n, void* behaviors, uint32_t count, float dt) {
    Behavior* b = static_cast<Behavior*>(behaviors);
    std::vector<uint8_t> named(n, 0);
    for (uint32_t i = 0; i < count; ++i) {
        const int32_t idx = (int32_t)b[i].indices[0];   // particle.wgsl:15 reads indicies as vec4<i32>
        if (idx < 0) continue;
        if ((uint32_t)idx >= n || named[idx]) return -1;
        named[idx] = 1;
    }
    for (uint32_t i = 0; i < count; ++i) {
        Behavior& r = b[i];
        const int32_t idx = (int32_t)r.indices[0];
        if (idx < 0) continue;                          // particle.wgsl:46-48: nothing is written
        float* p = pos_vis + (size_t)idx * 4;           // particle.wgsl:31-32: all four lanes
        for (int k = 0; k < 4; ++k) {
            const float v = r.velocity[k], a = r.acceleration[k], j = r.jerk[k];
            // particle.wgsl:36: v * dt + 0.5 * a * dt * dt + 1.0 / 6.0 * j * dt * dt * dt, left to right
            const float t0 = v * dt;
            float t1 = 0.5f * a;
            t1 = t1 * dt;
            t1 = t1 * dt;
            float t2 = C6 * j;
            t2 = t2 * dt;
            t2 = t2 * dt;
            t2 = t2 * dt;
            float dp = t0 + t1;
            dp = dp + t2;
            // particle.wgsl:37: a * dt + 0.5 * j * dt * dt
            const float u0 = a * dt;
            float u1 = 0.5f * j;
            u1 = u1 * dt;
            u1 = u1 * dt;
            const float dv = u0 + u1;
            // particle.wgsl:38
            const float da = j * dt;
            // particle.wgsl:40-42, 50-52
            p[k] = p[k] + dp;
            r.velocity[k] = v + dv;
            r.acceleration[k] = a + da;
        }
    }
    return 0;
}

}  // extern "C"
