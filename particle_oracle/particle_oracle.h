/*
 * particle_oracle.h -- CPU ORACLE of the particle step (src/morph/particle.wgsl:23-53, the reference's
 * `morph_particles` feature).  TEST INFRASTRUCTURE ONLY: the product (libbgs.so) never links, loads or calls it.
 * Built beside oracle/ (the render oracle) by __graft_entry__.build().
 *
 * The rule (include/bgs.h, bgs_cloud_particles_step), one scalar restatement of particle.wgsl:36-52 per behaviour, in
 * record order: a behaviour whose indices[0] reads negative as i32 writes nothing; otherwise, per lane of
 * p = pos_vis[indices[0]] (all four), every operation f32 round-to-nearest-even without FMA (-ffp-contract=off):
 *   dp = ((v*dt) + (((0.5f*a)*dt)*dt)) + ((((C6*j)*dt)*dt)*dt),  C6 = (float)(1.0 / 6.0)
 *   dv = (a*dt) + (((0.5f*j)*dt)*dt)
 *   da = j*dt
 *   pos_vis := p + dp, velocity := v + dv, acceleration := a + da; jerk and indices are unchanged.
 *
 * behaviors: count records of 64 B (u32 indices[4], f32 velocity[4], acceleration[4], jerk[4]), updated in place;
 * pos_vis: n * 4 floats, updated in place.  Returns 0, or -1 (nothing changed) when an active index is >= n or two
 * active behaviours name the same gaussian -- the inputs libbgs refuses.
 */
#ifndef PARTICLE_ORACLE_H
#define PARTICLE_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

int orc_particle_step(float* pos_vis, uint32_t n, void* behaviors, uint32_t count, float dt);
/* the f32 constant the step uses for WGSL's 1.0 / 6.0 */
float orc_particle_c6(void);

#ifdef __cplusplus
}
#endif
#endif
