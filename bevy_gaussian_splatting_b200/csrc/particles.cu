// particles.cu -- particle behaviours (src/morph/particle.rs, particle.wgsl; the `morph_particles` feature) on the
// device-resident cloud: one step moves each active behaviour's gaussian by its velocity, acceleration and jerk over
// `dt`, and advances the behaviour's own velocity and acceleration.
//
// One thread per behaviour.  The 64 B record (indices | velocity | acceleration | jerk) is four 16 B loads; the
// position is one 16 B gather by index.  The new position goes to both device copies -- the position plane (what
// key-gen streams) and the first 16 B of the gaussian's block (what the projection reads) -- and the new velocity and
// acceleration back into the record; jerk and indices are never stored.
//
// Arithmetic: particle.wgsl:36-38 in WGSL's left-associative order, each operation f32 round-to-nearest-even without
// FMA (explicit __fmul_rn / __fadd_rn; the file is also built with -fmad=false).  1.0 / 6.0 is WGSL's abstract
// constant, rounded to f32 once.  particle_oracle/particle_oracle.cpp restates it (test infrastructure).
#include "common.cuh"

namespace bgs {

constexpr int PARTICLE_THREADS = 256;
constexpr float PARTICLE_C6 = (float)(1.0 / 6.0);   // 0x3E2AAAAB

struct LaneStep {
    float p, v, a;
};

// one lane of particle.wgsl:36-42: dp = v*dt + 0.5*a*dt*dt + 1/6*j*dt*dt*dt, dv = a*dt + 0.5*j*dt*dt, da = j*dt
__device__ __forceinline__ LaneStep particle_lane(float p, float v, float a, float j, float dt) {
    const float dp = __fadd_rn(__fadd_rn(__fmul_rn(v, dt), __fmul_rn(__fmul_rn(__fmul_rn(0.5f, a), dt), dt)),
                               __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(PARTICLE_C6, j), dt), dt), dt));
    const float dv = __fadd_rn(__fmul_rn(a, dt), __fmul_rn(__fmul_rn(__fmul_rn(0.5f, j), dt), dt));
    const float da = __fmul_rn(j, dt);
    return {__fadd_rn(p, dp), __fadd_rn(v, dv), __fadd_rn(a, da)};
}

// behaviours: count records of 4 x float4 (indices as raw bits | velocity | acceleration | jerk).  An index whose
// i32 reading is negative (>= 2^31) is inactive: nothing is written (particle.wgsl:46-48).
__global__ void __launch_bounds__(PARTICLE_THREADS) particle_step_kernel(float4* __restrict__ behaviors, uint32_t count,
                                                                         float dt, float4* __restrict__ pos,
                                                                         float4* __restrict__ blocks, uint32_t block_stride) {
    const uint32_t b = blockIdx.x * PARTICLE_THREADS + threadIdx.x;
    if (b >= count) return;
    float4* rec = behaviors + (size_t)b * 4;
    const float4 ix = rec[0], v = rec[1], a = rec[2], j = rec[3];
    const uint32_t idx = __float_as_uint(ix.x);
    if ((int32_t)idx < 0) return;
    const float4 p = pos[idx];
    const LaneStep x = particle_lane(p.x, v.x, a.x, j.x, dt), y = particle_lane(p.y, v.y, a.y, j.y, dt),
                   z = particle_lane(p.z, v.z, a.z, j.z, dt), w = particle_lane(p.w, v.w, a.w, j.w, dt);
    const float4 np = make_float4(x.p, y.p, z.p, w.p);
    pos[idx] = np;
    blocks[(size_t)idx * block_stride] = np;
    rec[1] = make_float4(x.v, y.v, z.v, w.v);
    rec[2] = make_float4(x.a, y.a, z.a, w.a);
}

// block_stride: 16 B chunks per gaussian-major block (f16 layouts 8, f32 16)
void launch_particle_step(void* behaviors, uint32_t count, float dt, float4* pos, void* blocks, uint32_t block_stride,
                          cudaStream_t stream) {
    const uint32_t grid = (count + PARTICLE_THREADS - 1) / PARTICLE_THREADS;
    particle_step_kernel<<<grid, PARTICLE_THREADS, 0, stream>>>(reinterpret_cast<float4*>(behaviors), count, dt, pos,
                                                                reinterpret_cast<float4*>(blocks), block_stride);
}

}  // namespace bgs
