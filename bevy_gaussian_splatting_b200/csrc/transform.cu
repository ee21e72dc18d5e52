// transform.cu -- bgs_cloud_transform (include/bgs.h): a similarity transform baked into a resident cloud in place, its
// spherical harmonics rotated with it; and bgs_cloud_bounds' pass over the position plane.
//
// The transform: each warp owns 32 consecutive gaussians.  It stages their blocks through shared memory with coalesced
// 16 B copies, one thread then transforms one gaussian's whole block in registers (one gaussian's SH rotation reads
// every SH chunk of its block, so the work cannot be split per chunk as the interpolation's is), and the warp copies the
// blocks back, again coalesced.  A gaussian the mode leaves alone is read but never written, in either copy; the pad
// chunks are neither read nor written.  The shared-memory slot of a chunk is XOR-swizzled by its block, so that both the
// warp's copies (consecutive chunks) and the per-thread block reads (one block per lane) are free of bank conflicts.
//
// Arithmetic (the constants are the host's, cloud.cu: transform_params): every operation f32 round-to-nearest-even
// without FMA (explicit __fmul_rn / __fadd_rn / __fsub_rn; the file is also built with -fmad=false), in the order
// bgs.h pins.  f16 halves are widened exactly and narrowed round-to-nearest-even.  transform_oracle/ restates it (test
// infrastructure).
#include "launch.cuh"

namespace bgs {

constexpr int XF_WARPS = 4;
constexpr int XF_THREADS = XF_WARPS * 32;
constexpr int BOUNDS_THREADS = 256;

// shared-memory slot of chunk c of the warp's block b (blocks of CH = 4, 8 or 16 chunks): within every group of eight
// lanes (one shared-memory wavefront of 16 B accesses) the eight slots fall in eight distinct 16 B bank groups
template <uint32_t CH>
__device__ __forceinline__ uint32_t xf_slot(uint32_t b, uint32_t c) {
    if constexpr (CH >= 8) return b * CH + (c ^ (b & 7u));
    else return b * CH + (c ^ ((b >> 1) & 3u));
}

__device__ __forceinline__ float f32_of(uint32_t w) { return __uint_as_float(w); }
__device__ __forceinline__ uint32_t bits_of(float f) { return __float_as_uint(f); }

// coefficient h (= 3 k + channel) of the block's SH lanes, which start at word W0
template <CloudLayout L>
__device__ __forceinline__ float sh_get(const uint32_t* w, uint32_t W0, uint32_t h) {
    if constexpr (is_f16(L)) return (h & 1u) ? half_hi(w[W0 + h / 2]) : half_lo(w[W0 + h / 2]);
    else return f32_of(w[W0 + h]);
}
template <CloudLayout L>
__device__ __forceinline__ void sh_set(uint32_t* w, uint32_t W0, uint32_t h, float v) {
    if constexpr (is_f16(L)) {
        const uint32_t hv = (uint32_t)__half_as_ushort(__float2half_rn(v));
        uint32_t& x = w[W0 + h / 2];
        x = (h & 1u) ? ((x & 0x0000FFFFu) | (hv << 16)) : ((x & 0xFFFF0000u) | hv);
    } else {
        w[W0 + h] = bits_of(v);
    }
}

// band l (1..3) of every channel: c'_i = sum_j E[i][j] c_j over j ascending, E = D_l^T row-major (2l+1)^2
template <CloudLayout L, uint32_t l>
__device__ __forceinline__ void sh_band(uint32_t* w, uint32_t W0, const float* E) {
    constexpr uint32_t m = 2 * l + 1, k0 = l * l;
#pragma unroll
    for (uint32_t ch = 0; ch < 3; ++ch) {
        float in[m];
#pragma unroll
        for (uint32_t j = 0; j < m; ++j) in[j] = sh_get<L>(w, W0, 3 * (k0 + j) + ch);
#pragma unroll
        for (uint32_t i = 0; i < m; ++i) {
            float acc = __fmul_rn(E[i * m], in[0]);
#pragma unroll
            for (uint32_t j = 1; j < m; ++j) acc = __fadd_rn(acc, __fmul_rn(E[i * m + j], in[j]));
            sh_set<L>(w, W0, 3 * (k0 + i) + ch, acc);
        }
    }
}

// q_R (x) q, Hamilton product in storage order (w, x, y, z)
__device__ __forceinline__ void quat_mul(const float a[4], const float b[4], float r[4]) {
    r[0] = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2])), __fmul_rn(a[3], b[3]));
    r[1] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0])), __fmul_rn(a[2], b[3])), __fmul_rn(a[3], b[2]));
    r[2] = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(a[0], b[2]), __fmul_rn(a[1], b[3])), __fmul_rn(a[2], b[0])), __fmul_rn(a[3], b[1]));
    r[3] = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(a[0], b[3]), __fmul_rn(a[1], b[2])), __fmul_rn(a[2], b[1])), __fmul_rn(a[3], b[0]));
}

// Sigma' = A Sigma A^T (A = the matrix's 3x3 block = s R), in the projection's T Sigma T^t order (project.cu: sigma3d);
// c: Sigma's six entries [0][0], [1][0], [2][0], [1][1], [2][1], [2][2]
__device__ __forceinline__ void cov_transform(const float* m, const float c[6], float out[6]) {
    const float S[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
    float X[3][3], T[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            X[i][j] = __fadd_rn(__fadd_rn(__fmul_rn(m[i], S[0][j]), __fmul_rn(m[4 + i], S[1][j])), __fmul_rn(m[8 + i], S[2][j]));
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            T[i][j] = __fadd_rn(__fadd_rn(__fmul_rn(X[i][0], m[j]), __fmul_rn(X[i][1], m[4 + j])), __fmul_rn(X[i][2], m[8 + j]));
    out[0] = T[0][0]; out[1] = T[1][0]; out[2] = T[2][0]; out[3] = T[1][1]; out[4] = T[2][1]; out[5] = T[2][2];
}

// one gaussian's block, as CH x 4 words, transformed in place
template <CloudLayout L, uint32_t D>
__device__ __forceinline__ void transform_block(uint32_t* w, const TransformParams& P) {
    // position: mat4_point's order (project_math.cuh); the visibility lane keeps its bits
    const float x = f32_of(w[0]), y = f32_of(w[1]), z = f32_of(w[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
        w[r] = bits_of(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.m[r], x), __fmul_rn(P.m[4 + r], y)), __fmul_rn(P.m[8 + r], z)),
                                 P.m[12 + r]));
    constexpr uint32_t S = 4 * SECOND_CHUNK;
    if constexpr (L == CloudLayout::F32) {
        const float q[4] = {f32_of(w[S]), f32_of(w[S + 1]), f32_of(w[S + 2]), f32_of(w[S + 3])};
        float r[4];
        quat_mul(P.q, q, r);
#pragma unroll
        for (int k = 0; k < 4; ++k) w[S + k] = bits_of(r[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) w[4 * SO_CHUNK + k] = bits_of(__fmul_rn(P.s, f32_of(w[4 * SO_CHUNK + k])));
    } else if constexpr (L == CloudLayout::F16) {
        float a[4], b[4];   // (w, x, y, z) | (scale x, y, z, opacity)
        second_lanes(w[S], w[S + 1], a);
        second_lanes(w[S + 2], w[S + 3], b);
        float r[4];
        quat_mul(P.q, a, r);
        w[S] = pack_halves(r[0], r[1]);
        w[S + 1] = pack_halves(r[2], r[3]);
        w[S + 2] = pack_halves(__fmul_rn(P.s, b[0]), __fmul_rn(P.s, b[1]));
        w[S + 3] = ((uint32_t)__half_as_ushort(__float2half_rn(__fmul_rn(P.s, b[2]))) << 16) | (w[S + 3] & 0xFFFFu);
    } else {   // F16Cov: c0, c1 | c2, c3 | c4, c5 | the opacity word, kept
        float a[4], b[4];
        second_lanes(w[S], w[S + 1], a);
        second_lanes(w[S + 2], w[S + 3], b);
        const float c[6] = {a[0], a[1], a[2], a[3], b[0], b[1]};
        float o[6];
        cov_transform(P.m, c, o);
        w[S] = pack_halves(o[0], o[1]);
        w[S + 1] = pack_halves(o[2], o[3]);
        w[S + 2] = pack_halves(o[4], o[5]);
    }
    constexpr uint32_t W0 = 4 * sh_first(L);
    if constexpr (D >= 1) sh_band<L, 1>(w, W0, P.sh1);
    if constexpr (D >= 2) sh_band<L, 2>(w, W0, P.sh2);
    if constexpr (D >= 3) sh_band<L, 3>(w, W0, P.sh3);
}

template <CloudLayout L, uint32_t D>
__global__ void __launch_bounds__(XF_THREADS, 4) transform_kernel(CloudView cl, uint32_t n, const __grid_constant__ TransformParams P,
                                                              uint32_t selected_only) {
    constexpr uint32_t CH = chunks(L, D);
    __shared__ uint4 stage[XF_WARPS][32 * CH];
    const uint32_t lane = threadIdx.x & 31u, wi = threadIdx.x >> 5;
    const size_t base = ((size_t)blockIdx.x * XF_WARPS + wi) * 32u;
    if (base >= n) return;   // (whole warps only)
    const uint32_t m = (uint32_t)min((size_t)32, n - base);
    uint4* s = stage[wi];
    uint4* g = cl.blocks + base * CH;
#pragma unroll
    for (uint32_t k = 0; k < CH; ++k) {
        const uint32_t u = k * 32u + lane, b = u / CH, c = u % CH;
        if (b < m && !is_pad(L, D, c)) s[xf_slot<CH>(b, c)] = g[u];
    }
    __syncwarp();
    bool write = false;
    if (lane < m) {
        uint32_t w[CH * 4];
#pragma unroll
        for (uint32_t c = 0; c < CH; ++c) {
            if (is_pad(L, D, c)) continue;
            const uint4 v = s[xf_slot<CH>(lane, c)];
            w[4 * c] = v.x; w[4 * c + 1] = v.y; w[4 * c + 2] = v.z; w[4 * c + 3] = v.w;
        }
        write = !selected_only || !(f32_of(w[3]) < 0.5f);
        if (write) {
            transform_block<L, D>(w, P);
#pragma unroll
            for (uint32_t c = 0; c < CH; ++c)
                if (!is_pad(L, D, c)) s[xf_slot<CH>(lane, c)] = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
            cl.pos[base + lane] = make_float4(f32_of(w[0]), f32_of(w[1]), f32_of(w[2]), f32_of(w[3]));
        }
    }
    const uint32_t written = __ballot_sync(0xffffffffu, write);
#pragma unroll
    for (uint32_t k = 0; k < CH; ++k) {
        const uint32_t u = k * 32u + lane, b = u / CH, c = u % CH;
        if (b < m && ((written >> b) & 1u) && !is_pad(L, D, c)) g[u] = s[xf_slot<CH>(b, c)];
    }
}

void launch_transform(CloudLayout layout, uint32_t sh_degree, CloudView cloud, uint32_t n, const TransformParams& p,
                      uint32_t selected_only, cudaStream_t stream) {
    if (n == 0) return;
    const uint32_t grid = (uint32_t)(((size_t)n + XF_THREADS - 1) / XF_THREADS);
    with_layout_degree(layout, sh_degree, [&](auto L, auto D) {   // (bgs_cloud_transform refuses 4D clouds)
        if constexpr (!is_4d(decltype(L)::value))
            transform_kernel<decltype(L)::value, decltype(D)::value><<<grid, XF_THREADS, 0, stream>>>(cloud, n, p, selected_only);
    });
}

// ---- bounds: an order-preserving u32 key of a finite f32 (-0 sorts just below +0), reduced with atomicMin / atomicMax

__device__ __forceinline__ uint32_t order_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// words: min keys x, y, z (set to 0xFFFFFFFF before) | max keys x, y, z (0) | count (0)
__global__ void __launch_bounds__(BOUNDS_THREADS) bounds_kernel(const float4* __restrict__ pos, uint32_t n, uint32_t selected_only,
                                                                uint32_t* __restrict__ words) {
    const float inf = __uint_as_float(0x7F800000u);
    float lo[3] = {inf, inf, inf}, hi[3] = {-inf, -inf, -inf};
    uint32_t cnt = 0;
    for (size_t i = (size_t)blockIdx.x * BOUNDS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * BOUNDS_THREADS) {
        const float4 p = __ldg(pos + i);
        const bool finite = fabsf(p.x) < inf && fabsf(p.y) < inf && fabsf(p.z) < inf;
        if (finite && (!selected_only || !(p.w < 0.5f))) {
            lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
            hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
            ++cnt;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
            hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
        }
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31u) == 0 && cnt) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            atomicMin(words + k, order_key(lo[k]));
            atomicMax(words + 3 + k, order_key(hi[k]));
        }
        atomicAdd(words + 6, cnt);
    }
}

void launch_bounds(const float4* pos, uint32_t n, uint32_t selected_only, uint32_t* words, int sm_count, cudaStream_t stream) {
    if (n == 0) return;
    const uint32_t need = (uint32_t)(((size_t)n + BOUNDS_THREADS - 1) / BOUNDS_THREADS);
    const uint32_t grid = std::min<uint32_t>(need, (uint32_t)sm_count * 8u);
    bounds_kernel<<<grid, BOUNDS_THREADS, 0, stream>>>(pos, n, selected_only, words);
}

}  // namespace bgs
