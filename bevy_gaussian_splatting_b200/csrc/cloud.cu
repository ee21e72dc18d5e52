// cloud.cu -- the extern "C" calls of libbgs (include/bgs.h) on a resident cloud: upload and destroy, selection edits,
// particle behaviours, positions and visibility read-back, interpolation, subset and download.  None of them is part of
// a frame; the order in which they and the frames reach a cloud is host.cuh's.
#include <cmath>
#include <cstring>
#include <algorithm>
#include <new>
#include <vector>

#include "host.cuh"

namespace {

// Releases a cloud that a call failed to finish, and reports why.
bgs_status drop_cloud(bgs_context* c, const char* call, bgs_cloud* cl, cudaError_t e) {
    bgs_cloud_destroy(cl);
    return fail(c, status_of(e), "%s: %s", call, cudaGetErrorString(e));
}

// A new cloud of n gaussians in the given layout and SH degree on the context's device, its planes allocated but not
// yet written.
bgs_status new_cloud(bgs_context* c, const char* call, uint32_t n, CloudLayout layout, uint32_t sh_degree, bgs_cloud** out) {
    bgs_cloud* cl = new (std::nothrow) bgs_cloud();
    if (!cl) return fail(c, BGS_ENOMEM, "%s: out of host memory", call);
    cl->device = c->device; cl->n = n; cl->layout = layout; cl->sh_degree = sh_degree;
    cudaError_t e = cudaMalloc(&cl->pos, (size_t)n * plane_bytes(layout, sh_degree, PLANE_POS));
    if (e == cudaSuccess) e = cudaMalloc(&cl->blocks, (size_t)n * block_bytes(layout, sh_degree));
    if (e != cudaSuccess) return drop_cloud(c, call, cl, e);
    *out = cl;
    return BGS_OK;
}

// One device word read back: copied to the context's own pinned word on the render stream, which is then drained.
bgs_status read_word(bgs_context* c, const uint32_t* word, uint32_t* out) {
    CU(c, cudaMemcpyAsync(c->h_word, word, 4, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    *out = *c->h_word;
    return BGS_OK;
}

// Device scratch of one call, released on the stream when it goes out of scope.
struct StreamScratch {
    void* p = nullptr;
    cudaStream_t q;
    explicit StreamScratch(cudaStream_t s) : q(s) {}
    StreamScratch(const StreamScratch&) = delete;
    StreamScratch& operator=(const StreamScratch&) = delete;
    ~StreamScratch() { if (p) cudaFreeAsync(p, q); }
    cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, q); }
};

// gaussians per chunk of a download: the device staging arrays hold one chunk (f32: 28 MB), each of the context's two
// pinned bounce buffers one chunk's planes (f32: 30 MB).  4D gaussians are wider: their chunks hold as many gaussians
// as fit the same bounce buffers
constexpr uint32_t DOWNLOAD_CHUNK = 1u << 17;
constexpr size_t DOWNLOAD_BOUNCE_BYTES = (size_t)DOWNLOAD_CHUNK * planar_bytes(CloudLayout::F32, SH_DEGREE_MAX);
static_assert(planar_bytes(CloudLayout::F32, SH_DEGREE_MAX) >= planar_bytes(CloudLayout::F16, SH_DEGREE_MAX),
              "the f32 chunk is the largest 3D one");

// the family of download call a layout answers to (0: _f32, 1: _f16, both f16 layouts; 2: _4d)
int download_family(CloudLayout l) { return is_4d(l) ? 2 : is_f16(l) ? 1 : 0; }

// n rows of `width` bytes between arrays of pitch src_pitch and dst_pitch (one contiguous copy when both are `width`)
cudaError_t copy_rows(void* dst, size_t dst_pitch, const void* src, size_t src_pitch, size_t width, size_t n,
                      cudaMemcpyKind kind, cudaStream_t q) {
    if (dst_pitch == width && src_pitch == width) return cudaMemcpyAsync(dst, src, n * width, kind, q);
    return cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, width, n, kind, q);
}

// The rest of a new cloud's upload: its staged planes (the position plane is the cloud's own; the others go to device
// scratch, the SH plane at whole chunks per gaussian) are written by stage(d), repacked into the gaussian-major blocks the
// projection gathers, and freed again.  stage returns BGS_OK, or a status it has reported; on any failure the cloud is
// released and *out stays NULL.
template <class Stage>
bgs_status stage_and_repack(bgs_context* ctx, const char* call, bgs_cloud* cl, Stage stage, bgs_cloud** out) {
    const CloudLayout layout = cl->layout;
    const uint32_t n = cl->n, sh_degree = cl->sh_degree;
    void* d[PLANES] = {cl->pos, nullptr, nullptr, nullptr, nullptr};
    cudaError_t e = cudaSuccess;
    for (int p = PLANE_SH; p < PLANES && e == cudaSuccess; ++p)
        if (plane_bytes(layout, sh_degree, p)) e = cudaMalloc(&d[p], (size_t)n * staged_bytes(layout, sh_degree, p));
    bgs_status st = BGS_OK;
    if (e == cudaSuccess) st = stage(d);
    if (e == cudaSuccess && st == BGS_OK) {
        launch_repack(layout, sh_degree, d[PLANE_SH], d[PLANE_ROT], d[PLANE_SO], d[PLANE_TT], n, cl->view(), ctx->stream);
        e = cudaStreamSynchronize(ctx->stream);
    }
    for (int p = PLANE_SH; p < PLANES; ++p) cudaFree(d[p]);
    if (e != cudaSuccess) return drop_cloud(ctx, call, cl, e);
    if (st != BGS_OK) {
        bgs_cloud_destroy(cl);
        return st;
    }
    *out = cl;
    return BGS_OK;
}

struct KhrSlot {
    const char* name;
    const bgs_khr_accessor* a;
};

uint32_t khr_component_bytes(uint32_t type) {
    return type == KHR_I8 || type == KHR_U8 ? 1u : type == KHR_I16 || type == KHR_U16 ? 2u : type == KHR_F32 ? 4u : 0u;
}

// the (components, component type, normalised) combinations each slot accepts (scene.rs:1590-1960); sh: the SH slots
bool khr_accepted(const KhrSlot& s, bool sh) {
    const bgs_khr_accessor& a = *s.a;
    const uint32_t t = a.component_type, c = a.components;
    const bool f32 = t == KHR_F32, norm = a.normalized != 0;
    if (sh || !strcmp(s.name, "POSITION")) return c == 3 && f32;
    if (!strcmp(s.name, "ROTATION")) return c == 4 && (f32 || ((t == KHR_I8 || t == KHR_I16) && norm));
    if (!strcmp(s.name, "SCALE")) return c == 3 && (f32 || t == KHR_I8 || t == KHR_I16);
    if (!strcmp(s.name, "OPACITY")) return c == 1 && (f32 || ((t == KHR_U8 || t == KHR_U16) && norm));
    return (c == 3 || c == 4) && (f32 || t == KHR_U8 || t == KHR_U16);   // COLOR_0
}

bgs_status khr_check(bgs_context* c, const KhrSlot& s, bool sh) {
    const bgs_khr_accessor& a = *s.a;
    if (!a.data) return fail(c, BGS_EINVAL, "upload_khr: %s has no data", s.name);
    if (!khr_accepted(s, sh))
        return fail(c, BGS_EINVAL, "upload_khr: %s does not accept %u components of component type %u (normalized %u)", s.name,
                    a.components, a.component_type, a.normalized);
    const uint32_t cb = khr_component_bytes(a.component_type);
    if (a.byte_stride < cb * a.components || a.byte_stride % cb)
        return fail(c, BGS_EINVAL, "upload_khr: %s byte_stride %u is below its element size %u or not a multiple of %u", s.name,
                    a.byte_stride, cb * a.components, cb);
    return BGS_OK;
}

// ---- bgs_cloud_transform's host half (the rule: include/bgs.h), in f64

// the renderer's SH band l (1..3) at the direction d: project.cu's sh_basis polynomials times its c_shc constants (here
// at f64, the decimal values spherical_harmonics.wgsl gives)
void sh_band_basis(int l, const double d[3], double* y) {
    const double x = d[0], yy_ = d[1], z = d[2];
    const double xx = x * x, yy = yy_ * yy_, zz = z * z;
    if (l == 1) {
        y[0] = -0.4886025119029199 * yy_; y[1] = 0.4886025119029199 * z; y[2] = -0.4886025119029199 * x;
    } else if (l == 2) {
        y[0] = 1.0925484305920792 * (x * yy_); y[1] = -1.0925484305920792 * (yy_ * z);
        y[2] = 0.31539156525252005 * ((2.0 * zz - xx) - yy); y[3] = -1.0925484305920792 * (x * z);
        y[4] = 0.5462742152960396 * (xx - yy);
    } else {
        y[0] = -0.5900435899266435 * (yy_ * (3.0 * xx - yy)); y[1] = 2.890611442640554 * ((x * yy_) * z);
        y[2] = -0.4570457994644658 * (yy_ * ((4.0 * zz - xx) - yy)); y[3] = 0.3731763325901154 * (z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy));
        y[4] = -0.4570457994644658 * (x * ((4.0 * zz - xx) - yy)); y[5] = 1.445305721320277 * (z * (xx - yy));
        y[6] = -0.5900435899266435 * (x * (xx - 3.0 * yy));
    }
}

// E_l = D_l^T (row-major), D_l defined by Y_l(R^T d) = D_l Y_l(d): the least-squares solution of Y E = Z over 64 fixed
// directions d_k (a Fibonacci sphere), Y's rows Y_l(d_k) and Z's Y_l(R^T d_k), through the normal equations and
// Gauss-Jordan elimination with partial pivoting.  Entries below 2^-40 in magnitude are exactly 0.
void sh_rotation(const double R[3][3], int l, double* E) {
    const int m = 2 * l + 1;
    constexpr int N = 64;
    double G[7][14] = {};   // [Y^T Y | Y^T Z]
    for (int k = 0; k < N; ++k) {
        const double z = 1.0 - (2.0 * k + 1.0) / N, r = std::sqrt(1.0 - z * z), phi = k * 2.399963229728653;
        const double d[3] = {r * std::cos(phi), r * std::sin(phi), z};
        const double rd[3] = {R[0][0] * d[0] + R[1][0] * d[1] + R[2][0] * d[2], R[0][1] * d[0] + R[1][1] * d[1] + R[2][1] * d[2],
                              R[0][2] * d[0] + R[1][2] * d[1] + R[2][2] * d[2]};
        double y[7], yr[7];
        sh_band_basis(l, d, y);
        sh_band_basis(l, rd, yr);
        for (int i = 0; i < m; ++i)
            for (int j = 0; j < m; ++j) { G[i][j] += y[i] * y[j]; G[i][m + j] += y[i] * yr[j]; }
    }
    for (int c = 0; c < m; ++c) {
        int p = c;
        for (int r = c + 1; r < m; ++r)
            if (std::fabs(G[r][c]) > std::fabs(G[p][c])) p = r;
        for (int j = 0; j < 2 * m; ++j) std::swap(G[c][j], G[p][j]);
        const double inv = 1.0 / G[c][c];
        for (int j = 0; j < 2 * m; ++j) G[c][j] *= inv;
        for (int r = 0; r < m; ++r)
            if (r != c) {
                const double f = G[r][c];
                for (int j = 0; j < 2 * m; ++j) G[r][j] -= f * G[c][j];
            }
    }
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < m; ++j) {
            const double e = G[i][m + j];
            E[i * m + j] = std::fabs(e) < 0x1p-40 ? 0.0 : e;
        }
}

// The matrix's check and the kernel's constants; false (with the reason in `why`) for a matrix the call refuses
bool transform_params(const float* M, TransformParams* P, const char** why) {
    for (int k = 0; k < 16; ++k)
        if (!std::isfinite(M[k])) { *why = "an entry is not finite"; return false; }
    if (M[3] != 0.0f || M[7] != 0.0f || M[11] != 0.0f || M[15] != 1.0f) { *why = "the bottom row is not (0, 0, 0, 1)"; return false; }
    double A[3][3];   // A[row][col]
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[i][j] = M[4 * j + i];
    auto dot = [&](int a, int b) { return (A[0][a] * A[0][b] + A[1][a] * A[1][b]) + A[2][a] * A[2][b]; };
    const double s2 = ((dot(0, 0) + dot(1, 1)) + dot(2, 2)) / 3.0;
    if (!(s2 > 0.0)) { *why = "the 3x3 block is zero"; return false; }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            if (!(std::fabs(dot(i, j) - (i == j ? s2 : 0.0)) <= 1e-5 * s2)) {
                *why = "the 3x3 block is not a rotation times a uniform scale (shear or non-uniform scale)";
                return false;
            }
    const double det = (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])) +
                       A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
    if (!(det > 0.0)) { *why = "the 3x3 block is a reflection"; return false; }
    const double s = std::sqrt(s2);
    double R[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = A[i][j] / s;
    // Shepperd: the largest of tr, R00, R11, R22 (the first on a tie) picks the component taken from a square root
    const double tr = (R[0][0] + R[1][1]) + R[2][2];
    double q[4];   // w, x, y, z
    int b = 0;
    const double cand[4] = {tr, R[0][0], R[1][1], R[2][2]};
    for (int k = 1; k < 4; ++k)
        if (cand[k] > cand[b]) b = k;
    if (b == 0) {
        const double t = 0.5 * std::sqrt(1.0 + tr), f = 0.25 / t;
        q[0] = t; q[1] = (R[2][1] - R[1][2]) * f; q[2] = (R[0][2] - R[2][0]) * f; q[3] = (R[1][0] - R[0][1]) * f;
    } else if (b == 1) {
        const double t = 0.5 * std::sqrt(((1.0 + R[0][0]) - R[1][1]) - R[2][2]), f = 0.25 / t;
        q[0] = (R[2][1] - R[1][2]) * f; q[1] = t; q[2] = (R[0][1] + R[1][0]) * f; q[3] = (R[0][2] + R[2][0]) * f;
    } else if (b == 2) {
        const double t = 0.5 * std::sqrt(((1.0 - R[0][0]) + R[1][1]) - R[2][2]), f = 0.25 / t;
        q[0] = (R[0][2] - R[2][0]) * f; q[1] = (R[0][1] + R[1][0]) * f; q[2] = t; q[3] = (R[1][2] + R[2][1]) * f;
    } else {
        const double t = 0.5 * std::sqrt(((1.0 - R[0][0]) - R[1][1]) + R[2][2]), f = 0.25 / t;
        q[0] = (R[1][0] - R[0][1]) * f; q[1] = (R[0][2] + R[2][0]) * f; q[2] = (R[1][2] + R[2][1]) * f; q[3] = t;
    }
    const double qn = std::sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
    const double sg = q[0] < 0.0 ? -1.0 : 1.0;
    for (double& v : q) v = sg * v / qn;
    // the SH follow the rotation of the unit quaternion (in f64, before rounding): R_q = R_std(q)
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double Rq[3][3] = {{1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y)},
                             {2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x)},
                             {2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)}};
    for (int k = 0; k < 16; ++k) P->m[k] = M[k];
    for (int k = 0; k < 4; ++k) P->q[k] = (float)q[k];
    P->s = (float)s;
    float* const bands[3] = {P->sh1, P->sh2, P->sh3};
    for (int l = 1; l <= 3; ++l) {
        double E[49];
        sh_rotation(Rq, l, E);
        for (int k = 0; k < (2 * l + 1) * (2 * l + 1); ++k) bands[l - 1][k] = (float)E[k];
    }
    return true;
}

}  // namespace

extern "C" {

static bgs_status upload_common(bgs_context* ctx, uint32_t n, CloudLayout layout, uint32_t sh_degree, const float* pos_vis,
                                const void* sh, const void* rot, const void* so, const void* tt, bgs_cloud** out) {
    if (!ctx || !out) return BGS_EINVAL;
    *out = nullptr;
    if (sh_degree > SH_DEGREE_MAX) return fail(ctx, BGS_EINVAL, "cloud upload: sh_degree %u is not in [0, 3]", sh_degree);
    const void* src[PLANES] = {pos_vis, sh, rot, so, tt};
    for (int p = 0; p < PLANES; ++p)
        if (plane_bytes(layout, sh_degree, p) && !src[p]) return fail(ctx, BGS_EINVAL, "cloud upload: null plane pointer");
    if (n == 0 || n >= (1u << 30)) return fail(ctx, BGS_EINVAL, "cloud upload: n must be in [1, 2^30)");
    CU(ctx, cudaSetDevice(ctx->device));
    bgs_cloud* cl = nullptr;
    TRY(new_cloud(ctx, "cloud upload", n, layout, sh_degree, &cl));
    // the caller's planes, each staged SH row's last chunk zero past the plane's width
    return stage_and_repack(ctx, "cloud upload", cl, [&](void* const* d) {
        cudaError_t e = cudaSuccess;
        for (int p = 0; p < PLANES && e == cudaSuccess; ++p) {
            const size_t width = plane_bytes(layout, sh_degree, p), staged = staged_bytes(layout, sh_degree, p);
            if (width == 0) continue;
            if (staged != width) e = cudaMemsetAsync(d[p], 0, (size_t)n * staged, ctx->stream);
            if (e == cudaSuccess) e = copy_rows(d[p], staged, src[p], width, width, n, cudaMemcpyHostToDevice, ctx->stream);
        }
        return e == cudaSuccess ? BGS_OK : fail(ctx, status_of(e), "cloud upload: %s", cudaGetErrorString(e));
    }, out);
}

bgs_status bgs_cloud_upload_f32(bgs_context* ctx, uint32_t n, const float* pos_vis, const float* sh,
                                const float* rot_wxyz, const float* scale_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F32, SH_DEGREE_MAX, pos_vis, sh, rot_wxyz, scale_opacity, nullptr, out);
}

bgs_status bgs_cloud_upload_f32_sh(bgs_context* ctx, uint32_t n, uint32_t sh_degree, const float* pos_vis, const float* sh,
                                   const float* rot_wxyz, const float* scale_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F32, sh_degree, pos_vis, sh, rot_wxyz, scale_opacity, nullptr, out);
}

bgs_status bgs_cloud_upload_f16(bgs_context* ctx, uint32_t n, const float* pos_vis, const uint32_t* sh_packed,
                                const uint32_t* rot_scale_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F16, SH_DEGREE_MAX, pos_vis, sh_packed, rot_scale_opacity, nullptr, nullptr, out);
}

bgs_status bgs_cloud_upload_f16_sh(bgs_context* ctx, uint32_t n, uint32_t sh_degree, const float* pos_vis,
                                   const uint32_t* sh_packed, const uint32_t* rot_scale_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F16, sh_degree, pos_vis, sh_packed, rot_scale_opacity, nullptr, nullptr, out);
}

bgs_status bgs_cloud_upload_f16_cov(bgs_context* ctx, uint32_t n, const float* pos_vis, const uint32_t* sh_packed,
                                    const uint32_t* cov3d_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F16Cov, SH_DEGREE_MAX, pos_vis, sh_packed, cov3d_opacity, nullptr, nullptr, out);
}

bgs_status bgs_cloud_upload_f16_cov_sh(bgs_context* ctx, uint32_t n, uint32_t sh_degree, const float* pos_vis,
                                       const uint32_t* sh_packed, const uint32_t* cov3d_opacity, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F16Cov, sh_degree, pos_vis, sh_packed, cov3d_opacity, nullptr, nullptr, out);
}

bgs_status bgs_cloud_upload_4d(bgs_context* ctx, uint32_t n, const float* pos_vis, const float* sh, const float* rotations,
                               const float* scale_opacity, const float* timestamp_timescale, bgs_cloud** out) {
    return upload_common(ctx, n, CloudLayout::F32x4D, SH_DEGREE_MAX, pos_vis, sh, rotations, scale_opacity, timestamp_timescale,
                         out);
}

// ---- KHR_gaussian_splatting primitives (khr.cu; the rule: include/bgs.h)

bgs_status bgs_cloud_upload_khr(bgs_context* ctx, const bgs_khr_primitive* prim, uint32_t f16, uint32_t* out_zero_quats,
                                bgs_cloud** out) {
    if (!ctx || !out) return BGS_EINVAL;
    *out = nullptr;
    if (!prim) return fail(ctx, BGS_EINVAL, "upload_khr: null primitive");
    const uint32_t n = prim->n, d = prim->sh_degree;
    if (n == 0 || n >= (1u << 30)) return fail(ctx, BGS_EINVAL, "upload_khr: n must be in [1, 2^30)");
    if (d > SH_DEGREE_MAX) return fail(ctx, BGS_EINVAL, "upload_khr: sh_degree %u is not in [0, 3]", d);
    static const char* const kSh[16] = {"SH_DEGREE_0_COEF_0", "SH_DEGREE_1_COEF_0", "SH_DEGREE_1_COEF_1", "SH_DEGREE_1_COEF_2",
                                        "SH_DEGREE_2_COEF_0", "SH_DEGREE_2_COEF_1", "SH_DEGREE_2_COEF_2", "SH_DEGREE_2_COEF_3",
                                        "SH_DEGREE_2_COEF_4", "SH_DEGREE_3_COEF_0", "SH_DEGREE_3_COEF_1", "SH_DEGREE_3_COEF_2",
                                        "SH_DEGREE_3_COEF_3", "SH_DEGREE_3_COEF_4", "SH_DEGREE_3_COEF_5", "SH_DEGREE_3_COEF_6"};
    // slots 0..3 the required attributes, then COLOR_0 (without SH) or the SH coefficients
    const bool has_sh = d > 0 || prim->sh[0].data;
    const uint32_t bands = has_sh ? sh_bands(d) : 0u;
    std::vector<KhrSlot> slots = {{"POSITION", &prim->position}, {"ROTATION", &prim->rotation}, {"SCALE", &prim->scale},
                                  {"OPACITY", &prim->opacity}};
    const bool has_color = !has_sh && prim->color_0.data;
    if (has_color) slots.push_back({"COLOR_0", &prim->color_0});
    for (uint32_t k = 0; k < bands; ++k) slots.push_back({kSh[k], &prim->sh[k]});
    for (size_t s = 0; s < slots.size(); ++s) TRY(khr_check(ctx, slots[s], s >= 4 && has_sh));
    CU(ctx, cudaSetDevice(ctx->device));

    // one device copy of each accessor's span, each at a 256 B boundary, then the two result words
    Layout l;
    std::vector<size_t> off(slots.size()), span(slots.size());
    for (size_t s = 0; s < slots.size(); ++s) {
        const bgs_khr_accessor& a = *slots[s].a;
        span[s] = (size_t)(n - 1) * a.byte_stride + (size_t)khr_component_bytes(a.component_type) * a.components;
        off[s] = l.add(span[s]);
    }
    const size_t o_words = l.add(8);
    const CloudLayout layout = f16 ? CloudLayout::F16 : CloudLayout::F32;
    bgs_cloud* cl = nullptr;
    TRY(new_cloud(ctx, "upload_khr", n, layout, bands ? d : 0u, &cl));
    StreamScratch scratch(ctx->stream);
    uint32_t zero_quats = 0;
    TRY(stage_and_repack(ctx, "upload_khr", cl, [&](void* const* dp) {
        cudaError_t e = scratch.alloc(l.end);
        uint8_t* base = static_cast<uint8_t*>(scratch.p);
        KhrDecode k{};
        KhrSrc* src[5 + 16] = {&k.position, &k.rotation, &k.scale, &k.opacity, has_color ? &k.color : &k.sh[0]};
        for (uint32_t j = 1; j < bands; ++j) src[4 + j] = &k.sh[j];
        for (size_t s = 0; s < slots.size() && e == cudaSuccess; ++s) {
            const bgs_khr_accessor& a = *slots[s].a;
            *src[s] = KhrSrc{base + off[s], a.byte_stride, a.component_type, a.normalized};
            e = cudaMemcpyAsync(base + off[s], a.data, span[s], cudaMemcpyHostToDevice, ctx->stream);
        }
        uint32_t words[2] = {0, 0};
        uint32_t* d_words = reinterpret_cast<uint32_t*>(base + o_words);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_words, 0, 8, ctx->stream);
        if (e == cudaSuccess) {
            k.n = n; k.bands = bands; k.sh_units = (uint32_t)(staged_bytes(layout, cl->sh_degree, PLANE_SH) / 16);
            launch_khr_decode(k, f16 != 0, cl->pos, dp[PLANE_SH], dp[PLANE_ROT], dp[PLANE_SO], d_words, ctx->stream);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(words, d_words, 8, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) return fail(ctx, status_of(e), "upload_khr: %s", cudaGetErrorString(e));
        static const char* const kRule[6] = {"POSITION contains non-finite values", "ROTATION is non-finite after normalising",
                                             "SCALE gives a non-finite exp(scale)", "OPACITY is NaN or outside [0, 1]",
                                             "an SH coefficient is non-finite", "COLOR_0 contains non-finite values"};
        for (int b = 0; b < 6; ++b)
            if (words[0] & (1u << b)) return fail(ctx, BGS_EINVAL, "upload_khr: %s", kRule[b]);
        zero_quats = words[1];
        return BGS_OK;
    }, out));
    if (out_zero_quats) *out_zero_quats = zero_quats;
    return BGS_OK;
}

bgs_status bgs_cloud_sh_degree(const bgs_cloud* cl, uint32_t* out) {
    if (!cl || !out) return BGS_EINVAL;
    *out = cl->sh_degree;
    return BGS_OK;
}

void bgs_cloud_destroy(bgs_cloud* cl) {
    if (!cl) return;
    cudaSetDevice(cl->device);
    {
        // every live context (clouds are shared by the contexts of one GPU) drops its references: queued frames
        // that still read the planes are drained first, the debug hooks lose their frame.  Contexts with queued
        // interpolations (which may read this cloud) are drained too.
        std::lock_guard<std::mutex> lk(g_registry_mu);
        for (bgs_context* c : g_contexts) {
            if (c->device == cl->device && c->reads_pending.load(std::memory_order_relaxed))
                c->each_stream([](cudaStream_t& s, int) { cudaStreamSynchronize(s); });
            if (c->pend.reads(cl) || c->last.reads(cl)) {
                if (c->async_pending || c->pend.reads(cl)) c->each_stream([](cudaStream_t& s, int) { cudaStreamSynchronize(s); });
                if (c->pend.reads(cl)) { c->pend.forget(); c->pend.n = 0; }
                if (c->last.reads(cl)) { c->last.forget(); c->have_frame = false; }
            }
        }
        detach_listed_cloud(cl);   // (entity lists: their frames are drained above; rendering them is refused until repaired)
    }
    if (cl->ev_write) {   // particle steps still queued on any context write the planes
        cudaEventSynchronize(cl->ev_write);
        cudaEventDestroy(cl->ev_write);
    }
    cudaFree(cl->pos); cudaFree(cl->blocks);
    delete cl;
}

// ---- selection edits of a resident cloud (select.cu).  The visibility lane lives in both of the cloud's copies
// (cloud_layout.cuh): every write updates both.

bgs_status bgs_cloud_select_sparse(bgs_context* c, bgs_cloud* cl, float radius, uint32_t threshold, uint32_t* out_selected) {
    if (!cl) return fail(c, BGS_EINVAL, "select_sparse: null cloud");
    if (!(radius >= 0.0f) || std::isinf(radius)) return fail(c, BGS_EINVAL, "select_sparse: radius must be finite and >= 0");
    TRY(enter_call(c, "select_sparse", cl->device));
    TRY(before_cloud_write(c, cl));
    const uint32_t n = cl->n;
    const float r2 = radius * radius;
    cudaStream_t q = c->stream;
    uint32_t selected = 0;
    if (threshold == 0u || r2 == 0.0f) {
        // no count can reach a threshold of 0; no distance is below a radius whose square is 0 (every count is 0)
        selected = threshold == 0u ? 0u : n;
        launch_select_fill(cl->view(), n, threshold == 0u ? 0.0f : 1.0f, q);
        CU(c, cudaGetLastError());
        CU(c, cudaStreamSynchronize(q));
    } else {
        // the frame's scratch: key / value ping-pong buffers and depth-sort status rows (the sort), the record buffer
        // (positions in bucket order).  The debug hooks lose the last frame; the hints the next frame plans from stay.
        TRY(ensure_cloud_scratch(c, n));
        TRY(ensure_status(c, c->status_depth, c->status_n, n));
        const uint32_t nb = select_num_buckets(n);
        const int passes = select_sort_passes(nb);
        Layout l;
        const size_t o_words = l.add(3 * 4), o_hist = l.add(4 * 256 * 4);
        const size_t o_rng = l.add(((size_t)nb + 1) * sizeof(uint2));   // nb + 1: the sentinel key's too
        TRY(c->select_scratch.grow(c, l.end, false));
        c->have_frame = false;
        uint32_t* words = reinterpret_cast<uint32_t*>(c->select_scratch.p + o_words);   // [0] sort count, [1] barrier, [2] selected
        uint32_t* hist = reinterpret_cast<uint32_t*>(c->select_scratch.p + o_hist);
        uint2* ranges = reinterpret_cast<uint2*>(c->select_scratch.p + o_rng);
        CU(c, cudaMemsetAsync(c->select_scratch.p, 0, l.end, q));
        launch_select_keys(cl->pos, n, radius, nb, c->keys[0].p, c->vals[0].p, &words[0], q);
        CU(c, cudaGetLastError());
        CU(c, launch_radix_sort(c->keys[0].p, c->vals[0].p, c->keys[1].p, c->vals[1].p, &words[0], n, n, hist, 1,
                                c->status_depth.p, (size_t)radix_num_tiles(c->status_n) * 256, next_epoch(c), &words[1], passes,
                                0, ranges, c->sm_count, c->rs_per_sm, q));
        launch_select_count(cl->view(), c->vals[passes & 1].p, ranges, n, radius, nb, r2, threshold,
                            reinterpret_cast<float4*>(c->recs.p), &words[2], q);
        CU(c, cudaGetLastError());
        TRY(read_word(c, &words[2], &selected));
    }
    if (out_selected) *out_selected = selected;
    return BGS_OK;
}

bgs_status bgs_cloud_visibility_get(bgs_context* c, const bgs_cloud* cl, float* out_vis) {
    if (!cl || !out_vis) return fail(c, BGS_EINVAL, "visibility_get: null cloud or array");
    TRY(enter_call(c, "visibility_get", cl->device));
    TRY(before_cloud_read(c, cl));
    CU(c, cudaMemcpy2DAsync(out_vis, 4, &cl->pos->w, sizeof(float4), 4, cl->n, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

bgs_status bgs_cloud_visibility_set(bgs_context* c, bgs_cloud* cl, const float* vis) {
    if (!cl || !vis) return fail(c, BGS_EINVAL, "visibility_set: null cloud or array");
    TRY(enter_call(c, "visibility_set", cl->device));
    TRY(before_cloud_write(c, cl));
    const CloudView v = cl->view();
    CU(c, cudaMemcpy2DAsync(&v.pos->w, sizeof(float4), vis, 4, 4, cl->n, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpy2DAsync(&reinterpret_cast<float4*>(v.blocks)[POS_CHUNK].w, block_bytes(cl->layout, cl->sh_degree), vis, 4, 4,
                            cl->n,
                            cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

bgs_status bgs_cloud_select_in_mesh(bgs_context* c, bgs_cloud* cl, const float* vertices, uint32_t nv, const uint32_t* indices,
                                    uint32_t nt, const float* mesh_from_cloud, uint32_t mode, uint32_t* out_inside) {
    if (!cl) return fail(c, BGS_EINVAL, "select_in_mesh: null cloud");
    if (nt > 0 && (!vertices || !indices)) return fail(c, BGS_EINVAL, "select_in_mesh: null vertices or indices");
    if (mode != BGS_SELECT_REPLACE && mode != BGS_SELECT_ADD) return fail(c, BGS_EINVAL, "select_in_mesh: unknown mode %u", mode);
    TRY(enter_call(c, "select_in_mesh", cl->device));
    for (size_t k = 0; k < (size_t)nt * 3; ++k)
        if (indices[k] >= nv) return fail(c, BGS_EINVAL, "select_in_mesh: index %u of triangle %zu is >= %u vertices", indices[k], k / 3, nv);
    if (nt >= (1u << 26)) return fail(c, BGS_ENOMEM, "select_in_mesh: more than 2^26 triangles");
    static const float identity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const float* M = mesh_from_cloud ? mesh_from_cloud : identity;
    TRY(before_cloud_write(c, cl));
    const uint32_t n = cl->n;
    cudaStream_t q = c->stream;

    // triangle side: setup (records, classes, grid bounds)
    Layout lt;
    const size_t o_w = lt.add(256);   // (mesh_words_bytes() <= 256)
    const size_t o_v = lt.add((size_t)nv * 12), o_i = lt.add((size_t)nt * 12);
    const size_t o_br = lt.add((size_t)nt * (2 * mesh_rec_bytes() + 32));   // binned records | binned boxes | global records
    const size_t o_bb = o_br + (size_t)nt * mesh_rec_bytes(), o_gr = o_bb + (size_t)nt * 32;
    TRY(c->mesh_tri.grow(c, lt.end, false));
    uint8_t* tb = c->mesh_tri.p;
    void* words = tb + o_w;
    std::vector<unsigned long long> wh_buf((mesh_words_bytes() + 7) / 8);
    void* wh = wh_buf.data();
    CU(c, cudaMemsetAsync(words, 0, 256, q));
    if (nt > 0) {
        CU(c, cudaMemcpyAsync(tb + o_v, vertices, (size_t)nv * 12, cudaMemcpyHostToDevice, q));
        CU(c, cudaMemcpyAsync(tb + o_i, indices, (size_t)nt * 12, cudaMemcpyHostToDevice, q));
        launch_mesh_setup(reinterpret_cast<const float*>(tb + o_v), reinterpret_cast<const uint32_t*>(tb + o_i), nt, tb + o_br,
                          tb + o_bb, tb + o_gr, words, q);
        CU(c, cudaGetLastError());
    }
    CU(c, cudaMemcpyAsync(wh, words, mesh_words_bytes(), cudaMemcpyDeviceToHost, q));
    CU(c, cudaStreamSynchronize(q));

    // grid side: the level, the pairs, their sort by cell
    int level = -1;
    const uint32_t* cell_tri = nullptr;
    const uint2* ranges = nullptr;
    if (mesh_words_n_bin(wh) > 0) {
        launch_mesh_levels(tb + o_bb, wh, words, q);
        CU(c, cudaGetLastError());
        CU(c, cudaMemcpyAsync(wh, words, mesh_words_bytes(), cudaMemcpyDeviceToHost, q));
        CU(c, cudaStreamSynchronize(q));
        uint64_t pairs64 = 0;
        uint32_t cells = 0;
        mesh_pick_level(wh, &level, &pairs64, &cells);
        const uint32_t pairs = (uint32_t)pairs64;
        Layout lp;
        const size_t o_hist = lp.add(4 * 256 * 4), o_rng = lp.add((size_t)cells * 8);
        const size_t o_k0 = lp.add((size_t)pairs * 4), o_v0 = lp.add((size_t)pairs * 4);
        const size_t o_k1 = lp.add((size_t)pairs * 4), o_v1 = lp.add((size_t)pairs * 4);
        TRY(c->mesh_pairs.grow(c, lp.padded(), false));
        TRY(ensure_status(c, c->status_pairs, c->status_np, pairs));
        uint8_t* pb = c->mesh_pairs.p;
        uint32_t* k0 = reinterpret_cast<uint32_t*>(pb + o_k0);
        uint32_t* v0 = reinterpret_cast<uint32_t*>(pb + o_v0);
        uint32_t* k1 = reinterpret_cast<uint32_t*>(pb + o_k1);
        uint32_t* v1 = reinterpret_cast<uint32_t*>(pb + o_v1);
        uint2* rng = reinterpret_cast<uint2*>(pb + o_rng);
        CU(c, cudaMemsetAsync(pb, 0, o_k0, q));   // histograms and ranges
        launch_mesh_emit(tb + o_bb, wh, level, k0, v0, words, q);
        CU(c, cudaGetLastError());
        const int passes = pair_passes(cells);
        CU(c, launch_radix_sort(k0, v0, k1, v1, mesh_words_pairs(words), pairs, pairs, reinterpret_cast<uint32_t*>(pb + o_hist), 1,
                                c->status_pairs.p, (size_t)radix_num_tiles(c->status_np) * 256, next_epoch(c),
                                mesh_words_barrier(words), passes, 0, rng, c->sm_count, c->rs_per_sm, q));
        cell_tri = (passes & 1) ? v1 : v0;
        ranges = rng;
    }

    // point side: the count and the lane
    launch_mesh_count(cl->view(), n, M, tb + o_br, tb + o_gr, cell_tri, ranges, wh, level, mode, words, q);
    CU(c, cudaGetLastError());
    uint32_t inside = 0;
    TRY(read_word(c, mesh_words_inside(words), &inside));
    if (out_inside) *out_inside = inside;
    return BGS_OK;
}

bgs_status bgs_cloud_select_in_view(bgs_context* c, bgs_cloud* cl, const bgs_cloud_uniform* uni, const bgs_view* view,
                                    const uint8_t* mask, int mask_is_device_ptr, uint32_t mode, uint32_t* out_inside) {
    if (!c) return BGS_EINVAL;
    if (!cl || !uni || !view || !mask) return fail(c, BGS_EINVAL, "select_in_view: null cloud, uniform, view or mask");
    if (mode != BGS_SELECT_REPLACE && mode != BGS_SELECT_ADD) return fail(c, BGS_EINVAL, "select_in_view: unknown mode %u", mode);
    TRY(enter_call(c, "select_in_view", cl->device));
    if (is_4d(cl->layout))
        return fail(c, BGS_EINVAL, "select_in_view: a Gaussian4d cloud (its drawn position depends on time: use bgs_render_entities_pick)");
    const int W = (int)view->viewport[2], H = (int)view->viewport[3];
    if (W <= 0 || H <= 0 || W > 65535 || H > 65535) return fail(c, BGS_EINVAL, "select_in_view: viewport %dx%d out of range", W, H);
    if (mask_is_device_ptr) {
        cudaPointerAttributes a = {};
        const cudaError_t e = cudaPointerGetAttributes(&a, mask);
        if (e != cudaSuccess) cudaGetLastError();   // (an unknown pointer: clear the error, refuse below)
        if (e != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != c->device)
            return fail(c, BGS_EINVAL, "select_in_view: mask %p is not device memory of device %d", (const void*)mask, c->device);
    }
    // the render calls' frame constants: only the model, the clip matrix and the viewport are read
    bgs_settings st = {};
    st.radix_sort_depth_bits = 32;
    const FrameConsts fc = frame_consts(cl, view, uni, &st, false);
    TRY(before_cloud_write(c, cl));
    cudaStream_t q = c->stream;
    const size_t mask_bytes = (size_t)W * H;
    TRY(c->view_select.grow(c, 256 + (mask_is_device_ptr ? 0 : mask_bytes), false));
    uint32_t* word = reinterpret_cast<uint32_t*>(c->view_select.p);
    const uint8_t* dmask = mask;
    if (!mask_is_device_ptr) {
        CU(c, cudaMemcpyAsync(c->view_select.p + 256, mask, mask_bytes, cudaMemcpyHostToDevice, q));
        dmask = c->view_select.p + 256;
    }
    CU(c, cudaMemsetAsync(word, 0, 4, q));
    launch_view_select(cl->view(), cl->n, fc, dmask, mode, word, q);
    CU(c, cudaGetLastError());
    uint32_t inside = 0;
    TRY(read_word(c, word, &inside));
    if (out_inside) *out_inside = inside;
    return BGS_OK;
}

// ---- particle behaviours (particles.cu).  The step is a queued write (host.cuh: queue_cloud_write), never drained;
// it also orders itself after the behaviours' earlier steps and marks itself on them.

bgs_status bgs_particles_create(bgs_context* c, const bgs_particle_behavior* behaviors, uint32_t count, bgs_particles** out) {
    if (!c || !out) return BGS_EINVAL;
    *out = nullptr;
    if (!behaviors) return fail(c, BGS_EINVAL, "particles_create: null behaviours");
    if (count == 0 || count >= (1u << 30)) return fail(c, BGS_EINVAL, "particles_create: count must be in [1, 2^30)");
    static_assert(sizeof(bgs_particle_behavior) == 64, "ParticleBehavior is 64 B");
    std::vector<uint32_t> active;
    active.reserve(count);
    for (uint32_t i = 0; i < count; ++i)
        if (behaviors[i].indices[0] < 0x80000000u) active.push_back(behaviors[i].indices[0]);
    std::sort(active.begin(), active.end());
    const auto dup = std::adjacent_find(active.begin(), active.end());
    if (dup != active.end()) return fail(c, BGS_EINVAL, "particles_create: two active behaviours name gaussian %u", *dup);
    CU(c, cudaSetDevice(c->device));
    bgs_particles* p = new (std::nothrow) bgs_particles();
    if (!p) return BGS_ENOMEM;
    p->device = c->device;
    p->count = count;
    p->max_index = active.empty() ? -1 : (int64_t)active.back();
    cudaError_t e = cudaMalloc(&p->d, (size_t)count * 64);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_write, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMemcpyAsync(p->d, behaviors, (size_t)count * 64, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        bgs_particles_destroy(p);
        return fail(c, status_of(e), "particles_create: %s", cudaGetErrorString(e));
    }
    *out = p;
    return BGS_OK;
}

bgs_status bgs_particles_get(bgs_context* c, const bgs_particles* p, bgs_particle_behavior* out) {
    if (!p || !out) return fail(c, BGS_EINVAL, "particles_get: null behaviours or array");
    TRY(enter_call(c, "particles_get", p->device, "behaviours live"));
    CU(c, cudaStreamWaitEvent(c->stream, p->ev_write, 0));   // every step of these behaviours, on any context
    CU(c, cudaMemcpyAsync(out, p->d, (size_t)p->count * 64, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

void bgs_particles_destroy(bgs_particles* p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->ev_write) {   // steps still queued on any context read and write the records
        cudaEventSynchronize(p->ev_write);
        cudaEventDestroy(p->ev_write);
    }
    cudaFree(p->d);
    delete p;
}

bgs_status bgs_cloud_particles_step(bgs_context* c, bgs_cloud* cl, bgs_particles* p, float delta_time) {
    if (!cl || !p) return fail(c, BGS_EINVAL, "particles_step: null cloud or behaviours");
    if (!std::isfinite(delta_time)) return fail(c, BGS_EINVAL, "particles_step: delta_time must be finite");
    // (-1: the two are on different devices, so neither can be the context's)
    TRY(enter_call(c, "particles_step", cl->device == p->device ? cl->device : -1, "cloud or behaviours live"));
    if (p->max_index >= (int64_t)cl->n)
        return fail(c, BGS_EINVAL, "particles_step: behaviour names gaussian %lld of a cloud of %u", (long long)p->max_index, cl->n);
    TRY(queue_cloud_write(c, cl, [&](cudaStream_t q) {
        CU(c, cudaStreamWaitEvent(q, p->ev_write, 0));
        launch_particle_step(p->d, p->count, delta_time, cl->view(), q);
        CU(c, cudaGetLastError());
        CU(c, cudaEventRecord(p->ev_write, q));
        return BGS_OK;
    }));
    c->step_pending = true;
    return BGS_OK;
}

bgs_status bgs_cloud_positions_get(bgs_context* c, const bgs_cloud* cl, float* out_pos_vis) {
    if (!cl || !out_pos_vis) return fail(c, BGS_EINVAL, "positions_get: null cloud or array");
    TRY(enter_call(c, "positions_get", cl->device));
    TRY(before_cloud_read(c, cl));
    CU(c, cudaMemcpyAsync(out_pos_vis, cl->pos, (size_t)cl->n * 16, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return BGS_OK;
}

// ---- interpolation (interpolate.cu).  A queued write of `out` that reads `lhs` and `rhs` (host.cuh:
// queue_cloud_write_reading), never drained.

// interpolate.wgsl:51-57 in f32: false (t untouched) for non-finite inputs or a NaN factor
static bool interpolation_factor(float time, float time_start, float time_stop, float* t) {
    if (!std::isfinite(time) || !std::isfinite(time_start) || !std::isfinite(time_stop)) return false;
    const float d = time_stop - time_start;
    float f;
    if (std::fabs(d) < 1e-6f) f = time >= time_stop ? 1.0f : 0.0f;
    else f = std::min(std::max((time - time_start) / d, 0.0f), 1.0f);
    if (std::isnan(f)) return false;   // (std::max / std::min would pass NaN through; it is caught here)
    *t = f;
    return true;
}

bgs_status bgs_cloud_interpolate(bgs_context* c, bgs_cloud* out, const bgs_cloud* lhs, const bgs_cloud* rhs, float time,
                                 float time_start, float time_stop) {
    if (!out || !lhs || !rhs) return fail(c, BGS_EINVAL, "interpolate: null cloud");
    // (-1: the three are not on one device, so not all are on the context's)
    TRY(enter_call(c, "interpolate", lhs->device == out->device && rhs->device == out->device ? out->device : -1, "clouds live"));
    if (lhs->n != out->n || rhs->n != out->n)
        return fail(c, BGS_EINVAL, "interpolate: lhs, rhs and out hold %u, %u and %u gaussians", lhs->n, rhs->n, out->n);
    if (lhs->layout != out->layout || rhs->layout != out->layout)
        return fail(c, BGS_EINVAL, "interpolate: lhs, rhs and out are not in one layout");
    if (lhs->sh_degree != out->sh_degree || rhs->sh_degree != out->sh_degree)
        return fail(c, BGS_EINVAL, "interpolate: lhs, rhs and out have SH degrees %u, %u and %u", lhs->sh_degree, rhs->sh_degree,
                    out->sh_degree);
    if (is_4d(out->layout)) return fail(c, BGS_EINVAL, "interpolate: Gaussian4d clouds are not interpolated");
    if (out == lhs || out == rhs) return fail(c, BGS_EINVAL, "interpolate: out is lhs or rhs");
    float t = 0.0f;
    if (!interpolation_factor(time, time_start, time_stop, &t))
        return fail(c, BGS_EINVAL, "interpolate: time %g, time_start %g, time_stop %g give no factor", time, time_start, time_stop);
    return queue_cloud_write_reading(c, out, lhs, rhs, [&](cudaStream_t q) {
        launch_interpolate(out->layout, out->sh_degree, lhs->view(), rhs->view(), out->n, t, out->view(), q);
        CU(c, cudaGetLastError());
        return BGS_OK;
    });
}

// ---- transform and bounds (transform.cu).  The transform is a queued write (host.cuh: queue_cloud_write), never
// drained, as the particle step is; the bounds only read the cloud (before_cloud_read), into their own words.

bgs_status bgs_cloud_transform(bgs_context* c, bgs_cloud* cl, const float* local_from_local, uint32_t mode) {
    if (!cl || !local_from_local) return fail(c, BGS_EINVAL, "transform: null cloud or matrix");
    if (mode != BGS_TRANSFORM_ALL && mode != BGS_TRANSFORM_SELECTED) return fail(c, BGS_EINVAL, "transform: unknown mode %u", mode);
    TRY(enter_call(c, "transform", cl->device));
    if (is_4d(cl->layout)) return fail(c, BGS_EINVAL, "transform: Gaussian4d clouds are not transformed");
    TransformParams P;
    const char* why = "";
    if (!transform_params(local_from_local, &P, &why)) return fail(c, BGS_EINVAL, "transform: %s", why);
    TRY(queue_cloud_write(c, cl, [&](cudaStream_t q) {
        launch_transform(cl->layout, cl->sh_degree, cl->view(), cl->n, P, mode == BGS_TRANSFORM_SELECTED, q);
        CU(c, cudaGetLastError());
        return BGS_OK;
    }));
    c->step_pending = true;
    return BGS_OK;
}

bgs_status bgs_cloud_bounds(bgs_context* c, const bgs_cloud* cl, uint32_t mode, float out_min[3], float out_max[3],
                            uint32_t* out_count) {
    if (!cl || !out_min || !out_max) return fail(c, BGS_EINVAL, "bounds: null cloud or output");
    if (mode != BGS_TRANSFORM_ALL && mode != BGS_TRANSFORM_SELECTED) return fail(c, BGS_EINVAL, "bounds: unknown mode %u", mode);
    TRY(enter_call(c, "bounds", cl->device));
    TRY(before_cloud_read(c, cl));
    cudaStream_t q = c->stream;
    TRY(c->bounds_words.grow(c, 7 * 4, false));
    uint32_t* words = c->bounds_words.p;
    CU(c, cudaMemsetAsync(words, 0xFF, 3 * 4, q));
    CU(c, cudaMemsetAsync(words + 3, 0, 4 * 4, q));
    launch_bounds(cl->pos, cl->n, mode == BGS_TRANSFORM_SELECTED, words, c->sm_count, q);
    CU(c, cudaGetLastError());
    uint32_t h[7];
    CU(c, cudaMemcpyAsync(h, words, sizeof h, cudaMemcpyDeviceToHost, q));
    CU(c, cudaStreamSynchronize(q));
    auto decode = [](uint32_t k) {
        const uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
        float f;
        memcpy(&f, &u, 4);
        return f;
    };
    for (int k = 0; k < 3; ++k) {
        out_min[k] = h[6] ? decode(h[k]) : INFINITY;
        out_max[k] = h[6] ? decode(h[3 + k]) : -INFINITY;
    }
    if (out_count) *out_count = h[6];
    return BGS_OK;
}

// ---- subset and download (subset.cu).  Both only read the source cloud (before_cloud_read), so neither drains another
// context's frames.  Their scratch is their own, allocated and released on the render stream within the call
// (stream-ordered: no device-wide synchronisation), so the frame's buffers, the debug hooks and the next frame's plan
// are untouched.

bgs_status bgs_cloud_subset(bgs_context* c, const bgs_cloud* cl, const uint32_t* indices, uint32_t k, bgs_cloud** out,
                            uint32_t* out_n) {
    if (out) *out = nullptr;
    if (!cl || !out) return fail(c, BGS_EINVAL, "subset: null cloud or out");
    TRY(enter_call(c, "subset", cl->device));
    if (!indices && k != 0) return fail(c, BGS_EINVAL, "subset: selection mode (indices == NULL) takes k == 0");
    if (indices && (k == 0 || k >= (1u << 30))) return fail(c, BGS_EINVAL, "subset: k must be in [1, 2^30)");
    for (uint32_t j = 0; indices && j < k; ++j)
        if (indices[j] >= cl->n) return fail(c, BGS_EINVAL, "subset: index %u at %u is >= the cloud's %u gaussians", indices[j], j, cl->n);
    TRY(before_cloud_read(c, cl));
    cudaStream_t q = c->stream;
    const uint32_t n = cl->n;
    StreamScratch scratch(q);
    // selection mode: mask words | CTA counts (-> offsets) | the total
    Layout l;
    const size_t o_mask = l.add((size_t)(n + 31) / 32 * 4), o_cnt = l.add((size_t)subset_num_ctas(n) * 4), o_tot = l.add(4);
    uint32_t kept = k;
    if (!indices) {
        CU(c, scratch.alloc(l.end));
        uint8_t* s = static_cast<uint8_t*>(scratch.p);
        launch_subset_count(cl->pos, n, reinterpret_cast<uint32_t*>(s + o_mask), reinterpret_cast<uint32_t*>(s + o_cnt),
                            reinterpret_cast<uint32_t*>(s + o_tot), q);
        CU(c, cudaGetLastError());
        TRY(read_word(c, reinterpret_cast<const uint32_t*>(s + o_tot), &kept));
        if (kept == 0) {
            if (out_n) *out_n = 0;
            return BGS_OK;
        }
    } else {
        CU(c, scratch.alloc((size_t)k * 4));
        CU(c, cudaMemcpyAsync(scratch.p, indices, (size_t)k * 4, cudaMemcpyHostToDevice, q));
    }
    bgs_cloud* nc = nullptr;
    TRY(new_cloud(c, "subset", kept, cl->layout, cl->sh_degree, &nc));
    if (!indices) {
        const uint8_t* s = static_cast<const uint8_t*>(scratch.p);
        launch_subset_scatter(cl->layout, cl->sh_degree, cl->view(), n, reinterpret_cast<const uint32_t*>(s + o_mask),
                              reinterpret_cast<const uint32_t*>(s + o_cnt), nc->view(), q);
    } else {
        launch_subset_gather(cl->layout, cl->sh_degree, cl->view(), static_cast<const uint32_t*>(scratch.p), k, nc->view(), q);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(q);
    if (e != cudaSuccess) return drop_cloud(c, "subset", nc, e);
    *out = nc;
    if (out_n) *out_n = kept;
    return BGS_OK;
}

// Per chunk: unpack into device staging, copy the chunk's position plane and the staged planes to a pinned bounce
// buffer, and -- while the next chunk goes the same way into the other bounce buffer -- copy it into the caller's arrays.
// any_degree: a call of the _sh family, which takes the SH plane at the cloud's degree; the others take degree 3 only.
static bgs_status download_common(bgs_context* c, const bgs_cloud* cl, int family, bool any_degree, float* pos_vis, void* sh,
                                  void* rot, void* so, void* tt) {
    if (!cl || !pos_vis || !sh || !rot || (family != 1 && !so) || (family == 2 && !tt))
        return fail(c, BGS_EINVAL, "download: null cloud or plane pointer");
    TRY(enter_call(c, "download", cl->device));
    const CloudLayout l = cl->layout;
    const uint32_t d = cl->sh_degree;
    static const char* const kFamily[3] = {"f32", "f16", "4D"};
    if (download_family(l) != family) return fail(c, BGS_EINVAL, "download: the cloud is in the %s layout", kFamily[download_family(l)]);
    if (!any_degree && d != SH_DEGREE_MAX)
        return fail(c, BGS_EINVAL, "download: the cloud has SH degree %u (bgs_cloud_download_%s_sh reads it)", d, kFamily[family]);
    TRY(before_cloud_read(c, cl));
    cudaStream_t q = c->stream;
    const uint32_t n = cl->n, m_max = std::min<uint32_t>(n, (uint32_t)(DOWNLOAD_BOUNCE_BYTES / planar_bytes(l, d)));
    // (sized once for the largest chunk of either layout: it never grows)
    if (!c->h_bounce) CU(c, cudaMallocHost(&c->h_bounce, 2 * DOWNLOAD_BOUNCE_BYTES));
    const size_t chunk_b = DOWNLOAD_BOUNCE_BYTES;
    StreamScratch staging(q);   // sh | rot | so | tt of one chunk, the SH plane at whole chunks per gaussian
    size_t staged_total = 0;
    for (int p = PLANE_SH; p < PLANES; ++p) staged_total += staged_bytes(l, d, p);
    CU(c, staging.alloc((size_t)m_max * staged_total));
    uint8_t* st[PLANES] = {nullptr, static_cast<uint8_t*>(staging.p)};
    for (int p = PLANE_SH + 1; p < PLANES; ++p) st[p] = st[p - 1] + (size_t)m_max * staged_bytes(l, d, p - 1);
    cudaEvent_t ev[2] = {nullptr, nullptr};
    struct Events { cudaEvent_t* e; ~Events() { for (int k = 0; k < 2; ++k) if (e[k]) cudaEventDestroy(e[k]); } } ev_guard{ev};
    for (cudaEvent_t& e : ev) CU(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    uint8_t* dst[PLANES] = {reinterpret_cast<uint8_t*>(pos_vis), static_cast<uint8_t*>(sh), static_cast<uint8_t*>(rot),
                            static_cast<uint8_t*>(so), static_cast<uint8_t*>(tt)};
    const uint32_t chunks = (n + m_max - 1) / m_max;
    // enqueue chunk i into bounce buffer i & 1
    auto enqueue = [&](uint32_t i) -> bgs_status {
        const uint32_t lo = i * m_max, m = std::min(m_max, n - lo);
        uint8_t* hb = c->h_bounce + (i & 1) * chunk_b;
        launch_unpack(l, d, cl->view(), lo, m, st[PLANE_SH], st[PLANE_ROT], st[PLANE_SO], st[PLANE_TT], q);
        CU(c, cudaGetLastError());
        const uint8_t* src[PLANES] = {reinterpret_cast<const uint8_t*>(cl->pos + lo), st[PLANE_SH], st[PLANE_ROT], st[PLANE_SO],
                                      st[PLANE_TT]};
        for (int p = 0; p < PLANES; ++p) {
            const size_t width = plane_bytes(l, d, p);
            if (width) CU(c, copy_rows(hb, width, src[p], p == PLANE_POS ? width : staged_bytes(l, d, p), width, m,
                                       cudaMemcpyDeviceToHost, q));
            hb += (size_t)m * width;
        }
        CU(c, cudaEventRecord(ev[i & 1], q));
        return BGS_OK;
    };
    TRY(enqueue(0));
    for (uint32_t i = 0; i < chunks; ++i) {
        if (i + 1 < chunks) TRY(enqueue(i + 1));
        CU(c, cudaEventSynchronize(ev[i & 1]));
        const uint32_t lo = i * m_max, m = std::min(m_max, n - lo);
        const uint8_t* hb = c->h_bounce + (i & 1) * chunk_b;
        for (int p = 0; p < PLANES; ++p) {
            const size_t b = plane_bytes(l, d, p);
            if (b) memcpy(dst[p] + (size_t)lo * b, hb, (size_t)m * b);
            hb += (size_t)m * b;
        }
    }
    return BGS_OK;
}

bgs_status bgs_cloud_download_f32(bgs_context* c, const bgs_cloud* cl, float* pos_vis, float* sh, float* rot_wxyz, float* scale_opacity) {
    return download_common(c, cl, 0, false, pos_vis, sh, rot_wxyz, scale_opacity, nullptr);
}

bgs_status bgs_cloud_download_f16(bgs_context* c, const bgs_cloud* cl, float* pos_vis, uint32_t* sh_packed, uint32_t* second_plane) {
    return download_common(c, cl, 1, false, pos_vis, sh_packed, second_plane, nullptr, nullptr);
}

bgs_status bgs_cloud_download_f32_sh(bgs_context* c, const bgs_cloud* cl, float* pos_vis, float* sh, float* rot_wxyz,
                                     float* scale_opacity) {
    return download_common(c, cl, 0, true, pos_vis, sh, rot_wxyz, scale_opacity, nullptr);
}

bgs_status bgs_cloud_download_f16_sh(bgs_context* c, const bgs_cloud* cl, float* pos_vis, uint32_t* sh_packed,
                                     uint32_t* second_plane) {
    return download_common(c, cl, 1, true, pos_vis, sh_packed, second_plane, nullptr, nullptr);
}

bgs_status bgs_cloud_download_4d(bgs_context* c, const bgs_cloud* cl, float* pos_vis, float* sh, float* rotations,
                                 float* scale_opacity, float* timestamp_timescale) {
    return download_common(c, cl, 2, false, pos_vis, sh, rotations, scale_opacity, timestamp_timescale);
}

}  // extern "C"
