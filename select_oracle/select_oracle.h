/*
 * select_oracle.h -- CPU ORACLE of SparseSelect (src/query/sparse.rs:24-54) and of point-in-mesh selection.  TEST INFRASTRUCTURE ONLY: the product
 * (libbgs.so) never links, loads or calls it.  Built beside oracle/ (the render oracle) by __graft_entry__.build().
 *
 * The selection rule (include/bgs.h, bgs_cloud_select_sparse):
 *   - positions are the plane's x, y, z as uploaded (pos_vis[4i .. 4i + 2]); every gaussian takes part, whatever its
 *     visibility;
 *   - count_i = #{j : d2 < r2}, j == i included, d2 = ((dx*dx + dy*dy) + dz*dz), dx = x_j - x_i (likewise y, z),
 *     r2 = radius*radius rounded to f32; every operation f32 round-to-nearest-even, no FMA (-ffp-contract=off);
 *   - gaussian i is selected (out_mask[i] = 1) iff count_i < threshold.
 *   A non-finite position has a NaN d2 against everything, itself included: count 0.  radius == 0 counts nothing;
 *   threshold == 0 selects nothing.
 * PARITY STATUS: the reference delegates the comparison to the kd-tree 0.6.2 crate, whose source is not available
 * here: `<` against `<=` and the accumulation order are **unpinned**.
 *
 * Two implementations of the same expression:
 *   orc_select_sparse       brute force over every pair, O(N^2), OpenMP: the definition;
 *   orc_select_sparse_grid  the hashed grid of libbgs's select.cu (cell and bucket functions restated), so the CPU
 *                           tests reach the same cell boundaries and bucket collisions the GPU does.  Sizes the brute
 *                           force cannot reach (the GPU tests at 1-6 M gaussians) are checked against this one.
 * Both return 0, or -1 for a radius that is NaN, infinite or negative.  *out_selected (may be NULL) = popcount.
 */
#ifndef SELECT_ORACLE_H
#define SELECT_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

int orc_select_sparse(uint32_t n, const float* pos_vis, float radius, uint32_t threshold, uint8_t* out_mask,
                      uint32_t* out_selected, int threads);
int orc_select_sparse_grid(uint32_t n, const float* pos_vis, float radius, uint32_t threshold, uint8_t* out_mask,
                           uint32_t* out_selected, int threads);
/* The grid's functions, per gaussian: the bucket (n_buckets for a non-finite position), and the three cell
 * coordinates.  Returns n_buckets. */
uint32_t orc_select_buckets(uint32_t n, const float* pos_vis, float radius, uint32_t* out_bucket, int64_t* out_cell3);

/* Point in mesh (include/bgs.h, bgs_cloud_select_in_mesh; src/query/raycast.rs:54-124): out_mask[i] = 1 iff the +x
 * ray from mesh_from_cloud * (x, y, z, 1) (column-major, NULL = identity) hits an odd number of the nt triangles
 * (vertices nv x 3 f32, indices nt x 3 u32), each decided by ray_intersects_triangle (raycast.rs:92-124) in glam's
 * scalar Vec3 order, f32 without contraction.  PARITY STATUS: glam's operation order is **unpinned** (the crate is
 * absent here).
 *   orc_select_in_mesh       every (point, triangle) pair: the definition;
 *   orc_select_in_mesh_grid  libbgs's mesh_select.cu restated (triangle setup and classes, slack, grid ladder and
 *                            pair budget, cell function), so the CPU tests reach the cell boundaries the GPU does.
 * Both return 0, or -1 for null arrays with nt > 0 or an index >= nv.  *out_inside (may be NULL) = popcount.
 * orc_mesh_plan: out_counts = (binned, global, ny, nz) of the chosen level, *out_level (-1: no grid), *out_pairs.
 * orc_mesh_boxes: per triangle, class 0 dropped / 1 binned / 2 global and the binned box (ylo, yhi, zlo, zhi). */
int orc_select_in_mesh(uint32_t n, const float* pos_vis, uint32_t nv, const float* vertices, uint32_t nt, const uint32_t* indices,
                       const float* mesh_from_cloud, uint8_t* out_mask, uint32_t* out_inside, int threads);
int orc_select_in_mesh_grid(uint32_t n, const float* pos_vis, uint32_t nv, const float* vertices, uint32_t nt,
                            const uint32_t* indices, const float* mesh_from_cloud, uint8_t* out_mask, uint32_t* out_inside,
                            int threads);
int orc_mesh_plan(uint32_t nv, const float* vertices, uint32_t nt, const uint32_t* indices, uint32_t* out_counts,
                  int32_t* out_level, uint64_t* out_pairs);
int orc_mesh_boxes(uint32_t nv, const float* vertices, uint32_t nt, const uint32_t* indices, double* out_box, int32_t* out_class);

#ifdef __cplusplus
}
#endif
#endif
