/*
 * select_oracle.h -- CPU ORACLE of SparseSelect (src/query/sparse.rs:24-54).  TEST INFRASTRUCTURE ONLY: the product
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

#ifdef __cplusplus
}
#endif
#endif
