// transform_oracle.h -- CPU oracle of bgs_cloud_transform (include/bgs.h).  TEST INFRASTRUCTURE ONLY: it restates the
// rule scalar by scalar, with its own matrix check, quaternion and SH rotation builder, so that the GPU's result can be
// compared against it.  Built with -ffp-contract=off and no fast-math: every f32 operation is one IEEE
// round-to-nearest-even operation, in the order bgs.h pins.
#pragma once
#include <cstdint>

extern "C" {

enum { ORC_XF_F32 = 0, ORC_XF_F16 = 1, ORC_XF_COV = 2 };

// E = D_l^T row-major ((2l+1)^2 doubles) for the rotation R (row-major 3x3, f64), D_l defined by Y_l(R^T d) = D_l Y_l(d)
// over the renderer's band-l basis.  l in 1..3.
void orc_xf_sh_matrix(const double* R, int l, double* E);

// The matrix check and the kernel's constants: 0 and q_R (w, x, y, z), s and E_1, E_2, E_3 (f32) for a matrix the call
// accepts; 1 for one it refuses.  Any output pointer may be null.
int orc_xf_params(const float* M, float* q, float* s, float* E1, float* E2, float* E3);

// The transform of n gaussians given as their upload planes (f32: pos_vis, sh (S_d floats), rot, scale_opacity; f16
// and cov: pos_vis, sh_packed (S_d / 2 words), second plane), in place, at SH degree d; mode 0 all, 1 selected.
// sh_bound (n x S_d doubles, may be null): per SH lane, sum_j |E_ij c_j| in f64 over the lane's band (0 for lanes the
// transform does not touch).  Returns 1 (and changes nothing) for a matrix the call refuses.
int orc_xf_apply(uint32_t n, int layout, uint32_t d, const float* M, uint32_t mode, void* const* planes, double* sh_bound);

}
