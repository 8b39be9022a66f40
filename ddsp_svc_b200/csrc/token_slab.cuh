// The fixed run of frames of one utterance that a two-stage token sum adds in fp64 before the slabs are added in order
// (reflow_bwd.cu, diffusion_bwd.cu).  One constant for both: diffusion_bwd.cu's df_layer_backward writes its slab sums
// in the workspace layout that reflow_bwd.cu's rf_step_sums reads and b2d_rf_backward_workspace_bytes sizes.
#pragma once
constexpr int kTokenSlab = 32;
