/*
 * ngp_b200.h -- C ABI of libngp_b200.so: the H100-native (sm_90a) Instant-NGP inner loop behind
 * JNeRF's operator boundary.
 *
 * Every entry point is what a `jt.code(...)` body of the reference would call in place of its inline
 * kernel launches (see INTEGRATION.md for the Jittor-side stubs).  Conventions, mirroring the reference
 * (SURVEY.md section 8b):
 *   - all pointers are DEVICE pointers owned by the caller (the reference's ops never allocate:
 *     HE/grid_encode.py:55-61, OPS/fully_fused_mlp.py:83); 16-byte aligned;
 *   - `stream` is a cudaStream_t passed as void* (the reference hard-codes stream 0, e.g.
 *     HE/grid_encode.py:77, DGS/ray_sampler.py:49); the library is re-entrant per stream;
 *   - the process-global `jittor::rng` (OPS/global_vars.py:5-27) becomes an explicit (state, inc) pair;
 *   - every function returns 0 on success, non-zero on error; ngp_last_error() gives the message
 *     (the reference throws std::runtime_error from host code or leaves launches unchecked);
 *   - dtype: 0 = float32, 1 = float16 (the reference's `grad_t` / `in0_type`).
 * Paths in comments are relative to python/jnerf/ of the JNeRF reference:
 *   HE = models/position_encoders/hash_encoder, SH = models/position_encoders/sh_encoder,
 *   DGS = models/samplers/density_grid_sampler, OPS = ops/code_ops.
 */
#ifndef NGP_B200_H
#define NGP_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define NGP_F32 0
#define NGP_F16 1
#define NGP_N_LEVELS 16        /* HE/hash_encoder.py:17-18 hard-codes L=16, F=2, base 16 */
#define NGP_LEVEL_BYTES 32

const char* ngp_last_error(void);
int ngp_version(void);
/* number of SMs of the current device (grid sizing of the persistent kernels) */
int ngp_sm_count(void);
/* debug aid: 1 if a tensor-core pipeline wait timed out since the last call (synchronises the device) */
int ngp_debug_timeout_flag(void);

/* ---- R1  level table ------------------------------------------------------------------------------
 * HE/grid_encode.py:17-39: per-level offsets (host, doubles).  offsets_out has n_levels+1 entries. */
int ngp_hash_offsets(double aabb_scale, int n_levels, int base_resolution, int log2_hashmap_size,
                     uint32_t* offsets_out_host, double* per_level_scale_out);
/* Device-side per-level record {scale, resolution, offset, size, hashed}: evaluates the reference kernel's own
 * expression exp2f(level*log2_pls)*base-1 (HE/op_header/HashEncode.h:149-151) once, on the device.
 * levels_dev: NGP_N_LEVELS * NGP_LEVEL_BYTES bytes. */
int ngp_hash_level_table(void* stream, const uint32_t* offsets_host, int n_levels, uint32_t base_resolution,
                         float log2_per_level_scale, void* levels_dev);
/* the same with the three multipliers of cfg.hash_func, get_index(p0,p1,p2) = p0*prime0 ^ p1*prime1 ^ p2*prime2
 * (HE/hash_encoder.py:13-16 pastes the config string into the kernel source; the configs use 1, 19349663, 83492791) */
int ngp_hash_level_table_primes(void* stream, const uint32_t* offsets_host, int n_levels, uint32_t base_resolution,
                                float log2_per_level_scale, void* levels_dev, uint32_t prime0, uint32_t prime1, uint32_t prime2);

/* ---- R2/R3  hash-grid encode -------------------------------------------------------------------------
 * Replaces extract_position + kernel_grid + transpose_encoded_position (HashEncode.h:36-50,117-252,254-268;
 * call site HE/grid_encode.py:66-129).  x (n,3) f32 in [0,1]; grid [level][entry][2] of dtype; out (n,32). */
int ngp_hash_fwd(void* stream, uint32_t n, const float* x, const void* grid, int dtype, const void* levels_dev, void* out);
/* Replaces transpose_gradients + cudaMemsetAsync + kernel_grid_backward (HashEncode.h:270-284,299-396;
 * HE/grid_encode.py:131-190).  grid_grad (n_params of dtype) is zeroed here, as the reference does (:153). */
int ngp_hash_bwd(void* stream, uint32_t n, const float* x, const void* dy, int dtype, const void* levels_dev,
                 void* grid_grad, uint64_t n_params);

/* ---- R4  spherical harmonics, degree 4 (SH/op_header/SphericalEncode.h:44-150; SH/sh_encoder.py:26-53) ---- */
int ngp_sh_fwd(void* stream, uint32_t n, const float* dirs, int dtype, void* out);

/* ---- R7  fully-fused MLP (wgmma) ---------------------------------------------------------------------
 * Replaces mlp_fused_forward_func / mlp_fused_backward_func + the cuBLAS wgrad chain
 * (OPS/op_header/fully_fused_mlp_header.h:26-60; OPS/fully_fused_mlp.py:58-75,101-143).
 * WIDTH 64, input 32, output padded to 16, ReLU hidden, no output activation, no bias, fp16.
 * weights: flat [W0 (64x32) | Wh (64x64) x n_hidden_matmuls | Wout (16x64)], each (out,in) row-major
 *          (OPS/fully_fused_mlp.py:26-40).
 * inter:   ((n_hidden_matmuls+1)*n, 64) post-ReLU activations, block k = hidden layer k; may be NULL.
 * n need not be a multiple of 128 (the reference pads, :78-82; here rows are masked). */
int ngp_mlp_fwd(void* stream, const void* weights, const void* input, void* inter, void* output,
                uint32_t n_hidden_matmuls, uint32_t n);
/* dY (n,16) ROW-major.  dX (n,32) and temps ((n_hidden_matmuls+1)*n,64; block j = gradient at hidden layer
 * n_hidden_matmuls-j, the reference's reverse order, fully_fused_mlp.py:127-142) may be NULL.
 * dW: fp32, same flat layout as weights, OVERWRITTEN; rows >= n_out_valid of the last layer are zero (:136). */
int ngp_mlp_bwd(void* stream, const void* weights, const void* input, const void* inter, const void* dY,
                void* dX, void* temps, float* dW, uint32_t n_hidden_matmuls, uint32_t n_out_valid, uint32_t n);
/* Data-gradient chain only -- what the reference's link-level mlp_fused_backward_func returns (fully_fused_mlp_header.h:29-43;
 * call site OPS/fully_fused_mlp.py:101-115): dY_feature_major is (16,n) (the reference passes grads.transpose(), :117), temps
 * as above, dX (n,32) optional; no weight gradients (the reference leaves those to five cuBLAS GEMMs, :123-143). */
int ngp_mlp_bwd_dgrad(void* stream, const void* weights, const void* inter, const void* dY_feature_major, void* dX, void* temps,
                      uint32_t n_hidden_matmuls, uint32_t n);
int ngp_mlp_param_count(uint32_t n_hidden_matmuls);
/* The two C++ symbols of the reference's prebuilt fully_fused_mlp_function.o (mlp_fused_forward_func / mlp_fused_backward_func,
 * OPS/op_header/fully_fused_mlp_header.h:26-60) are exported too, with their original mangled names, by csrc/compat_tcnn.cu:
 * OPS/fully_fused_mlp.py links against libngp_b200.so unchanged (INTEGRATION.md section 3). */

/* ---- R7+R2+R4 fused: NGPNetworks.execute (models/networks/ngp_network.py:77-84) -----------------------
 * coords (n_max,7) f32 = NerfCoordinate {pos[3], dt, dir[3]} (DGS/op_header/ray_sampler_header.h:548-574).
 * n_dev: optional device uint32 with the live row count (rows beyond it are skipped, no host sync); NULL = n_max.
 * out (n_max,4) fp16 = {rgb, sigma_raw}; enc_save (n_max,32) fp16 (kept for backward) may be NULL.
 * Rows at or past the live count are not written, except that a 16-byte-aligned enc_save may also have the rows of the last live
 * 128-row tile written up to the tile's end or n_max (they are stored by TMA, one whole tile at a time). */
int ngp_network_fwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* grid,
                    const void* levels_dev, const void* w_density, const void* w_rgb, void* out, void* enc_save);
/* Backward of the above: dout (n_max,4) fp16 -> grid_grad (fp16, ACCUMULATED: caller zeroes),
 * dw_density / dw_rgb (fp32, ACCUMULATED: caller zeroes).  Recomputes the MLP forward from enc_save.
 * Deterministic (the result does not depend on how the GPU schedules the work), except for a call captured in a CUDA graph on a
 * stream that has not run an uncaptured call with this level table before (that one reduces with order-dependent rounding), and for
 * the entries of a level table that grew in place past the table the stream saw first. */
int ngp_network_bwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* enc_save,
                    const void* levels_dev, const void* w_density, const void* w_rgb, const void* dout,
                    void* grid_grad, float* dw_density, float* dw_rgb);
/* The same backward into caller-owned scratch, for ngp_train_sweep: the hash-grid gradient ACCUMULATES into fx, 16 bytes per table
 * entry (two signed 64-bit fixed-point sums in units of 2^-32, all zero before the first call: ngp_train_sweep clears what it reads),
 * and every CTA STORES its weight-gradient sums into its slot of w_part.  Nothing is reduced, rounded, allocated or read back, so the
 * call is deterministic inside CUDA-graph capture too.  n_entries is the level table's entry count (offset + size of its last
 * level); buffers smaller than ngp_network_bwd_fx_bytes(n_entries) gives are refused. */
int ngp_network_bwd_fx_bytes(uint64_t n_entries, uint64_t* fx_bytes, uint64_t* part_bytes);
int ngp_network_bwd_fx(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* enc_save,
                       const void* levels_dev, const void* w_density, const void* w_rgb, const void* dout, uint32_t n_entries,
                       void* fx, uint64_t fx_bytes, float* w_part, uint64_t part_bytes);
/* NGPNetworks.density (ngp_network.py:86-89): pos (n,3) f32 -> sigma_raw (n) fp16 */
int ngp_density_fwd(void* stream, uint32_t n, const float* pos, const void* grid, const void* levels_dev,
                    const void* w_density, void* sigma_out);
/* The gradient of sigma_raw (the density MLP's first output, before exp) with respect to the position row[0:3] of NerfCoordinate rows
 * coords (n_max,7) f32 -> grad_out (n_max,3) f32, for normal maps (V6).  The reference has no counterpart (it differentiates the density
 * only with respect to the table and the weights).  Per row, sum over levels of J_l^T dsigma/denc_l: J_l the 2x3 derivative of level l's
 * trilinear interpolation, dsigma/denc = W0d^T (relu'(hd) .* Woutd[0, :]), with the ReLU mask of the forward's own fp16 density layer 0
 * (hd is formed as ngp_network_fwd forms it, bit for bit) and everything else in fp32.  Hashed and dense levels alike.  n_dev as for
 * ngp_network_fwd: rows at or past it are not written.  A NULL coords, grid, levels, w_density or grad_out with n_max > 0 is an error. */
int ngp_density_grad(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* grid, const void* levels_dev,
                     const void* w_density, float* grad_out);

/* ---- F1-F4  vanilla NeRF: FrequencyEncoder + OriginNeRFNetworks (position_encoders/freq_encoder/freq_encoder.py:22-50,
 * models/networks/ori_nerf_network.py:10-70), csrc/nerf_mlp.cu, DESIGN.md section 10 ---------------------------------------------
 * params: ONE flat fp16 vector of *count_out (ngp_nerf_param_count) entries, 16-byte aligned, in the kernels' padded layout (DESIGN.md
 * section 10; jnerf_b200/plugin/nerf.py maps it to the reference's parameter names).
 * F1: the sizes of the forward's saved activations and of the backward's scratch for n_max rows (~5 KB a row each). */
int ngp_nerf_param_count(uint64_t* count_out);
int ngp_nerf_workspace_bytes(uint32_t n_max, uint64_t* saved_bytes, uint64_t* scratch_bytes);
/* F2: OriginNeRFNetworks.execute (ori_nerf_network.py:34-56) on NerfCoordinate rows coords (n_max,7) f32: pos = row[0:3],
 * dir = row[4:7] -> out (n_max,4) fp16 {rgb, alpha}, the layout the composite kernels read.  n_dev as for ngp_network_fwd: rows at
 * or past it are not written.  saved (may be NULL): every layer's input, what ngp_nerf_bwd reads. */
int ngp_nerf_fwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const float* coords, const void* params, void* out, void* saved);
/* F3: OriginNeRFNetworks.density (ori_nerf_network.py:58-67): pos (n,3) f32 -> alpha (n) fp16, bit for bit column 3 of ngp_nerf_fwd */
int ngp_nerf_density(void* stream, uint32_t n, const float* pos, const void* params, void* sigma_out);
/* F4: backward of F2 from dout (n_max,4) fp16 and F2's saved activations -> grad (one fp32 per parameter, OVERWRITTEN) of every
 * weight and bias.  No gradient into the encoding or the coordinates.  Deterministic: no float atomics, sums in a fixed order. */
int ngp_nerf_bwd(void* stream, uint32_t n_max, const uint32_t* n_dev, const void* params, const void* saved, const void* dout, void* scratch,
                 float* grad);

/* ---- P1-P13  Mip-NeRF (contrib/mipnerf of the reference: models/samplers/mip_sampler/mip_sampler.py, utils/miputils.py,
 * models/networks/mip_network.py, dataset/nerf_datasets.py:22-235, dataset/nerf.py), csrc/mip_sampler.cu + csrc/mip_mlp.cu +
 * csrc/mip_multiscale.cu + csrc/mip_mlp_wide.cu, DESIGN.md section 11 --------------------------------------------------------------------------------------------
 * A ray row is 12 floats: origin[3], direction[3] (unnormalised), viewdir[3], base radius, near, far.  t holds S + 1 fenceposts a ray
 * (S = n_samples <= 128 for the per-ray kernels).  Network rows are (ray, interval) pairs, row r = interval r % S of ray r / S.  The
 * kernels that draw uniforms give ray g the pcg32 draws [g (S + 1), (g + 1)(S + 1)) of the stream at (rng_state, rng_inc), in fencepost
 * order; the caller advances its stream by n_rays (S + 1) after such a call.  ray_shape: 0 cone, 1 cylinder.
 * P1: rays and targets of pixels pix (img * H + y) * W + x: c2w (n_img, 12) row-major 3x4 NeRF camera-to-world, images_rgba
 * (n_img * H * W, 4) uint8, target = rgb / 255 (n, 3).  Bit for bit the reference's fp32 numpy ray generation. */
int ngp_mip_rays(void* stream, uint32_t n, const uint32_t* pix, uint32_t W, uint32_t H, const float* c2w, float focal, float near, float far,
                 const uint8_t* images_rgba, float* rays_out, float* target_out);
/* P2: sample_along_rays (miputils.py:324-362): t_out (n_rays, S + 1), linear in depth or in disparity, jittered when randomized. */
int ngp_mip_sample(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, int lindisp, int randomized, uint64_t rng_state,
                   uint64_t rng_inc, float* t_out);
/* P3: resample_along_rays (:365-408): blur-pool of weights (n_rays, S) + resample_padding, inverse-CDF sampling of S + 1 sorted new
 * fenceposts within [t_0, t_S] into t_out (not aliasing t). */
int ngp_mip_resample(void* stream, uint32_t n_rays, uint32_t n_samples, const float* t, const float* weights, float resample_padding,
                     int randomized, uint64_t rng_state, uint64_t rng_inc, float* t_out);
/* P4: cast_rays + integrated_pos_enc of degrees [min_deg, min_deg + 8) (:215-275) -> enc_out (N, 48), and pos_enc(viewdir, 0, 4)
 * (:120-127) -> view_out (N, 27), fp32, the reference's column orders; integrate = 0 is disable_integration.  N = n_rays * S. */
int ngp_mip_encode(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate, int min_deg,
                   float* enc_out, float* view_out);
/* P5: MipNerfMLP.execute on the fused kernels of F1-F4: the encodings of P4 computed on chip, params in the layout of
 * ngp_nerf_param_count (jnerf_b200/plugin/mip.py maps it to the reference's names), out (N, 4) fp16 {raw rgb, raw density}; saved (may
 * be NULL, ngp_nerf_workspace_bytes(N) bytes) is what ngp_nerf_bwd reads.  Two calls whose rows are multiples of 128 may save into
 * consecutive parts of one buffer and share one ngp_nerf_bwd. */
int ngp_mip_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate, int min_deg,
                const void* params, void* out, void* saved);
/* P6: rays2rgb + volumetric_rendering (mip_sampler.py:83-96, miputils.py:278-321) of raw (n_rays * S, 4) of dtype: rgb (n_rays, 3), acc,
 * distance (clipped to [t_0, t_S]; t_0 where acc = 0) and, unless NULL, the weights (n_rays, S). */
int ngp_mip_composite_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, int dtype, const float* t, const float* rays,
                          float rgb_padding, float density_bias, int white_bkgd, float* rgb_out, float* acc_out, float* distance_out,
                          float* weights_out);
/* P7: the training loss of both levels (runner.py:83-92) and its backward in one launch: raw (2 n_rays * S, 4) and t (2 n_rays, S + 1)
 * hold the coarse level, then the fine level, of the n_rays rays.  loss = coarse_loss_mult L_coarse + L_fine with
 * L = sum_r mask_r |rgb_r - target_r|^2 / sum_r mask_r (mask NULL: all ones).  rgb_out (2 n_rays, 3), loss_out (2 n_rays) the per-ray
 * terms of that sum, draw_out (2 n_rays * S, 4) of dtype = grad_scale * dloss / draw. */
int ngp_mip_composite_loss_bwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, int dtype, const float* t, const float* rays,
                               const float* target, const float* mask, float rgb_padding, float density_bias, int white_bkgd, float coarse_loss_mult,
                               float grad_scale, float* rgb_out, float* loss_out, void* draw_out);
/* P8: rays, targets and loss weights of the multiscale datasets (dataset/nerf.py: Blenders :207-314, Multicam :108-204), csrc/mip_multiscale.cu.
 * n_images images of different sizes: global pixel p of image i is offsets[i] + y W_i + x (offsets (n_images + 1) ascending, wh (n_images, 2)
 * = {W_i, H_i} with H_i >= 3); cams (n_images, 24) = {pix2cam 3x3, cam2world 3x4 (both row-major), lossmult, near, far}; images_rgba
 * (offsets[n_images], 4), uint8 (read as v / 255) or, with float_images, fp32.  focal != 0: the directions of P1's camera model with that
 * focal length (Blenders); focal = 0: (x + .5, y + .5, 1) @ pix2cam^T @ cam2world[:3, :3]^T (Multicam).  rays_out (n, 12), target_out
 * (n, 3) = rgb a + (1 - a) with white_bkgd, else rgb; lossmult_out (n). */
int ngp_mip_rays_multi(void* stream, uint32_t n, const uint32_t* pix, uint32_t n_images, const uint32_t* offsets, const uint32_t* wh,
                       const float* cams, float focal, int white_bkgd, const void* images_rgba, int float_images, float* rays_out, float* target_out,
                       float* lossmult_out);
/* P10-P13: MipNerfMLP's fused network at degs = 8 or 16 IPE degrees (max_deg_point - min_deg_point), csrc/mip_mlp_wide.cu.  degs = 8 is
 * P5 + F4 (ngp_nerf_*) unchanged.  degs = 16: kernel layer 0 reads 96 columns, the skip layer 352 (the 96 encoding columns, then h4),
 * ngp_mip_param_count gives 618 912 fp16 parameters; saved (ngp_mip_workspace_bytes' first size) holds 320 groups of 8 halfs a row.  As
 * with P5, two forwards whose rows are multiples of 128 may save into consecutive parts of one buffer and share one ngp_mip_bwd_deg,
 * which writes the fp32 gradient of the flat parameters into grad, deterministically. */
int ngp_mip_param_count(int degs, uint64_t* count_out);
int ngp_mip_workspace_bytes(int degs, uint32_t n_max, uint64_t* saved_bytes, uint64_t* scratch_bytes);
int ngp_mip_fwd_deg(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate,
                    int min_deg, int degs, const void* params, void* out, void* saved);
int ngp_mip_bwd_deg(void* stream, uint32_t n_max, int degs, const void* params, const void* saved, const void* dout, void* scratch, float* grad);
/* P9: P4 at degs = 8 or 16 IPE degrees: enc_out (N, 6 degs), view_out (N, 27).  Equal to P4 bit for bit at degs = 8. */
int ngp_mip_encode_deg(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* t, int ray_shape, int integrate,
                       int min_deg, int degs, float* enc_out, float* view_out);

/* ---- N1-N5  pixelNeRF (contrib/pixelnerf of the reference), csrc/pixelnerf.cu, DESIGN.md section 13 -----------------------------------------
 * rays (n_rays, 6) fp32 origin then direction (not normalised); z (n_samples) the sample depths shared by every ray (Render.py:22-26).
 * params: ngp_pixelnerf_param_count fp16 values in the layout of plugin/pixelnerf.py (mlp.0 padded to 64 input columns).
 * feats (n_ref, feat_h, feat_w, 512) fp16 channel-last; cams (n_ref, 12) fp32: R_t = c2w[:3,:3]^T row-major, then the camera position;
 * scale = (H / 2) / focal.  raw (n_rays n_samples, 4) fp16: relu(o0), sigmoid(o1:4). */
int ngp_pixelnerf_param_count(uint64_t* count_out);
/* N1: buffer sizes for n_rows = n_rays n_samples sample rows: saved (training forward), infer (forward with saved NULL), bwd (backward scratch). */
int ngp_pixelnerf_workspace_bytes(uint32_t n_ref, uint32_t n_rows, uint64_t* saved_bytes, uint64_t* infer_bytes, uint64_t* bwd_bytes);
/* N2: Render.py:10-15 + Dataset.py:86-94 + Network.py:66-94: projection, feature gather, network.  saved non-NULL: the training forward,
 * keeping what ngp_pixelnerf_bwd reads; saved NULL: inference, temporaries in scratch.  raw is the same bit for bit either way.
 * pixel_aligned = 0 is the reference's projection (uv = p.xy / p.z / scale, v negated), 1 the pinhole one (both negated, then v). */
int ngp_pixelnerf_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const float* rays, const float* z, const void* params, const void* feats,
                      uint32_t n_ref, uint32_t feat_h, uint32_t feat_w, const float* cams, float scale, int pixel_aligned, void* raw_out, void* saved,
                      void* scratch);
/* N3: the backward of N2 from draw (like raw) into grad (param_count fp32, overwritten), deterministic.  Replaces main.py:46's
 * optimizer.step(loss) gradient. */
int ngp_pixelnerf_bwd(void* stream, uint32_t n_rays, uint32_t n_samples, uint32_t n_ref, const void* params, const void* feats, const void* saved,
                      const void* raw, const void* draw, void* scratch, float* grad);
/* N4: Render.py:16-18 + :34-46: rgb (n_rays, 3), depth, acc (n_rays, may be NULL); n_samples <= 64. */
int ngp_pixelnerf_composite_fwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, const float* z, const float* rays, float* rgb_out,
                                float* depth_out, float* acc_out);
/* N5: N4, main.py:45's MSE over the 3 n_rays colour entries (loss_out: per-ray terms that sum to it) and draw_out = grad_scale dloss / draw
 * in fp16, saturated to +-65504. */
int ngp_pixelnerf_composite_loss_bwd(void* stream, uint32_t n_rays, uint32_t n_samples, const void* raw, const float* z, const float* rays,
                                     const float* target, float grad_scale, float* rgb_out, float* loss_out, void* draw_out);

/* ---- X1-X9  Plenoxels (contrib/plenoxel of the reference: models/networks/svox2_network.py, ops/svox_ops/op/op_header/*.h),
 * csrc/svox.cu, DESIGN.md section 12 ----------------------------------------------------------------------------------------------
 * A grid is links (X, Y, Z) int32 row-major (< 0: empty), density (capacity) and sh (capacity, 27) fp32, SH degree 2 channel-major.
 * xform (host, 6 floats): offset[3], scaling[3] from world to grid coordinates (_offset * reso - 0.5, _scaling * reso).  opts (host, 4
 * floats): step_size, sigma_thresh, stop_thresh, background_brightness.  Cameras: c2w row-major 3x4 OpenCV camera-to-world, pixel
 * (img * H + y) * W + x, ray through the pixel centre.  Gradients are signed 64-bit fixed point, 2^48 units per 1.0, added with integer
 * atomics (order-independent); a term or sum out of range ORs 1 into *flag (device), which stays set until the caller clears it.
 * X1: one training step of n_rays pixels: forward, dL/drgb = 2 (rgb - gt) / (3 n_rays) with gt the RGBA image composited on white,
 * the backward into grad_density / grad_sh (added to), and the per-ray squared error sqerr_out (n_rays). */
int ngp_svox_train_step(void* stream, uint32_t n_rays, const int32_t* pix, uint32_t W, uint32_t H, const float* c2w, float fx, float fy, float cx,
                        float cy, const uint8_t* images_rgba, const int32_t* links, int X, int Y, int Z, const float* density, const float* sh,
                        const float* xform, const float* opts, long long* grad_density, long long* grad_sh, float* sqerr_out, unsigned* flag);
/* X2: rgb_out (n, 3) of pixels [first, first + n) (row-major y * W + x) of one camera c2w (12 floats). */
int ngp_svox_render(void* stream, uint32_t n, uint32_t first, uint32_t W, const float* c2w, float fx, float fy, float cx, float cy, const int32_t* links,
                    int X, int Y, int Z, const float* density, const float* sh, const float* xform, const float* opts, float* rgb_out);
/* X3: sparse TV of columns [0, dim) of data (capacity, dim) over the cells (start + i) mod (X Y Z), i < n_cells, added into grad
 * (loss_kernel.h:51-118; scale is lambda / n_cells). */
int ngp_svox_tv_grad(void* stream, const int32_t* links, int X, int Y, int Z, const float* data, uint32_t dim, uint32_t start, uint32_t n_cells,
                     float scale, int ignore_edge, long long* grad, unsigned* flag);
/* X4: RMSprop over density (n_density) and sh (n_sh entries): v = a v + (1 - a) g^2, p -= lr g / (sqrt(v) + eps) with g the
 * fixed-point gradient, which is set to 0. */
int ngp_svox_rmsprop(void* stream, uint64_t n_density, uint64_t n_sh, float* density, float* sh, long long* grad_density, long long* grad_sh,
                     float* rms_density, float* rms_sh, float lr_density, float lr_sh, float alpha_density, float alpha_sh, float eps);
/* X5: trilerp of density (and, want_sh, of the 27 SH columns) at n points (n, 3) given in grid coordinates. */
int ngp_svox_sample(void* stream, uint32_t n, const float* points, const int32_t* links, int X, int Y, int Z, const float* density, const float* sh,
                    int want_sh, float* density_out, float* sh_out);
/* X6: max over the rays of one camera (W x H) of each sample's weight, onto the 8 corners of its cell of the dense grid data (X, Y, Z):
 * weight_out (X, Y, Z) is max-ed into. */
int ngp_svox_weight_render(void* stream, uint32_t W, uint32_t H, const float* c2w, float fx, float fy, float cx, float cy, const float* data, int X, int Y,
                           int Z, const float* xform, float step_size, float stop_thresh, float* weight_out);
/* X7: out = the 26-neighbourhood dilation of mask (X, Y, Z) uint8. */
int ngp_svox_dilate(void* stream, int X, int Y, int Z, const uint8_t* mask, uint8_t* out);
/* X8: bytes of the workspace of X9. */
int ngp_svox_compact_workspace_bytes(int X, int Y, int Z, uint64_t* bytes_out);
/* X9: links_out (X, Y, Z) = the exclusive count of kept cells before each kept cell, -1 elsewhere; kept cell c gets density_out[c] =
 * dense_density of the cell and points_out[c] = lattice[0:3] + (x, y, z) * lattice[3:6] (host lattice).  capacity = number of kept
 * cells. */
int ngp_svox_compact(void* stream, int X, int Y, int Z, const uint8_t* mask, const float* dense_density, const float* lattice, uint32_t capacity,
                     void* workspace, int32_t* links_out, float* density_out, float* points_out);

/* ---- M1-M4  mesh extraction (tools/extract_mesh.py of the reference: a trained model -> mesh-origin.ply / mesh-color.ply) --------
 * Resolution n must be in [2, 1024]; vertices are (V,3) f32, triangles (T,3) int32 (V, T < 2^31); counts are 64-bit.
 * workspace: *bytes_out of ngp_mesh_workspace_bytes(n, 0, 0, .) for ngp_marching_cubes, of (0, V, T, .) for the other two.
 * Every result is bit-reproducible (fixed numbering, fixed summation order; DESIGN.md section 4 "Mesh extraction"). */
int ngp_mesh_workspace_bytes(uint32_t n, uint64_t n_verts, uint64_t n_tris, uint64_t* bytes_out);
/* M1: the n^3 density lattice of extract_mesh.py:42-70 -- row (i*n + j)*n + k at model position (i, j, k)/(n-1) (the unit cube, not the
 * aabb), field_out[row] = float(int(max(sigma_raw, 0))) (:68).  Positions are made in the kernel (no coordinate buffer); sigma_raw is
 * bit-identical to ngp_density_fwd at the same positions. */
int ngp_density_lattice(void* stream, uint32_t n, const void* grid, const void* levels_dev, const void* w_density, float* field_out);
/* M1 on vanilla NeRF (extract_mesh.py:42-70 querying OriginNeRFNetworks, ori_nerf_network.py:58-67), csrc/nerf_lattice.cu: the same rows
 * and positions, field_out[row] = float(int(max(alpha_raw, 0))) with alpha_raw bit-identical to ngp_nerf_density at the same position.
 * params: the flat fp16 vector of ngp_nerf_fwd, 16-byte aligned.  Positions are made in the kernel (no coordinate buffer). */
int ngp_nerf_density_lattice(void* stream, uint32_t n, const void* params, float* field_out);
/* M2: mcubes.marching_cubes(sigma, iso) + the vertex frame of :78-84 (lattice position / n, first two columns swapped).  A vertex per
 * lattice edge whose endpoints straddle iso (inside: value > iso), numbered in lattice-edge order; triangles in cell order, their
 * right-hand normals pointing towards lower values in the written frame.  counts_host[0..1] = vertices, triangles, read back once.
 * verts = tris = NULL: count only (call again with buffers of at least those sizes). */
int ngp_marching_cubes(void* stream, uint32_t n, const float* field, float iso, void* workspace, float* verts, uint64_t max_verts,
                       int32_t* tris, uint64_t max_tris, uint64_t* counts_host);
/* M3: Open3D cluster_connected_triangles + argmax + remove_triangles_by_index + remove_unreferenced_vertices (:92-97): the largest set of
 * triangles joined through shared edges (a tie keeps the set holding the lowest triangle), triangles and vertices compacted in order.
 * verts_out (n_verts,3) / tris_out (n_tris,3) capacities; counts_host[0..1] = kept vertices, kept triangles (synchronises). */
int ngp_mesh_largest_component(void* stream, uint64_t n_verts, uint64_t n_tris, const float* verts, const int32_t* tris, void* workspace,
                               float* verts_out, int32_t* tris_out, uint64_t* counts_host);
/* M4: Open3D compute_vertex_normals (:106): per vertex the sum of its triangles' (v1-v0)x(v2-v0) in triangle order, normalised (a zero
 * sum stays zero).  normals (n_verts,3). */
int ngp_mesh_vertex_normals(void* stream, uint64_t n_verts, uint64_t n_tris, const float* verts, const int32_t* tris, void* workspace,
                            float* normals);
/* M5/M6: mcubes.smooth(sigma) of --mcube_smooth (:27-31, 74-78), to be marched at iso 0 (DESIGN.md section 7 states the contract).
 * method: 0 auto (constrained for n <= 512, gaussian above), 1 constrained (signed distance from an exact EDT, then a bounded fp64 Jacobi
 * solve on the band |D| < 4, at most max_iters iterations, stopping early on the energy test every 10), 2 gaussian (sigma 3 of
 * field - 0.5 in fp64, mode 'reflect'; max_iters is ignored).  max_iters = 0 with the constrained method gives D itself.
 * field and field_out are separate n^3 fp32 lattices.  info_host[0..2] = method used, iterations run, band variables (the constrained
 * method reads them back once and synchronises; the gaussian one does not synchronise).  Bit-reproducible.
 * M5 workspace, each part rounded up to 256 bytes: constrained 8 n^3 (two int32 lattices) + 4 ceil(n^3 / 2048) + 24 + 8 * 1024
 *   + 64 n^3 (neighbour table, x, Qx and bound of up to n^3 band variables), about 9.7 GB at n = 512; gaussian 8 n^3 (one fp64 lattice). */
int ngp_mesh_smooth_workspace_bytes(uint32_t n, uint32_t method, uint64_t* bytes_out);
int ngp_mesh_smooth(void* stream, uint32_t n, const float* field, uint32_t method, uint32_t max_iters, void* workspace,
                    uint64_t workspace_bytes, float* field_out, uint32_t* info_host);

/* ---- R6  ray march (DGS/ray_sampler.py:20-72 -> DGS/op_header/ray_sampler.h:4-114) -------------------
 * counters[0] = rays accepted, counters[1] = total samples (both zeroed here, ray_sampler.py:29).
 * numsteps (R,2) = {count, base}; base is the exclusive prefix sum in RAY ORDER (deterministic; the reference
 * uses atomicAdd order).  coords (max_samples,7) rows [0,total) are written; nothing is memset (the reference
 * clears 117 MB per call, ray_sampler.py:50).  const_dt selects the generated calc_dt
 * (DGS/density_grid_sampler.py:107-115).  workspace: ngp_march_workspace_bytes(n_rays). */
uint64_t ngp_march_workspace_bytes(uint32_t n_rays);
int ngp_march(void* stream, uint32_t n_rays, float aabb_lo, float aabb_hi, uint32_t max_samples, const float* rays_o,
              const float* rays_d, const uint8_t* bitfield, float cone_angle, float near_distance, uint32_t cascades,
              int const_dt, uint64_t rng_state, uint64_t rng_inc, uint32_t* counters, uint32_t* ray_indices,
              uint32_t* numsteps, float* coords, void* workspace);
/* R5 compaction (DGS/compacted_coord.py:28-70 -> compacted_coord.h:4-76): per-ray copy into a buffer of
 * max_compacted rows with truncation; rows [min(total,max), max_compacted) are zero-filled like the reference's
 * jt.zeros (compacted_coord.py:39).  counters[0] = samples, counters[1] = rays with >0 samples. */
int ngp_compact(void* stream, uint32_t n_rays, uint32_t max_compacted, const float* coords_in, const uint32_t* numsteps_in,
                float* coords_out, uint32_t* numsteps_out, uint32_t* counters, int zero_fill);

/* ---- R8/R9  volume-render composite (DGS/calc_rgb.py -> DGS/op_header/calc_rgb.h) ---------------------- */
int ngp_composite_fwd(void* stream, uint32_t n_rays, const void* net_out, int dtype, const float* coords,
                      const uint32_t* numsteps_in, const uint32_t* numsteps_compacted, const float* bg, uint32_t cascades,
                      float* rgb_out);
int ngp_composite_bwd(void* stream, uint32_t n_rays, uint32_t n_elements, const void* net_out, int dtype, const float* coords,
                      const uint32_t* numsteps_compacted, const float* loss_grad, const float* rgb_ray,
                      const float* density_grid_mean, uint32_t cascades, void* dnet_out);
int ngp_composite_infer(void* stream, uint32_t n_rays, const void* net_out, int dtype, const float* coords,
                        const uint32_t* numsteps, uint32_t cascades, float* rgb_out, float* alpha_out);
/* Fused training tail: composite fwd (calc_rgb.h:10-74) + Huber(delta) gradient (models/losses/huber_loss.py:11-14)
 * + composite bwd (calc_rgb.h:76-148) in one pass per ray; also returns rgb and the per-ray summed loss.
 * reg_scale multiplies the density regulariser of calc_rgb.h:112,139 (1 on one GPU; the world size under data parallelism, where
 * the summed shard gradients are scaled by 1 / world but the regulariser is an absolute per-sample term). */
int ngp_composite_loss_bwd(void* stream, uint32_t n_rays, uint32_t n_elements, const void* net_out, const float* coords,
                           const uint32_t* numsteps_in, const uint32_t* numsteps_compacted, const float* bg,
                           const float* target, float huber_delta, const float* density_grid_mean, uint32_t cascades,
                           float* rgb_out, float* loss_out, void* dnet_out, float reg_scale);

/* ---- V1-V6  whole-frame renderer with early ray termination (runner/runner.py:197-264: render_img / render_img_with_pose) ------------
 * Stands in for the tiled inference path of the reference -- ray_sampler.h per n_rays_per_batch tile, the network, then
 * compute_rgbs_inference (calc_rgb.h:151-212) over every sample -- with a wavefront loop over rounds that drops a ray once it is opaque
 * (DESIGN.md section 4, "Rendering").  Per ray: rgb without background, alpha = 1 - T, and the number of composited samples.
 * One call sequence: ngp_render_init, then per round ngp_render_march_round -> ngp_network_fwd over the round's rows ->
 * ngp_render_composite_round, until the alive count is 0.  With min_transmittance = 0 every ray composites exactly the samples
 * ngp_march gives it; the outputs do not depend on k_steps or the capacity.  Capacity 0, a NULL workspace and jitter_tile 0 are errors.
 * V1: layout_out[0..3] = workspace bytes, then the byte offsets inside it of the round's rows ((capacity,7) f32 NerfCoordinate),
 * of the network outputs for them ((capacity,4) fp16) and of the device uint32 round row count (the n_dev of ngp_network_fwd). */
int ngp_render_workspace_bytes(uint32_t n_rays, uint32_t capacity, uint64_t* layout_out);
/* V2: slab test, near distance and jitter (ray_sampler.h:29-48).  Ray g jitters with the state advanced by
 * (g / jitter_tile) * 2^32 + (g % jitter_tile) * 8: what ngp_march draws when the rays are marched jitter_tile at a time with one
 * rng.advance() between tiles (the caller advances its state by ceil(n_rays / jitter_tile) * 2^32 afterwards).  Rays that miss the box
 * finish with rgb 0, alpha 0, 0 samples.  Zeroes the outputs, builds the alive list; *n_alive_host = its length (synchronises). */
int ngp_render_init(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, float aabb_lo, float aabb_hi, const float* rays_o,
                    const float* rays_d, float cone_angle, float near_distance, uint32_t cascades, int const_dt, uint64_t rng_state,
                    uint64_t rng_inc, uint32_t jitter_tile, float* rgb_out, float* alpha_out, uint32_t* n_samples_out, uint32_t* n_alive_host);
/* V3: each of the first min(n_alive, capacity / k_steps) alive rays continues the march of ray_sampler.h:50-72 from its saved state for
 * up to k_steps samples (a ray ends after 2^20 steps of its t sequence, occupied or skipped, as in ngp_march); their NerfCoordinate rows go to the workspace, dense in ray order, and their total to the device row count. */
int ngp_render_march_round(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, uint32_t n_alive, uint32_t k_steps, float aabb_lo,
                           float aabb_hi, const float* rays_o, const float* rays_d, const uint8_t* bitfield, float cone_angle, uint32_t cascades,
                           int const_dt);
/* V4: each marched ray composites its rows in order (calc_rgb.h:151-212 per sample); it stops after the first sample that brings T below
 * min_transmittance, or when its march has ended (fewer than k_steps samples this round).  Same n_alive / k_steps as V3.  The other rays
 * form the next alive list (order kept); *n_alive_host = its length (synchronises). */
int ngp_render_composite_round(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, uint32_t n_alive, uint32_t k_steps,
                               float min_transmittance, uint32_t cascades, float* rgb_out, float* alpha_out, uint32_t* n_samples_out,
                               uint32_t* n_alive_host);
/* V5: ngp_render_composite_round that also accumulates depth_out[g] += w_i * t_i over the samples it composites: the same weights
 * w_i = alpha_i * T_i, the same samples in the same order and the same stopping rule, with t_i the sample's ray parameter in model (NGP)
 * units.  The reference has no counterpart (its renderer returns colour only); the convention is pixelNeRF's depth_map = sum(w * z)
 * (render_rays), unnormalised: divide by alpha and by the dataset's scale for the expected distance in NeRF world units.  The caller zeroes
 * depth_out (n_rays floats) before the first round; rays that miss the box are never composited and keep 0.  Call it in place of V4 in
 * every round of a frame; rgb, alpha and sample counts are bit-identical to V4's.  A NULL depth_out is an error. */
int ngp_render_composite_round_depth(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, uint32_t n_alive, uint32_t k_steps,
                                     float min_transmittance, uint32_t cascades, float* rgb_out, float* alpha_out, uint32_t* n_samples_out,
                                     float* depth_out, uint32_t* n_alive_host);
/* V6: ngp_render_composite_round that also accumulates normal_out[3g .. 3g+3) += w_i * n_i over the samples it composites, n_i =
 * -grad_i / |grad_i| (0 where grad_i is 0) with grad_i row i of grad_rows: the round's (capacity,3) f32 density gradients, written by
 * ngp_density_grad over the round's rows after the network.  The same weights, samples, order and stopping rule as V4, so the sum is
 * the opacity-weighted mean outward normal in model (NGP) axes, unnormalised: normalise it, and cycle the axes back for NeRF world axes.
 * The reference has no counterpart.  depth_out may be NULL; if not, it accumulates as in V5, so one render gives colour, depth and
 * normals.  The caller zeroes normal_out (3 n_rays floats) and depth_out before the first round.  rgb, alpha, sample counts and depth
 * are bit-identical to V4's and V5's.  A NULL grad_rows or normal_out is an error. */
int ngp_render_composite_round_normals(void* stream, uint32_t n_rays, uint32_t capacity, void* workspace, uint32_t n_alive, uint32_t k_steps,
                                       float min_transmittance, uint32_t cascades, float* rgb_out, float* alpha_out, uint32_t* n_samples_out,
                                       const float* grad_rows, float* normal_out, float* depth_out, uint32_t* n_alive_host);

/* ---- R10 occupancy-grid maintenance (DGS/density_grid_sampler.py:204-264 + five headers) ------------- */
int ngp_grid_mark_untrained(void* stream, uint32_t n_elements, float* grid, uint32_t n_images, const float* focal_lengths,
                            const float* xforms, int res_x, int res_y);
/* ngp_grid_mark_untrained for captures whose frames carry their own cameras (extends mark_untrained_density_grid.h, which takes one
 * symmetric frustum per image): extents is a 16-byte aligned (n_images, 4) f32 device array of every image's normalised frustum
 * (x_lo, x_hi, y_lo, y_hi) in camera coordinates (x right, y down, z forward), signed, so an off-centre principal point or a lens is
 * represented exactly. */
int ngp_grid_mark_untrained_cams(void* stream, uint32_t n_elements, float* grid, uint32_t n_images, const float* extents, const float* xforms);
int ngp_grid_generate_samples(void* stream, uint32_t n_elements, uint64_t rng_state, uint64_t rng_inc, const uint32_t* step_dev,
                              float aabb_lo, float aabb_hi, const float* grid_in, float* positions_out, uint32_t* indices_out,
                              uint32_t n_cascades, float thresh);
int ngp_grid_splat(void* stream, uint32_t n, const uint32_t* indices, const void* mlp_out, int dtype, float* grid_tmp);
int ngp_grid_ema(void* stream, uint32_t n_elements, float decay, float* grid, const float* grid_tmp);
/* mean over cascade 0 + grid_to_bitfield + max-pools (DGS/update_bitfield.py:13-37). mean_out: device float[1] */
int ngp_grid_update_bitfield(void* stream, const float* grid, float* mean_out, uint8_t* bitfield, uint32_t cascades);

/* ---- N1  fused Adam + EMA + gradient zeroing (optims/adam.py, ema.py, expdecay.py) -------------------- */
int ngp_adam_ema(void* stream, uint64_t n, void* param, int param_dtype, void* grad, int grad_dtype, float grad_scale,
                 float* m, float* v, float* master, float lr, float beta1, float beta2, float eps, uint32_t step,
                 float ema_decay, int zero_grad);
/* The optimizer tail of a single-GPU training step after ngp_network_bwd_fx(n_max = bwd_rows, fx, w_part), one launch: the weight
 * gradients summed from the slots, the table gradient rounded from the fixed-point sums, fx cleared again, and Adam+EMA (grad_scale 1)
 * on the fp16 table (2 * n_entries parameters) and both fp16 MLP weight vectors.  Bit for bit what ngp_network_bwd into zeroed
 * gradients followed by ngp_adam_ema(zero_grad) on each of the three gives. */
int ngp_train_sweep(void* stream, uint64_t n_entries, void* table, float* m, float* v, float* master, void* fx, const float* w_part,
                    uint32_t bwd_rows, void* w_density, float* wd_m, float* wd_v, float* wd_master, void* w_rgb, float* wr_m,
                    float* wr_v, float* wr_master, float lr, float beta1, float beta2, float eps, uint32_t step, float ema_decay);

/* ---- 8e data-parallel exchange fused with the optimizer, over NVLink peer memory ------------------------------------
 * The reference has no multi-GPU path for NGP (SURVEY.md 8e; its only exchange is jt.mpi all-reduce inside nn optimizers,
 * python/jnerf/optims/adam.py:8-16 via jt.nn.Adam).  One launch per step replaces gradient all-reduce + Adam + EMA:
 * reduce-scatter by pulling the peers' gradient slices, Adam+EMA on this rank's slice of the padded hash table, all-gather
 * by pushing the fp16 slice into every peer's table, all-reduce + update of the MLP weights; flag hand-shake in peer memory.
 * peer_* are HOST arrays of `world` DEVICE pointers (own rank = local buffers, others = ngp_ipc_open mappings):
 *   peer_table / peer_table_grad: fp16, world*slice_len elements; peer_w_grad: fp32 n_w; peer_flags: 64 zero-initialised words.
 * m/v/master: this rank's slice state (slice_len fp32 each); w_*: local MLP weights (fp16) and their fp32 state (n_w).
 * epoch: 1,2,3,... identical on all ranks.  Gradients are NOT zeroed: call ngp_dp_exchange_wait(epoch) first, then clear them. */
int ngp_dp_exchange_step(void* stream, int world, int rank, uint64_t slice_len, uint32_t n_w, void* const* peer_table,
                         void* const* peer_table_grad, float* const* peer_w_grad, uint32_t* const* peer_flags, uint32_t epoch, float* m,
                         float* v, float* master, void* w_param, float* w_m, float* w_v, float* w_master, float grad_scale, float lr,
                         float beta1, float beta2, float eps, uint32_t step, float ema_decay);
/* Stream-ordered wait until every peer finished epoch `epoch` (their stores into this rank's table are visible and they no
 * longer read this rank's gradients).  Traps after 20 s instead of hanging. */
int ngp_dp_exchange_wait(void* stream, int world, const uint32_t* my_flags, uint32_t epoch);
/* CUDA IPC plumbing: export the allocation containing dev_ptr (64-byte handle + byte offset), map a peer's export. */
int ngp_ipc_export(const void* dev_ptr, uint8_t* handle64, uint64_t* offset);
int ngp_ipc_open(const uint8_t* handle64, uint64_t offset, void** dev_ptr);
int ngp_ipc_close(void* dev_ptr, uint64_t offset);

/* ---- N2  ray generation + target blend (dataset/dataset.py:172-188, runner/runner.py:65-68) ------------ */
int ngp_raygen(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms,
               const float* focal, const float* principal, uint32_t* img_id_out, float* rays_o, float* rays_d);

/* ray generation + RGBA gather (uint8/255 or f32 images, (n_img*H*W,4)) + target = rgb*a + bg*(1-a) in one launch */
int ngp_prepare_batch(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms,
                      const float* focal, const float* principal, const void* images_rgba, int image_is_u8, const float* bg,
                      uint32_t* img_id_out, float* rays_o, float* rays_d, float* target);

/* ngp_raygen / ngp_prepare_batch through a radial-tangential lens (extends dataset/dataset.py:123-126 and ray_sampler.h:37, which read
 * k1, k2, p1, p2 into camera_distortion and never apply them): distortion is a 16-byte aligned (n_img, 4) f32 device array of every
 * image's (k1, k2, p1, p2).  Each pixel's normalised coordinate ((u - cx)/fx, (v - cy)/fy) is undistorted by Newton's method in fp32
 * (OpenCV's model, y down) before it is turned into a direction.  prepare_batch_lens gives the rays of raygen_lens bit for bit and the
 * targets of ngp_prepare_batch bit for bit.  A NULL distortion is an error; for a pinhole capture call the entry points above. */
int ngp_raygen_lens(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms,
                    const float* focal, const float* principal, const float* distortion, uint32_t* img_id_out, float* rays_o, float* rays_d);
int ngp_prepare_batch_lens(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t W, uint32_t H, const float* xforms,
                           const float* focal, const float* principal, const float* distortion, const void* images_rgba, int image_is_u8,
                           const float* bg, uint32_t* img_id_out, float* rays_o, float* rays_d, float* target);

/* ngp_raygen / ngp_prepare_batch for captures whose frames carry their own cameras and image sizes (extends dataset/dataset.py:172-188,
 * which takes one W, H for all images): image i is wh[i] = (w, h) pixels (an 8-byte aligned (n_images, 2) uint32 device array) and
 * owns the global pixel ids [pixel_offsets[i], pixel_offsets[i+1]) of the ragged (total_pixels, 4) RGBA table, row-major; pixel_offsets
 * holds the n_images + 1 prefix sums of w*h.  A NULL distortion builds pinhole rays, else every pixel goes through its image's lens as in
 * ngp_raygen_lens.  On a capture whose images all share one size the rays and targets are those of ngp_raygen / ngp_prepare_batch (or
 * their _lens forms) bit for bit. */
int ngp_raygen_cams(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t n_images, const uint32_t* pixel_offsets, const uint32_t* wh,
                    const float* xforms, const float* focal, const float* principal, const float* distortion, uint32_t* img_id_out, float* rays_o,
                    float* rays_d);
int ngp_prepare_batch_cams(void* stream, uint32_t n, const uint32_t* pix_index, uint32_t n_images, const uint32_t* pixel_offsets, const uint32_t* wh,
                           const float* xforms, const float* focal, const float* principal, const float* distortion, const void* images_rgba,
                           int image_is_u8, const float* bg, uint32_t* img_id_out, float* rays_o, float* rays_d, float* target);

/* target = rgb*a + bg*(1-a) (runner/runner.py:68) for a batch whose RGBA (n,4) f32 is already gathered (host-fed ray batches) */
int ngp_blend_target(void* stream, uint32_t n, const float* rgba, const float* bg, float* target);

/* pcg32 helpers (ops/op_include/pcg32/pcg32.h): host-side, pure integer */
void ngp_pcg32_seed(uint64_t initstate, uint64_t initseq, uint64_t* state_inc);
void ngp_pcg32_advance(uint64_t* state_inc, int64_t delta);

#ifdef __cplusplus
}
#endif
#endif
