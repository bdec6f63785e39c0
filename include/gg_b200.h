/*
 * gg_b200.h -- C ABI of libgg_b200.so: the sm_90a kernels behind GANgealing's op-level hot path.
 *
 * Every entry point replaces one native binding (or one cluster of ATen launches) of the reference
 * wpeebles/gangealing; the reference location is cited on each declaration (paths relative to the
 * reference checkout).  Conventions, identical for all entry points:
 *
 *   - plain pointers and sizes only, no torch types; all pointers are DEVICE pointers unless the
 *     parameter name ends in `_host`;
 *   - the caller owns every buffer (inputs, outputs, workspaces); the library allocates nothing,
 *     keeps no mutable global state and never synchronises the device;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - return value: 0 = ok, negative = error (GG_ERR_*); gg_last_error() returns a thread-local
 *     human-readable message for the last failing call on this thread.  Never calls exit();
 *   - re-entrant: safe to call concurrently from the Python main thread and PyTorch's autograd thread;
 *   - tensors are dense ("contiguous") in the layout stated per function; element type is selected
 *     by a gg_dtype code; accumulation is always fp32.
 *   - staged (bulk-TMA) kernels may READ, never write, up to 15 bytes before/after an input buffer so
 *     that transfers are 16-byte aligned; those bytes never influence results.  (Any CUDA allocation
 *     is at least 256-byte granular, so the enclosing 16-byte window is always mapped.)
 */
#ifndef GG_B200_H_
#define GG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GG_API __attribute__((visibility("default")))

/* element types */
enum { GG_F32 = 0, GG_F16 = 1, GG_BF16 = 2, GG_F64 = 3 };

/* error codes */
enum {
  GG_OK = 0,
  GG_ERR_BAD_ARG = -1,      /* null pointer, negative size, inconsistent shape            */
  GG_ERR_UNSUPPORTED = -2,  /* dtype / mode not implemented by this entry point           */
  GG_ERR_CUDA = -3          /* a CUDA runtime call failed; message holds cudaGetErrorString */
};

/* padding modes of the samplers (torch.nn.functional.grid_sample's padding_mode) */
enum { GG_PAD_ZEROS = 0, GG_PAD_BORDER = 1, GG_PAD_REFLECTION = 2 };

GG_API int gg_version(void);                 /* ABI version, bumped on any signature change */
GG_API const char* gg_last_error(void);      /* thread-local, never NULL */
GG_API int gg_sm_count(void);                /* multiProcessorCount of the current device (cached) */

/* ------------------------------------------------------------------------------------------------
 * fused_bias_act -- replaces `fused.fused_bias_act(input, bias, refer, act, grad, alpha, scale)`
 *   reference: models/stylegan2/op/fused_bias_act.cpp:11-21, fused_bias_act_kernel.cu:18-99
 *   x'   = x + bias[(i / step_b) % size_b]            (bias == NULL: no bias)
 *   act=1: y = x'                       (grad 0/1), 0 (grad 2)
 *   act=3: y = x'   > 0 ? x' : alpha*x' (grad 0)
 *          y = ref  > 0 ? x' : alpha*x' (grad 1; ref = saved forward OUTPUT), 0 (grad 2)
 *   out = y * scale
 *   x/out/ref: `size_x` elements of `dtype`; bias: `size_b` elements of `dtype`.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_fused_bias_act(void* out, const void* x, const void* bias, const void* ref, int dtype,
                             int act, int grad, float alpha, float scale, int64_t size_x,
                             int64_t step_b, int64_t size_b, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_noise_bias_act -- NoiseInjection + FusedLeakyReLU of a StyledConv in one pass
 *   reference: models/stylegan2/networks.py:291-298 (noise) + :344-350 + op/fused_act.py:52-58
 *   out[n,c,p] = lrelu(row_scale[n*C+c]*x[n,c,p] + noise_weight[0]*noise[n,p] + bias[c], alpha) * scale
 *   x/out: (N, C, HW) `dtype`;  noise: (N, HW) `dtype` or NULL;  noise_weight: 1 fp32 (device) or
 *   NULL (=1);  bias: C fp32 or NULL;  row_scale: N*C fp32 or NULL (=1; the demodulation coefficients when
 *   the convolution ran with shared weights on modulated activations).
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_noise_bias_act(void* out, const void* x, const void* noise, const float* noise_weight,
                             const float* bias, const float* row_scale, int dtype, float alpha, float scale,
                             int64_t N, int64_t C, int64_t HW, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_channel_scale -- per-(sample, channel) scaling of an activation, the modulation of
 *   reference models/stylegan2/networks.py:236,243 applied to the convolution's INPUT instead of its weights:
 *   conv(scale*W*s[b,i], x) == conv(scale*W, x*s[b,i])  -> weight-shared (dense, tensor-core friendly) convolutions.
 *   out[r,p] = x[r,p] * s[r]        rows r = n*C + c, p < HW
 *   row_dot[r] = sum_p x[r,p]*y[r,p]   (optional; with y = upstream gradient this is d/ds; fp32, deterministic;
 *   needs gg_channel_scale_workspace(rows, HW) bytes)
 * ---------------------------------------------------------------------------------------------- */
GG_API int64_t gg_channel_scale_workspace(int64_t rows, int64_t HW);
GG_API int gg_channel_scale(void* out, float* row_dot, void* workspace, const void* x, const void* y,
                            const float* s, int dtype, int64_t rows, int64_t HW, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_bias_act_backward -- FusedLeakyReLUFunctionBackward in one pass
 *   reference: models/stylegan2/op/fused_act.py:20-38 (kernel call act=3,grad=1 + grad_input.sum(dims))
 *   gx[n,c,p] = (out[n,c,p] > 0 ? g : alpha*g) * scale
 *   grad_bias[c] = sum_{n,p} gx[n,c,p]      (fp32; skipped when grad_bias == NULL)
 *   Deterministic two-stage reduction; `workspace` must hold gg_bias_act_backward_workspace() bytes
 *   (may be NULL when grad_bias is NULL).
 * ---------------------------------------------------------------------------------------------- */
GG_API int64_t gg_bias_act_backward_workspace(int64_t N, int64_t C, int64_t HW);
GG_API int gg_bias_act_backward(void* gx, float* grad_bias, void* workspace, const void* g,
                                const void* out, int dtype, float alpha, float scale, int64_t N,
                                int64_t C, int64_t HW, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_upfirdn2d -- replaces `upfirdn2d_op.upfirdn2d(input, kernel, up_x, up_y, down_x, down_y,
 *                                                  pad_x0, pad_x1, pad_y0, pad_y1)`
 *   reference: models/stylegan2/op/upfirdn2d.cpp:12-23, upfirdn2d_kernel.cu:209-369
 *   (semantics: upfirdn2d.py:159-200 -- zero-insert upsample, pad/crop, TRUE convolution with
 *    `kernel`, decimate).  in: (major, in_h, in_w) dense; out: (major, out_h, out_w) with
 *    out_h = (in_h*up_y + pad_y0 + pad_y1 - kernel_h) / down_y + 1 (same for w); the reference's
 *    trailing `minor` dimension is always 1 in GANgealing and is not modelled.
 *   kernel: kernel_h*kernel_w fp32 taps (device), NOT flipped (the library flips, as the reference).
 *   Dispatch: up=down=1 and kernel <= 4x4 -> bulk-TMA staged band kernel; otherwise generic gather.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_upfirdn2d(void* out, const void* in, const float* kernel, int dtype, int64_t major,
                        int in_h, int in_w, int kernel_h, int kernel_w, int up_x, int up_y,
                        int down_x, int down_y, int pad_x0, int pad_x1, int pad_y0, int pad_y1,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_blur_noise_bias_act -- the fused StyledConv(upsample) tail: Blur -> NoiseInjection ->
 *   FusedLeakyReLU in ONE pass over the activation (the "fused upfirdn2d+bias-act path").
 *   reference: models/stylegan2/networks.py:266 (blur) + :346-348 (noise, activate);
 *              op/upfirdn2d_kernel.cu:107-207 + op/fused_bias_act_kernel.cu:18-49
 *   t = upfirdn2d(in, kernel, up=1, down=1, pad)               (kernel <= 4x4)
 *   out[n,c,y,x] = lrelu(row_scale[n*C+c]*t + noise_weight[0]*noise[n,y,x] + bias[c], alpha) * scale
 *   in: (N*C, in_h, in_w) dtype; out: (N*C, out_h, out_w); noise: (N, out_h, out_w) dtype or NULL;
 *   noise_weight: 1 fp32 or NULL(=1); bias: C fp32 or NULL; row_scale: N*C fp32 or NULL (=1; lets a
 *   caller fold the per-sample demodulation of a weight-shared conv into the tail);
 *   act: 1 linear, 3 leaky-relu.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_blur_noise_bias_act(void* out, const void* in, const float* kernel, const void* noise,
                                  const float* noise_weight, const float* bias,
                                  const float* row_scale, int dtype, int64_t N, int64_t C, int in_h,
                                  int in_w, int kernel_h, int kernel_w, int pad_x0, int pad_x1,
                                  int pad_y0, int pad_y1, int act, float alpha, float scale,
                                  void* stream);

/* ------------------------------------------------------------------------------------------------
 * Antialiased (mip-mapped) bilinear grid sampling -- replaces MipmapWarp / Warp
 *   reference: models/spatial_transformers/antialiased_sampling.py:9-16 (Warp), :35-238 (MipmapWarp)
 *   and the ATen kernels behind F.grid_sample(align_corners=False) / F.interpolate / F.conv2d they call.
 *
 *   Pyramid: level i (1..extra_levels) = i applications of [ReflectionPad2d(1) -> depthwise
 *   [1,3,3,1]^2/64 stride-2 conv] (:111-117) to the source, after the reference's reflect padding to the
 *   next power of two when the width is not one (:130-137).  Stored fp32, level-major, at native
 *   resolution: gg_mipmap_pyramid_elems() floats (returns -1 if the size cannot host that many levels,
 *   exactly when the reference's stack construction would fail).
 *
 *   forward : out[n,c,y,x] = lerp(S_floor(l), S_ceil(l), l mod 1),  S_i = bilinear sample of level i
 *             upsampled x2^i (align_corners=False) at grid[n,y,x]; l = clamp(log2(max 4-neighbour
 *             distance of the (size-1)-scaled coordinates, each >= 1), 0, max_level) clamped >= min_level
 *             (:62-97, :181-210).  extra_levels == 0: plain bilinear grid_sample (Warp).
 *             levels_out (N,Ho,Wo) fp32 receives l (NULL to skip).
 *   backward: gradients w.r.t. the source (through every pyramid level; grad_src/grad_pyramid are fp32,
 *             ZERO-INITIALISED by the caller and accumulated with atomics; finish with
 *             gg_mipmap_build_backward) and w.r.t. the grid (sampling position AND level-of-detail terms,
 *             like autograd through the reference; grad_grid fp32, written: gathered in a fixed order, without
 *             atomics, so it is the same in every run).
 *   src/out/grad_out: `dtype`; grid: fp32 (N, Ho, Wo, 2), normalised to [-1, 1].
 * ---------------------------------------------------------------------------------------------- */
GG_API int64_t gg_mipmap_pyramid_elems(int64_t planes, int hs, int ws, int extra_levels);
GG_API int gg_mipmap_build(float* pyramid, const void* src, int dtype, int64_t planes, int hs, int ws,
                           int extra_levels, void* stream);
GG_API int gg_mipmap_build_backward(float* grad_src, float* grad_pyramid, int64_t planes, int hs, int ws,
                                    int extra_levels, void* stream);
GG_API int gg_mipmap_warp_forward(void* out, float* levels_out, const void* src, const float* pyramid,
                                  const float* grid, int dtype, int64_t N, int C, int hs, int ws, int ho,
                                  int wo, int extra_levels, float max_level, float min_level,
                                  int padding_mode, void* stream);
GG_API int gg_mipmap_warp_backward(float* grad_src, float* grad_pyramid, float* grad_grid,
                                   const void* grad_out, const void* src, const float* pyramid,
                                   const float* grid, int dtype, int64_t N, int C, int hs, int ws, int ho,
                                   int wo, int extra_levels, float max_level, float min_level,
                                   int padding_mode, void* stream);
/* The sampler's INTEGER work, exported for exact parity tests (no reference counterpart: ATen's grid_sampler_2d and
 * antialiased_sampling.py:228-229 compute these integers internally).  indices: int32 (N, Ho, Wo, 4), 16-byte aligned =
 * (x0, y0, l0, l1): north-west bilinear corner after the padding-mode transform, floor / ceil of the level of detail --
 * evaluated by the same device functions as the forward sampler of gg_mipmap_warp_forward / gg_stn_sample_forward. */
GG_API int gg_warp_sample_indices(int32_t* indices, const float* grid, int64_t N, int hs, int ws, int ho, int wo,
                                  float max_level, float min_level, int padding_mode, void* stream);
/* Congealing animations: vis_correspondence.py:183-205 (smoothly_sample_image) and :335-380 (create_average_image), i.e.
 * warper(data, base.lerp(target, alpha_t)) for T lerp weights at once.  The grid of frame t, sample n is
 * lerp(base[n], target[n], alphas[t]) with torch.lerp's formula (bitwise torch.lerp on the device); the level of detail and
 * the trilinear sample are gg_mipmap_warp_forward's.  One pyramid (gg_mipmap_build of src) serves all T frames.
 *   base (N or 1, ho, wo, 2) fp32: base_stride = ho*wo*2, or 0 for one broadcast grid; target (N, ho, wo, 2) fp32;
 *   alphas (T,) fp32 on the device; T >= 1.
 *   gg_mipmap_warp_lerp_forward: out (T, N, C, ho, wo) `dtype`; grid_out (T, N, ho, wo, 2) fp32 or NULL.
 *   gg_mipmap_warp_lerp_mean: acc (T, C, ho, wo) fp32, s = 0; for n = 0..N-1 in order: s += sample_n(frame t) (each value
 *     rounded to `dtype` as gg_mipmap_warp_lerp_forward stores it); acc = accumulate ? acc + s : s.  No atomics: bitwise
 *     reproducible, and bitwise a sequential fp32 sum of gg_mipmap_warp_lerp_forward's frames.  1 <= C <= 4. */
GG_API int gg_mipmap_warp_lerp_forward(void* out, float* grid_out, const void* src, const float* pyramid, const float* base,
                                       int64_t base_stride, const float* target, const float* alphas, int T, int dtype,
                                       int64_t N, int C, int hs, int ws, int ho, int wo, int extra_levels, float max_level,
                                       float min_level, int padding_mode, void* stream);
GG_API int gg_mipmap_warp_lerp_mean(float* acc, const void* src, const float* pyramid, const float* base, int64_t base_stride,
                                    const float* target, const float* alphas, int T, int dtype, int64_t N, int C, int hs,
                                    int ws, int ho, int wo, int extra_levels, float max_level, float min_level,
                                    int padding_mode, int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Flow composition of the flow STN head -- replaces upsample_flow + identity add + apply_affine + alpha lerp
 *   reference: models/spatial_transformers/warping_heads.py:180-193 (RAFT convex upsampling: softmax over the
 *   9 mask logits x F.unfold(S*flow, 3x3, padding=1)), :239-244, :268-277 (apply_affine: [gx, gy, 1] @ M^T)
 *   low_flow (N, H, W, 2); mask (N, 9*S*S, H, W); identity_flow (S*H, S*W, 2) = F.affine_grid(identity);
 *   base_warp (N, 2, 3) or NULL; alpha (N) or NULL.  All fp32.
 *   forward : delta_flow (N, S*H, S*W, 2) and, if `flow` != NULL, flow = lerp(identity, affine(identity + delta), alpha)
 *   backward: grad_mask, grad_low_flow and grad_base_warp (written; grad_base_warp is zero unless grad_flow and
 *             base_warp are given); reduced in a fixed order, without atomics, so the result is the same in every run;
 *             grad_delta / grad_flow are the incoming gradients (either may be NULL).
 *   low_flow, identity_flow, delta_flow, flow, grad_low_flow, grad_delta and grad_flow are read or written as float2:
 *   a pointer off an 8-byte boundary is refused (GG_ERR_BAD_ARG) before any device work.  So are the float2 grids of
 *   the samplers below (grid, grid_out, delta_out, base, target, grad_grid, and mode 2's low and identity).
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_flow_compose_forward(float* delta_flow, float* flow, const float* low_flow, const float* mask,
                                   const float* identity_flow, const float* base_warp, const float* alpha,
                                   int64_t N, int H, int W, int S, void* stream);
GG_API int gg_flow_compose_backward(float* grad_mask, float* grad_low_flow, float* grad_base_warp,
                                    const float* grad_delta, const float* grad_flow, const float* low_flow,
                                    const float* mask, const float* identity_flow, const float* base_warp,
                                    const float* alpha, int64_t N, int H, int W, int S, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_splat2d_forward -- replaces `_splat.splat_forward_cuda(input, coordinates, values, sigma, soft_normalize)`
 *   reference: utils/splat2d_cuda/src/splat_gpu.c:12-42 (host: zeros/clone/clamp/divide) and
 *              splat_gpu_impl.cu:41-96 / splat_gpu_impl.cuh:11-22 (kernel `SplatForward`, extern-C `SplatForwardGpu`)
 *   For every point (x, y) inside the image (0 <= x < W, 0 <= y < H) and every pixel of its footprint
 *   [floor(y-2s), ceil(y+2s)] x [floor(x-2s), ceil(x+2s)] clipped to the image:
 *       a = exp(-((px-x)^2 + (py-y)^2) / (2 s^2));  A[py,px] += a;  S[c,py,px] += a * value[c]
 *   out = (input + S) / ((soft_normalize ? max(A, 1) : A) + 1e-8)
 *   input/out (N, C, H, W); coordinates (N, P, 2) as (x, y); values (N, P, C); sigma (N).  fp32 only, forward
 *   only (as the reference).  `workspace`: gg_splat2d_workspace() bytes (interleaved accumulators; the
 *   library zeroes it).
 * ---------------------------------------------------------------------------------------------- */
GG_API int64_t gg_splat2d_workspace(int64_t N, int C, int H, int W);
GG_API int gg_splat2d_forward(float* out, void* workspace, const float* input, const float* coordinates,
                              const float* values, const float* sigma, int64_t N, int64_t P, int C, int H,
                              int W, int soft_normalize, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_splat_composite_grid -- the label-propagation animation's frames (reference applications/vis_correspondence.py:133-158):
 *   for every frame t and image n, splat_points' two splats at points[t, n] (utils/vis_tools/helpers.py:178-187; the
 *   footprint, weight and bounds of gg_splat2d_forward at sigma), the alpha composite over images[t, n], then images2grid
 *   (helpers.py:39-43: torchvision make_grid(nrow, padding, normalize=True, range=(-1, 1)) and the uint8 quantisation):
 *       A = sum a, S_c = sum a * colors[c], S_alpha = sum a * alpha (= A when alpha is NULL)
 *       v = m * (S_c / (A + 1e-8)) + (1 - m) * img,  m = (S_alpha / (max(A, 1) + 1e-8)) * opacity
 *       out = uint8(clamp(((clamp(v, -1, 1) - (-1)) / 2) * 255 + 0.5, 0, 255))   (every operation rounded on its own)
 *   laid out as make_grid does: xmaps = min(nrow, N), ymaps = ceil(N / xmaps), pad value 0; N == 1: the bare image.
 *   out (T, Hg, Wg, 3) uint8; images (T, N, 3, R, R) fp32; points (T, N, P, 2) fp32 pixels (x, y), 8-byte aligned;
 *   colors (colors_n, P, 3) and alpha (alpha_n, P, 1) fp32 or NULL, broadcast over the frames, colors_n / alpha_n 1 or N.
 *   P == 0: points, colors and workspace may be NULL, and out is images2grid of the frames.  C must be 3.
 *   `workspace`: 16-byte aligned, workspace_bytes of it; frames are splatted in chunks of
 *   workspace_bytes / gg_splat_composite_grid_workspace(1, N, R, alpha != NULL) frames (at least one must fit).
 *   Float atomics: with more than two contributions per pixel the sums' last bits depend on their order.
 *   Arguments are validated before any device work (GG_ERR_BAD_ARG).
 * ---------------------------------------------------------------------------------------------- */
GG_API int64_t gg_splat_composite_grid_workspace(int64_t T_chunk, int64_t N, int R, int has_alpha);
GG_API int gg_splat_composite_grid(unsigned char* out, void* workspace, int64_t workspace_bytes, const float* images,
                                   const float* points, const float* colors, const float* alpha, float sigma,
                                   float opacity, int64_t T, int64_t N, int64_t P, int C, int R, int nrow, int padding,
                                   int colors_n, int alpha_n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * gg_splat_lookup_composite_grid -- a dense label or edit put on real images (reference
 *   applications/propagate_to_images.py:62-73): gg_splat_composite_grid for one grid (T = 1) whose points are looked up
 *   first.  For image n and point p:
 *       q = query[query_n == 1 ? 0 : n, p]                              (normalised congealed-frame coordinates)
 *       x, y = unnormalize(grid_sample(grid[n], q, 'border'), R, R)     (uncongeal_points, as gg_splat2d_lookup_forward:
 *                                                                        k = (R - 1) / R, m = R - 1)
 *       x = (R - 1) - x where flip[n]                                   (the point lands on the unflipped image)
 *   then the splats, composite and grid of gg_splat_composite_grid at (x, y), whose layout and bytes it shares.
 *   out (Hg, Wg, 3) uint8; points_out (N, P, 2) fp32 or NULL: the final pixel coordinates (the dense correspondences);
 *   images (N, 3, R, R) fp32; grid (N, grid_h, grid_w, 2) fp32; query (query_n, P, 2) fp32; flip (N,) bytes or NULL
 *   (no image flipped); colors (colors_n, P, 3), alpha (alpha_n, P, 1) or NULL.  query, grid and points_out 8-byte aligned.
 *   P == 0: grid, query, colors and workspace may be NULL, and out is images2grid of the images.  C must be 3.
 *   `workspace`: 16-byte aligned, at least gg_splat_composite_grid_workspace(1, N, R, alpha != NULL) bytes.
 *   Arguments are validated before any device work (GG_ERR_BAD_ARG).
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_splat_lookup_composite_grid(unsigned char* out, float* points_out, void* workspace, int64_t workspace_bytes,
                                          const float* images, const float* grid, const float* query,
                                          const unsigned char* flip, const float* colors, const float* alpha, float sigma,
                                          float opacity, int64_t N, int64_t P, int query_n, int C, int R, int grid_h,
                                          int grid_w, int nrow, int padding, int colors_n, int alpha_n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The STN's sampling in ONE pass (north_star: "antialiased bilinear grid_sample fused with flow-compose in one pass").
 * The sampling grid is generated per output pixel from the head's raw outputs instead of being read from memory:
 *   mode 1  SimilarityHead (reference warping_heads.py:120-136): grid = F.affine_grid(theta (N, 2, 3), align_corners=False)
 *   mode 2  FlowHead (warping_heads.py:180-193 upsample_flow, :239-244, :268-277 apply_affine): low (N, lh, lw, 2),
 *           mask (N, 9*s*s, lh, lw), identity (s*lh, s*lw, 2), optional base warp `theta` (N, 2, 3) and alpha (N);
 *           ho == s*lh, wo == s*lw
 * then the level-of-detail selection + trilinear sample of gg_mipmap_warp_forward (antialiased_sampling.py:35-238; the
 * same kernel, which there reads the grid) on `src` (N, C, hs, ws) and its `pyramid` (gg_mipmap_build; extra_levels == 0:
 * plain bilinear sampling).
 * Outputs: out (N, C, ho, wo); grid_out (N, ho, wo, 2) and delta_out (mode 2: the residual flow of the TV regulariser,
 * reference models/losses/loss.py:4-12) are written as by-products (NULL: skipped); levels_out (N, ho, wo) or NULL.
 * The backward pass is gg_mipmap_warp_backward on grid_out (+ gg_flow_compose_backward for mode 2).
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_stn_sample_forward(void* out, float* grid_out, float* delta_out, float* levels_out, const void* src,
                                 const float* pyramid, const float* theta, const float* low, const float* mask,
                                 const float* identity, const float* alpha, int mode, int dtype, int64_t N, int C,
                                 int hs, int ws, int ho, int wo, int lh, int lw, int s, int extra_levels,
                                 float max_level, float min_level, int padding_mode, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Modulated-convolution weight path -- replaces the tensor-op chain of ModulatedConv2d.forward
 *   reference: models/stylegan2/networks.py:233-253 (modulate, demodulate), :255-262 (layout for the up-conv)
 *   weight (O, I, kk) fp32 [kk = k*k]; style (B, I) fp32 (output of the modulation EqualLinear).
 *   gg_modconv_wsq      wsq[o,i] = sum_kk weight[o,i,kk]^2
 *   gg_modconv_demod    demod[b,o] = rsqrt(scale^2 * sum_i wsq[o,i]*style[b,i]^2 + eps)   (B <= 256)
 *                       wgmma.mma_async tf32 with a hi/lo operand split (fp32-grade accuracy), register accumulator
 *   gg_modconv_modulate out = scale * weight * style[b,i] * demod[b,o]   (demod == NULL: no demodulation)
 *                       transposed == 0: out (B, O, I, kk), `weight` given as (O, I, kk)
 *                       transposed != 0: out (B, I, O, kk), `weight` given PRE-TRANSPOSED as (I, O, kk)
 *                       (I*kk, resp. O*kk, must be a multiple of 4)
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_modconv_wsq(float* wsq, const float* weight, int O, int I, int kk, void* stream);
GG_API int gg_modconv_demod(float* demod, const float* wsq, const float* style, float scale, float eps, int B,
                            int O, int I, void* stream);
/* all layers of a generator in ONE launch: tables (host arrays of `layers` entries) of per-layer demod (B, O[l]) outputs,
 * wsq (O[l], I[l]), style (B, I[l]), scale, O, I; every layer shares the batch size B <= 256; layers <= 32. */
GG_API int gg_modconv_demod_batched(int layers, float* const* demod, const float* const* wsq, const float* const* style,
                                    const float* scale, const int* O, const int* I, float eps, int B, void* stream);
GG_API int gg_modconv_modulate(float* out, const float* weight, const float* style, const float* demod,
                               float scale, int B, int O, int I, int kk, int transposed, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Channels-last (N, H, W, C) variants of the StyledConv tail family.  Same math and reference citations as
 * gg_noise_bias_act / gg_bias_act_backward / gg_channel_scale / gg_blur_noise_bias_act; they exist so the generator's
 * activations can stay NHWC between cuDNN's (NHWC-native) tensor-core convolutions.
 *   dtype: GG_F32 or GG_BF16 = the STORAGE type of the activations (arithmetic is fp32; BASELINE config 3 runs bf16
 *     activations -- the reference has no bf16 at all: models/stylegan2/op/upfirdn2d_kernel.cu:311 dispatches
 *     float/double/half only).  An activation moves 16 bytes at a time: C % 4 == 0 (fp32) / C % 8 == 0 (bf16).
 *     noise, bias, row scales, reductions are always fp32.
 *   gg_blur_nhwc: upfirdn2d(up = down = 1, filter <= 4x4) on (N, H, W, C), C % 32 == 0 (fp32) / C % 64 == 0 (bf16), input
 *     rows streamed with 4-D TMA tensor-map loads whose out-of-bounds zero fill is the padding; `separable` != 0 asserts a
 *     rank-1 filter (two 4-tap passes; the caller tests this once per filter).  mode:
 *       0  out = B(in)                                                          (Blur, networks.py:70-86)
 *       1  o = lrelu(row_scale[n,c]*B(in) + noise_weight*noise[n,y,x] + bias[c], alpha)*scale   (networks.py:266,291-298,346-348)
 *          out = o (may be NULL) and/or out2 = o*scale2[n,c] (may be NULL): out2 is the NEXT modulated convolution's
 *          input with its style modulation applied (networks.py:236,243), written by the pass that produces o
 *       2  adjoint epilogue (backward of mode 1's blur): t = B(in); out = t*row_scale[n,c]; row_dot[n,c] = sum_yx t*mul[n,y,x,c]
 *          (mul: same shape as out; NULL row_dot: no reduction) -- `workspace` of gg_blur_nhwc_workspace() bytes
 *   gg_blur_nhwc_mask: mode 1 with the SIGN MASK of o in place of `out`: mask[n,y,x,w] bit b = (o[n,y,x,32w+b] > 0, tested
 *     on the value as stored in `dtype`), (N, H, W, C/32) uint32 -- what the activation's derivative (op/fused_act.py:20-38)
 *     needs of o when nothing is reduced over it (gg_styled_tail_backward_mask_nhwc).  out2 as in mode 1 (may be NULL).
 *   workspaces: gg_nhwc_rowwise_workspace(N, C, HW) bytes for the optional reductions (row_dot (N, C); grad_bias (C)).
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_noise_bias_act_nhwc(void* out, const void* x, const float* noise, const float* noise_weight,
                                  const float* bias, const float* row_scale, int dtype, float alpha, float scale,
                                  int64_t N, int C, int64_t HW, void* stream);
GG_API int64_t gg_nhwc_rowwise_workspace(int64_t N, int C, int64_t HW);
GG_API int gg_channel_scale_nhwc(void* out, float* row_dot, void* workspace, const void* x, const void* y,
                                 const float* s, int dtype, int64_t N, int C, int64_t HW, void* stream);
GG_API int gg_bias_act_backward_nhwc(void* gx, float* grad_bias, void* workspace, const void* g,
                                     const void* out_saved, int dtype, float alpha, float scale, int64_t N, int C,
                                     int64_t HW, void* stream);
GG_API int64_t gg_blur_nhwc_workspace(int dtype, int64_t N, int C, int in_h, int in_w, int kernel_h, int kernel_w,
                                      int pad_x0, int pad_x1, int pad_y0, int pad_y1);
GG_API int gg_blur_nhwc(void* out, void* out2, const void* in, const float* kernel, const float* noise,
                        const float* noise_weight, const float* bias, const float* row_scale, const float* scale2,
                        const void* mul, float* row_dot, void* workspace, int dtype, int64_t N, int C, int in_h,
                        int in_w, int kernel_h, int kernel_w, int separable, int pad_x0, int pad_x1, int pad_y0,
                        int pad_y1, int mode, int act, float alpha, float scale, void* stream);
GG_API int gg_blur_nhwc_mask(void* mask, void* out2, const void* in, const float* kernel, const float* noise,
                             const float* noise_weight, const float* bias, const float* row_scale, const float* scale2,
                             int dtype, int64_t N, int C, int in_h, int in_w, int kernel_h, int kernel_w, int separable,
                             int pad_x0, int pad_x1, int pad_y0, int pad_y1, int act, float alpha, float scale,
                             void* stream);

/* ------------------------------------------------------------------------------------------------
 * StyledConv / ToRGB tails fused across layer boundaries (csrc/styled.cu), channels-last, dtype as above.
 * reference: models/stylegan2/networks.py:291-298 (NoiseInjection), :346-348 (StyledConv.forward), :236,243 (the style
 * modulation of the NEXT ModulatedConv2d, applied to its input here because conv(scale*W*s, x) == conv(scale*W, x*s)),
 * :389-405 (ToRGB: 1x1 modulated convolution without demodulation + bias + up-sampled skip).
 *   gg_styled_tail_nhwc:  o = act(demod[n,c]*raw + noise_weight*noise[n,p] + bias[c])*scale       raw: (N, HW, C)
 *        out = o                         (NULL: not written -- only a later backward pass needs it)
 *        xs  = o*s_next[n,c]             (NULL: not written)
 *        rgb[n,o3,p] = sum_c wm[n,o3,c]*o + rgb_bias[o3] + skip[n,o3,p]    (NULL: not computed; planar (N, 3, HW) fp32)
 *      C % 32 == 0 (fp32) / C % 64 == 0 (bf16).  One read of raw.
 *   gg_styled_tail_backward_nhwc: one pass over (g_xs, out[, raw]) ->
 *        g_o = g_xs*s_next + sum_o3 wm[n,o3,c]*g_rgb[n,o3,p];  g_t = act'(out)*scale*g_o;  g_raw = g_t*demod[n,c]
 *        d_s_next[n,c] = sum_p g_xs*out;  d_demod[n,c] = sum_p g_t*raw;  d_wm[n,o3,c] = sum_p g_rgb[n,o3,p]*out
 *      (each NULL: skipped; g_xs or g_rgb may be NULL; demod NULL: g_raw = g_t -- the blur layers apply demod in
 *      gg_blur_nhwc mode 2).  `workspace`: gg_styled_tail_backward_workspace() bytes.  Deterministic reductions.
 *      reduce_pitch: floats between consecutive samples of the sum outputs -- C (each a dense (N, C) / (N, 3, C) tensor) or
 *      R*C when they are the row slices [d_s_next | d_demod | d_wm x3] (requested ones only, in that order) of ONE (N, R, C)
 *      block, which is then finished by a single launch.  0 is accepted for C; any other value is refused before any
 *      device work.  HW == 0: the requested sums are 0 (a sum over no pixels).
 *   gg_styled_tail_mask_nhwc: gg_styled_tail_nhwc with the sign mask of o (see gg_blur_nhwc_mask; (N, HW, C/32) uint32,
 *      required) in place of `out`.
 *   gg_styled_tail_backward_mask_nhwc: g_raw of gg_styled_tail_backward_nhwc (same operations, same order) with act'(out)
 *      read from the sign mask: one pass over (g_xs, mask) -> g_raw, no sums, no workspace.  C % 32 == 0.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_styled_tail_nhwc(void* out, void* xs, float* rgb, const void* raw, const float* noise,
                               const float* noise_weight, const float* bias, const float* demod, const float* s_next,
                               const float* wm, const float* rgb_bias, const float* skip, int dtype, int act,
                               float alpha, float scale, int64_t N, int C, int64_t HW, void* stream);
GG_API int64_t gg_styled_tail_backward_workspace(int dtype, int64_t N, int C, int64_t HW);
GG_API int gg_styled_tail_backward_nhwc(void* g_raw, float* d_s_next, float* d_demod, float* d_wm, void* workspace,
                                        const void* g_xs, const float* g_rgb, const void* out_saved, const void* raw,
                                        const float* s_next, const float* demod, const float* wm, int dtype,
                                        float alpha, float scale, int64_t N, int C, int64_t HW, int64_t reduce_pitch,
                                        void* stream);
GG_API int gg_styled_tail_mask_nhwc(void* mask, void* xs, float* rgb, const void* raw, const float* noise,
                                    const float* noise_weight, const float* bias, const float* demod,
                                    const float* s_next, const float* wm, const float* rgb_bias, const float* skip,
                                    int dtype, int act, float alpha, float scale, int64_t N, int C, int64_t HW,
                                    void* stream);
GG_API int gg_styled_tail_backward_mask_nhwc(void* g_raw, const void* g_xs, const float* g_rgb, const void* mask,
                                             const float* s_next, const float* demod, const float* wm, int dtype,
                                             float alpha, float scale, int64_t N, int C, int64_t HW, void* stream);

/* to-RGB on channels-last activations (reference models/stylegan2/networks.py:389-405 `ToRGB.forward`: a 1x1 modulated
 * convolution without demodulation + bias + the up-sampled skip image; the reference builds B filter banks and runs a
 * grouped convolution).  One pass over the activation:
 *   out[n,o,p] = sum_i wm[n,o,i] * x[n,p,i] + bias[o] + skip[n,o,p]      x: (N, HW, C) NHWC; wm: (N, 3, C) fp32
 *   out, skip (optional), g: planar (N, 3, HW).  C % 32 == 0, C <= 1024.
 * backward: gx[n,p,i] = sum_o wm[n,o,i] g[n,o,p]  (NULL: skipped);  gwm[n,o,i] = sum_p g[n,o,p] x[n,p,i]  (NULL: skipped;
 * otherwise `workspace` of gg_to_rgb_nhwc_workspace(N, C, HW) bytes, deterministic two-stage reduction). */
GG_API int64_t gg_to_rgb_nhwc_workspace(int64_t N, int C, int64_t HW);
GG_API int gg_to_rgb_nhwc_forward(float* out, const float* x, const float* wm, const float* bias, const float* skip,
                                  int64_t N, int C, int64_t HW, void* stream);
GG_API int gg_to_rgb_nhwc_backward(float* gx, float* gwm, void* workspace, const float* g, const float* x,
                                   const float* wm, int64_t N, int C, int64_t HW, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Perceptual-loss front end (SURVEY.md 8(f) rank 2) on channels-last feature maps.
 * reference: models/losses/lpips.py:26-28 normalize_tensor, :193-195 squared difference, :197-205 per-channel `lins`
 * weights or plain channel sum, :226 spatial_average.
 *   out[n] = 1/HW * sum_p sum_c w[c] * (f0[n,p,c]/(|f0[n,p,:]|+eps) - f1[n,p,c]/(|f1[n,p,:]|+eps))^2
 * f0, f1 (and g0, g1): (N, HW, C) NHWC stored as `dtype` = GG_F32 or GG_BF16 (fp32 arithmetic, fp32 out / grad_out);
 * weight: (C) fp32 or NULL (= 1); C a power of two < 128, or a multiple of 128 up to 1024.
 * forward needs gg_feature_distance_workspace(N, C, HW) bytes (deterministic two-stage reduction).
 * backward: g0 / g1 (either may be NULL) = grad_out[n] * d out[n] / d f0 / d f1, one pass over both maps. */
GG_API int64_t gg_feature_distance_workspace(int64_t N, int C, int64_t HW);
GG_API int gg_feature_distance_forward(float* out, void* workspace, const void* f0, const void* f1,
                                       const float* weight, int dtype, int64_t N, int C, int64_t HW, float eps,
                                       void* stream);
GG_API int gg_feature_distance_backward(void* g0, void* g1, const float* grad_out, const void* f0, const void* f1,
                                        const float* weight, int dtype, int64_t N, int C, int64_t HW, float eps,
                                        void* stream);

/* VGG16 slice boundary of the perceptual loss: Conv2d -> ReLU -> [tap] -> MaxPool2d(2, 2) -> Conv2d
 * (reference models/losses/lpips_backbones.py:106-121 = torchvision vgg16().features 2-4, 7-9, 14-16, 21-23; ATen
 * threshold / max_pool2d_with_indices and their backwards).  One pass each on channels-last maps:
 *   forward : y = relu(raw + bias[c]) (N, H, W, C) and pooled = max over 2x2 windows, stride 2 (N, H/2, W/2, C)
 *   backward: grad_raw = [y > 0] * (grad_y + [pixel is the FIRST maximum of its window, row-major] * grad_pooled);
 *             grad_y / grad_pooled may be NULL (= 0).  No index map: the arg-max is recomputed from y with ATen's rule.
 * raw / y / pooled / grads: `dtype` = GG_F32 or GG_BF16; bias: (C) fp32 or NULL; C % (16 / sizeof(dtype)) == 0; H, W even. */
GG_API int gg_bias_relu_pool_nhwc_forward(void* y, void* pooled, const void* raw, const float* bias, int dtype, int64_t N,
                                          int C, int H, int W, void* stream);
GG_API int gg_bias_relu_pool_nhwc_backward(void* grad_raw, const void* grad_y, const void* grad_pooled, const void* y,
                                           int dtype, int64_t N, int C, int H, int W, void* stream);

/* ------------------------------------------------------------------------------------------------
 * BilinearDownsample (SURVEY.md 8(f) rank 1): reference models/spatial_transformers/antialiased_sampling.py:241-256 --
 * ReflectionPad2d(stride/2) + depthwise 1x2s conv, stride (1,s) + depthwise 2sx1 conv, stride (s,1).  One gather:
 *   out[m,oy,ox] = sum_i sum_j taps_v[c][i] taps_h[c][j] in[m, R(oy*s+i-p), R(ox*s+j-p)],  p = s/2, R = reflection
 * in: (N, C, in_h, in_w) fp32 NCHW; taps_h / taps_v: (C, 2*stride) (the module's `kernel_horz` / `kernel_vert` buffers);
 * out: (N, C, (in_h+2p-2s)/s+1, (in_w+2p-2s)/s+1).  backward = the exact adjoint, gather form (deterministic). */
GG_API int gg_tent_downsample_forward(float* out, const float* in, const float* taps_h, const float* taps_v, int64_t N,
                                      int C, int in_h, int in_w, int stride, void* stream);
GG_API int gg_tent_downsample_backward(float* grad_in, const float* grad_out, const float* taps_h, const float* taps_v,
                                       int64_t N, int C, int in_h, int in_w, int stride, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Point-transfer path (SURVEY.md 8(f) rank 4), csrc/points.cu + csrc/splat.cu.
 *   gg_nn_argmin: reference spatial_transformer.py:655-668 (`congeal_points` of a flow STN): index[n, p] = argmin over the
 *     HW entries of grid (N, HW, 2) of |p|^2 + |g|^2 - 2 g.p (the reference's expanded form and rounding; first minimum
 *     wins) for points (N, P, 2).  No (N, H, W, P) distance tensor; `workspace` of gg_nn_argmin_workspace(N, P) bytes.
 *     Non-finite distances follow torch.argmin: the first NaN wins, an all-+inf row gives 0; every index is in [0, HW).
 *   gg_splat2d_lookup_forward: reference spatial_transformer.py:141-157 (`uncongeal_points`: F.grid_sample of the sampling
 *     grid at the query points, 'border', align_corners=False; `unnormalize` :621-623) fused into gg_splat2d_forward's point
 *     load: query (N, P, 2) normalised congealed-frame coordinates, grid (N, grid_h, grid_w, 2); pixel coordinate =
 *     ((g / unnorm_k) / 2 + 0.5) * unnorm_m with unnorm_k = (res-1)/res, unnorm_m = out_res - 1; points_out (N, P, 2) or NULL
 *     receives the looked-up coordinates.  C <= 3.
 * ---------------------------------------------------------------------------------------------- */
GG_API int64_t gg_nn_argmin_workspace(int64_t N, int64_t P);
GG_API int gg_nn_argmin(int64_t* index, void* workspace, const float* grid, const float* points, int64_t N, int64_t P, int HW,
                        void* stream);
/* Dense point tracking of the congealing animation: vis_correspondence.py:59-114 (pad_grid + nearest_neighbor_within_patch)
 * looped over frames as smoothly_sample_image (:183-205) does, one launch for all T frames (no Unfold tensor).
 * Frame t searches the patch x patch window around each point's centre of pad_grid(lerp(base, target, alphas[t])) -- the
 * (H+2) x (W+2) grid with the linear-extrapolation ring; window positions beyond it are Unfold's (0, 0) zero padding and
 * stay candidates -- with the expanded distance |p|^2 + |g|^2 - 2 g.p (separately rounded; first minimum in row-major
 * window order wins, and as with torch.argmin the first NaN, or the first candidate of an all-+inf window) and carries the
 * result as the next frame's centre.  The result index is flat_centre + dx + (H+2) dy,
 * unravelled over (H+2, W+2) with floor division (a window leaving the padded grid wraps around) and minus 1.
 *   track (T, N, P, 2) int64 (x, y) per frame; centers (N, P, 2) int64 IN: centres before frame 0 (each in [-1, H]; the
 *   caller validates), OUT: the last frame's result; points (N, P, 2) fp32 normalised; base / target (N, H, W, 2) fp32
 *   with H == W >= 2 (the reference indexes with grid.size(1) as the row stride); patch odd >= 1; alphas (T,) device. */
GG_API int gg_track_points_lerp(int64_t* track, int64_t* centers, const float* base, const float* target, const float* alphas,
                                const float* points, int T, int64_t N, int64_t P, int H, int W, int patch, void* stream);
GG_API int gg_splat2d_lookup_forward(float* out, float* points_out, void* workspace, const float* input, const float* grid,
                                     const float* query, const float* values, const float* sigma, int64_t N, int64_t P,
                                     int C, int H, int W, int grid_h, int grid_w, float unnorm_k, float unnorm_m,
                                     int soft_normalize, void* stream);

/* ------------------------------------------------------------------------------------------------
 * PCK-Transfer evaluation, csrc/pck.cu.
 *   gg_tv_per_sample: reference models/losses/loss.py:4-12 total_variation_loss(flow, reduce_batch=False) for a (N, H, W, 2)
 *     fp32 flow: out[n] = mean huber|d/dx| + mean huber|d/dy| of sample n.  One CTA per sample, no atomics (bitwise
 *     reproducible); H, W >= 2.
 *   gg_pck_transfer: one transfer direction of applications/pck.py:145-166 for B source -> destination pairs, i.e.
 *     ComposedSTN.transfer_points (spatial_transformer.py:159-198, :631-672, :141-157) + the PCK test, on quantities of ONE
 *     STN forward (replaces torch.inverse, the (N, H, W, P) distance tensor, argmin, unravel_index, grid_sample and ~40
 *     elementwise launches per direction):
 *       points / gt_points (B, P, 2) pixels of the S x S source / destination image; visible (B, P) 0/1 or NULL (all);
 *       thresh (B,) per-destination threshold; alphas (A,) DEVICE, 1 <= A <= 8;
 *       matrix_src (B, 2, 3) the source's similarity matrix (first STN);
 *       composed STN: delta_src (B, F, F, 2) the source's residual flow, identity (F, F, 2) the identity flow, grid_dst
 *       (B, grid_h, grid_w, 2) the destination's composed sampling grid, grid_h == grid_w == F; matrix_dst unused;
 *       similarity-only STN: delta_src = identity = grid_dst = NULL, matrix_dst (B, 2, 3) the destination's matrix.
 *     counts (A,) int64 is ACCUMULATED: counts[a] += #{(b, p): visible and |est - gt| <= alphas[a] * thresh[b]} (integer
 *     atomics: deterministic).  est_points (B, P, 2) and nn_index (B, P) (flat F x F index, composed STN) may be NULL.
 *     `workspace`: gg_pck_transfer_workspace(B, P, F) bytes (F = 0 for a similarity-only STN).  No sync, no allocation.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_tv_per_sample(float* out, const float* flow, int64_t N, int H, int W, void* stream);
GG_API int64_t gg_pck_transfer_workspace(int64_t B, int64_t P, int F);
GG_API int gg_pck_transfer(int64_t* counts, float* est_points, int64_t* nn_index, void* workspace, const float* points,
                           const float* gt_points, const float* visible, const float* thresh, const float* alphas,
                           const float* matrix_src, const float* matrix_dst, const float* delta_src, const float* identity,
                           const float* grid_dst, int64_t B, int64_t P, int A, int S, int F, int grid_h, int grid_w,
                           void* stream);

/* ------------------------------------------------------------------------------------------------
 * Laplacian pyramid blending, csrc/blend.cu: reference utils/laplacian_blending.py:56-107 (`LaplacianBlender.get_stacks` +
 * `forward`), as called by splat_points(blend_alg='laplacian' | 'laplacian_light') (utils/vis_tools/helpers.py:186-193).
 *   out = sum_{l<L-1} lerp(A_l - A_{l+1}, B_l - B_{l+1}, M_l) + lerp(A_{L-1}, B_{L-1}, M_{L-1}),
 *   G_0 = x, G_{l+1} = T_l G_l: a replicate-padded Gaussian blur with the 1-D taps of row l (applied along x, then y).
 * img0 / img1 / out / grads: (N, C, H, W) fp32 NCHW; mask / grad_mask: (N, 1, H, W) fp32 (broadcast over channels);
 * taps: DEVICE fp32 (levels-1, width), each row the normalised 1-D Gaussian of its level (NULL when levels == 1);
 * width odd, 1 <= width <= 63 (GG_ERR_BAD_ARG for even / non-positive, GG_ERR_UNSUPPORTED above 63); levels >= 1.
 * `workspace`: gg_laplacian_blend_workspace(N, C, H, W, levels, backward) bytes (0 when levels == 1, NULL allowed then).
 * Backward returns all three gradients (gather form, no atomics; bitwise reproducible).  Neither call synchronises. */
GG_API int64_t gg_laplacian_blend_workspace(int64_t N, int C, int H, int W, int levels, int backward);
GG_API int gg_laplacian_blend_forward(float* out, void* workspace, const float* img0, const float* img1, const float* mask,
                                      const float* taps, int64_t N, int C, int H, int W, int levels, int width, void* stream);
GG_API int gg_laplacian_blend_backward(float* grad_img0, float* grad_img1, float* grad_mask, void* workspace,
                                       const float* grad_out, const float* img0, const float* img1, const float* mask,
                                       const float* taps, int64_t N, int C, int H, int W, int levels, int width,
                                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training-loop bookkeeping (SURVEY.md 8(f) rank 3), csrc/optim.cu.
 *   gg_adam_ema_step: reference train.py:126-134 -- torch.optim.Adam.step() for every parameter of both optimisers and the
 *     EMA `accumulate(t_ema, t_module)` (models/__init__.py:19-24) -- as one multi-tensor pass.
 *     table: DEVICE array of rows {float* p; const float* g; float* m; float* v; float* ema (may be NULL); int64 numel;
 *     const float* lr (device scalar)}; block_tensor / block_chunk: DEVICE int arrays of `blocks` entries mapping a CTA to
 *     (table row, chunk of `chunk` elements); state: DEVICE float[3] = {step, 1 - b1^step, sqrt(1 - b2^step)} -- the call
 *     increments step first (torch's default Adam arithmetic: m, v, step_size = lr/bc1, denom = sqrt(v)/sqrt(bc2) + eps).
 *   gg_tv_loss_forward/backward: reference models/losses/loss.py:4-12 total_variation_loss(delta_flow (N, H, W, 2)),
 *     reduce_batch=True: out[0] = mean huber|d/dy| + mean huber|d/dx|; backward is gather-form (deterministic).
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_adam_ema_step(const void* table, const int* block_tensor, const int* block_chunk, int blocks, int chunk,
                            float* state, double beta1, double beta2, double eps, double ema_decay, void* stream);
GG_API int64_t gg_tv_loss_workspace(int64_t N, int H, int W);
GG_API int gg_tv_loss_forward(float* out, void* workspace, const float* flow, int64_t N, int H, int W, void* stream);
GG_API int gg_tv_loss_backward(float* grad_flow, const float* grad_out, const float* flow, int64_t N, int H, int W,
                               void* stream);

/* Equalised-learning-rate weights of a whole network in one launch: reference networks.py:121-127 (EqualConv2d) and :146-149
 * (EqualLinear) multiply `self.weight * self.scale` inside every forward (and autograd multiplies again in every backward).
 *   for each table row t:  dst_t[i] = (dst dtype) (src_t[i] * scale_t),  i < numel_t
 * table: device array of rows {const void* src; void* dst; int64 numel; float scale; int32 dtypes = src_dtype | dst_dtype << 8}
 * (32 bytes; dtypes GG_F32 / GG_BF16); CTA b handles elements [block_chunk[b]*chunk, +chunk) of tensor block_tensor[b]
 * (chunk a multiple of 4).  Forward: fp32 master weights -> scaled weights in the convolution's dtype; backward: gradients of
 * the scaled weights -> fp32 gradients of the master weights. */
GG_API int gg_scale_cast_multi(const void* table, const int* block_tensor, const int* block_chunk, int blocks, int chunk,
                               void* stream);

/* ------------------------------------------------------------------------------------------------
 * Latent-learner initialisation, csrc/pca.cu: the per-batch terms of IncrementalPCA's Gram form
 * (gangealing_b200/training/latent_learner.py; reference models/latent_learner.py:8-22).
 *   gg_batch_gram: for each of the B row blocks [batch_offsets[b], batch_offsets[b+1]) of the row-major fp32 (n, D) matrix w
 *     (DEVICE, 16-byte aligned): mean (B, D) fp64 the block's column mean (fixed summation order) and gram (B, D, D) fp64
 *     the full symmetric sum over its rows of (x - mean_b)(x - mean_b)^T, on the fp64 tensor cores (DMMA).  batch_offsets:
 *     HOST int64 array of B + 1 entries, offsets[0] >= 0, strictly increasing (GG_ERR_BAD_ARG otherwise); D a multiple of
 *     64 and at most 1024 (GG_ERR_UNSUPPORTED otherwise).  No atomics (bitwise reproducible), no sync, no allocation.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_batch_gram(double* gram, double* mean, const float* w, const int64_t* batch_offsets, int64_t B, int D,
                         void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training visuals, csrc/trainvis.cu (reference utils/vis_tools/training_vis.py, flow_vis.py).  Grids are uint8 (Hg, Wg, 3)
 * in torchvision make_grid's layout (nrow, padding, pad value 0, xmaps = min(nrow, N); N == 1: the bare image), the layout
 * gg_splat_composite_grid writes.  Arguments are validated before any device work (GG_ERR_BAD_ARG).
 *   gg_flow_image_grid: flow_to_image (flow_vis.py:106-130, flow_uv_to_colors :70-103) of flow (N, H, W, 2) fp32, 8-byte
 *     aligned, written as the grid.  u, v = flow * (H - 1); the radius maximum over the whole batch (np.max(rad), one
 *     reduction, atomicMax on the float bits: order-independent); numpy's precision as the reference runs it: float32 up
 *     to fk = (atan2(-v, -u) / pi + 1) / 2 * 54, float64 from f = fk - k0 on.  The value written is floor(255 * col): the
 *     reference's / 255, make_grid(range=(0, 1)) and * 255 + 0.5 return exactly that.  workspace: 4 bytes, 8-byte aligned.
 *   gg_image_grid: make_grid(normalize=True) with per-image ranges + images2grid (helpers.py:39-43): images (N, 3, H, W)
 *     fp32 dense; ranges (N, 2) fp32 (lo, hi), 8-byte aligned; clamp(lo, hi), sub(lo), div(max(hi - lo, 1e-5)), * 255,
 *     + 0.5, clamp(0, 255), truncation, every operation rounded on its own.  range=None, scale_each=True: each image's
 *     (min, max); a value_range: the same (lo, hi) for every image.
 *   gg_cluster_accumulate: routes congealed images to clusters (generate_cluster_congeal / real_cluster_congeal,
 *     training_vis.py:57-109).  Image n, slot s = sel[n] in [0, S): the element (c, y, x) of image n, flip s / K, head s % K
 *     is read at images + n*stride_n + (s/K)*stride_flip + (s%K)*stride_head + c*stride_c + y*stride_h + x*stride_w (so
 *     assign_fake_images_to_clusters' (2, N, K, C, H, W) output is passed as it is; a (N, C, H, W) batch with
 *     stride_flip = stride_head = 0).  It is added to sums[s % K] (K, C, H, W) fp32, counts[s % K] (K,) int64 is
 *     incremented, and while counts[s % K] < n_keep the image is copied to keep[s % K, counts[s % K]] (K, n_keep, C, H, W).
 *     Each sum element adds its images one by one in n order (no atomics): across calls, bitwise the sequential fp32 sum.
 *     sums, counts and keep carry over from call to call; the caller zeroes them first.  Entries outside [0, S) are skipped.
 * ---------------------------------------------------------------------------------------------- */
GG_API int gg_flow_image_grid(unsigned char* out, void* workspace, const float* flow, int64_t N, int H, int W, int nrow,
                              int padding, void* stream);
GG_API int gg_image_grid(unsigned char* out, const float* images, const float* ranges, int64_t N, int H, int W, int nrow,
                         int padding, void* stream);
GG_API int gg_cluster_accumulate(float* sums, int64_t* counts, float* keep, const float* images, const int64_t* sel,
                                 int64_t N, int S, int K, int C, int H, int W, int64_t stride_n, int64_t stride_flip,
                                 int64_t stride_head, int64_t stride_c, int64_t stride_h, int64_t stride_w, int n_keep,
                                 void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dataset congealing's pre-processing, csrc/letterbox.cu: prepare_data.py:53-77 border_pad followed by
 * applications/congeal_dataset.py:23-26 prepro, for a ragged batch of uint8 RGB images on the device.
 *   images: the N images packed in one buffer of images_bytes bytes, image n (h, w, 3) uint8 HWC at byte info[n].offset.
 *   out (N, 3, S, S) fp32: ((byte / 255) - 0.5) * 2, each operation rounded on its own.
 *   resize = 1: Pillow's (12.2) Image.resize(LANCZOS) of 8-bit RGB to (S, round_half_even(S*h/w)) for h <= w, else
 *     (round_half_even(S*w/h), S): separable fixed-point passes (22 fractional bits, sums from 1 << 21, clip to
 *     [0, 255]) over a uint8 intermediate, horizontal first unless h > 100 * w and nh < h, an axis that keeps its size skipped;
 *     coefficients in float64 as Pillow's precompute_coeffs.  Then np.pad(mode='edge') of the short axis by
 *     (floor((S - n) / 2), the rest).
 *   resize = 0: the edge pad only, S = max(h, w) for every image.
 *   flip: N bytes (nonzero: write the horizontal mirror of the padded square) or NULL.
 *   gg_letterbox_plan (host only, no device work): fills the derived fields of info_host[0..N) from (offset, h, w) and
 *     returns the workspace bytes through workspace_bytes_host.  gg_letterbox re-derives them from info_host and refuses
 *     a table that differs; the kernels read the same table from info (a device copy of info_host).
 *   Three launches: coefficient tables, the first pass of images that need two, then the second pass (or the copy) with
 *   the pad, the mirror and the normalisation.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int64_t offset;          /* in: byte offset of the image in `images` */
  int32_t h, w;            /* in: the image's size */
  int32_t nh, nw;          /* resized size (h, w without resize) */
  int32_t order;           /* passes: 0 none, 1 horizontal, 2 vertical, 3 horizontal then vertical, 4 vertical then
                              horizontal */
  int32_t ksize_h, ksize_v;  /* coefficients per output index of each pass (0: no such pass) */
  int32_t reserved;
  int64_t tmp_offset;      /* byte offset of the first pass's uint8 intermediate in the workspace (-1: none) */
  int64_t coef_h, coef_v;  /* int32 offsets of the coefficient tables in the workspace (-1: none): per output index
                              (first, count, ksize fixed-point weights) */
} GGLetterboxImage;

GG_API int gg_letterbox_plan(GGLetterboxImage* info_host, int64_t N, int S, int resize, int64_t images_bytes,
                             int64_t* workspace_bytes_host);
GG_API int gg_letterbox(float* out, void* workspace, int64_t workspace_bytes, const unsigned char* images,
                        int64_t images_bytes, const GGLetterboxImage* info_host, const GGLetterboxImage* info,
                        const unsigned char* flip, int64_t N, int S, int resize, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GG_B200_H_ */
