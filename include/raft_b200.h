/*
 * raft_b200.h -- C ABI of the H100-native RAFT recurrent-inference hot path.
 *
 * The reference (gonglixue/RAFT-tf) has NO native/FFI boundary: its hot path is a set of Python
 * graph-building functions called from RAFT.network_graph (networks/RAFT.py:78-109).  Each entry
 * point below replaces one of those functions (cited per symbol); the Python mirrors in
 * raft-tf_b200/networks/ keep the reference's names and signatures and call these through ctypes.
 *
 * Conventions
 *  - every function returns an int status: 0 = RB_OK, negative = error (see enum); nothing throws
 *    or aborts; rb_last_error() returns a thread-local description of the last failure;
 *  - every data pointer is a DEVICE pointer to a caller-owned, contiguous buffer unless the
 *    parameter name ends in _host; tensors are NHWC fp32 exactly like the reference's TF tensors;
 *  - `stream` is a cudaStream_t passed as void*; calls only ENQUEUE work on it -- no hidden
 *    synchronisation, no hidden allocation (scratch comes from caller buffers sized by the
 *    *_bytes queries) -- so every call except rb_update_weights_pack is CUDA-graph capturable;
 *  - `small` selects raft-small (radius 3, hidden 96, context 64) vs raft-things (4, 128, 128),
 *    mirroring args.small (networks/RAFT.py:37-40).
 */
#ifndef RAFT_B200_H_
#define RAFT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  RB_OK = 0,
  RB_ERR_BAD_SHAPE = -1,
  RB_ERR_BAD_ARG = -2,
  RB_ERR_UNSUPPORTED = -3,
  RB_ERR_CUDA = -4,
  RB_ERR_WORKSPACE = -5
};

/* Arithmetic back end for the GEMM-shaped ops (corr build, update-block convs).
 *   RB_MATH_TC       wgmma tensor cores, fp16 hi/lo split operands, 3 MMAs per product,
 *                    fp32 accumulation in registers (error ~2^-22 relative per product);
 *   RB_MATH_SIMT     the same split operands multiplied on the fp32 CUDA cores (bring-up /
 *                    cross-check path; identical buffers and epilogues);
 *   RB_MATH_TC_FP16  mixed precision at the boundary of upstream RAFT's --mixed_precision (torch autocast around fnet,
 *                    cnet and the update block; fp32 correlation and coords1 += delta):
 *                    - every conv (update block, convf1's window form, the hoisted `inp` convs, all encoder convs with
 *                      the stem and the stride-2 views, rb_conv2d / rb_conv2d_strided) is ONE wgmma per product:
 *                      fp16(a) * fp16(w), both the round-to-nearest hi plane (what autocast's cast gives), accumulated
 *                      in fp32 registers; the lo planes are not read;
 *                    - as in RB_MATH_TC: the correlation build (3 products), the lookups and the volume-free path, every
 *                      epilogue and elementwise op in fp32 (GRU gates, instance-norm apply, residuals, coords1 += delta,
 *                      mask softmax, upsampling), the instance-norm sums in fp64, every buffer layout -- epilogues still
 *                      write both planes, so a workspace stays valid when the mode changes between calls;
 *                    - combines with either semantics, the volume-free lookup and rb_frames_resize;
 *                    - deterministic like RB_MATH_TC: the same K order and split-K halves, so batched runs equal
 *                      per-sample runs and every tile configuration gives the same bits;
 *                    - not bit-identical to upstream under autocast, which keeps activations and elementwise ops in fp16
 *                      (here fp32), rounds the batch-norm conv's weights before the norm (here batch norm is folded
 *                      into the weights first) and sums in cuDNN's order.
 *                    The flow misses the 1e-3 bar of RB_MATH_TC by design: about 1e-2 max-abs against fp64 at 64x96 and
 *                    8 iterations, 1e-1 at 128x256 and 32 (DESIGN section 2).
 * On operands whose products and partial sums are exact in fp32, every back end returns the exact value of its own
 * arithmetic, whatever the tile configuration (tests/test_gpu_exact_conv.py pins this bit for bit).
 * Like the semantics, the mode is per thread and read when a kernel is launched (it may be set inside graph capture). */
enum { RB_MATH_TC = 0, RB_MATH_SIMT = 1, RB_MATH_TC_FP16 = 2 };

#define RB_NUM_LEVELS 4

int rb_version(void);
const char* rb_last_error(void);
/* Select the back end for subsequent calls on this thread (default RB_MATH_TC); other values -> RB_ERR_BAD_ARG. */
int rb_set_math_mode(int mode);
int rb_get_math_mode(void);
/* Numerics of the network for subsequent calls on this thread (default RB_SEMANTICS_REFERENCE); like the math mode it is
 * read when a kernel is launched, so it may be set inside CUDA-graph capture.  Unknown values -> RB_ERR_BAD_ARG.
 *   RB_SEMANTICS_REFERENCE  the TF port: truncating / clamping lookup, TF 'SAME' pads on stride-2 convs;
 *   RB_SEMANTICS_UPSTREAM   princeton-vl RAFT (PyTorch): the lookup is bilinear_sampler + F.grid_sample(align_corners=True,
 *                           padding_mode="zeros"), stride-2 convs pad k / 2 before.  It applies to rb_corr_lookup,
 *                           rb_update_lookup, rb_raft_iterate, rb_corr_otf_lookup, rb_update_lookup_otf, rb_encoder_forward and
 *                           rb_conv2d_strided.  The lookups need every pyramid level to be at least 2 x 2 (grid h, w >= 16)
 *                           and return RB_ERR_BAD_SHAPE before any CUDA call otherwise.
 * Upstream lookup, per tap at level l (W_l x H_l), each step rounded to fp32 on its own:
 *   x = c.x / 2^l + dx;  g = 2x / (W_l - 1) - 1;  ix = ((g + 1) * 0.5) * (W_l - 1);  ix = -100 unless |ix| <= 2^24 (NaN too);
 *   x0 = floor(ix), x1 = x0 + 1 (unclamped), the same for y;  nw = (x1 - ix)(y1 - iy), ne = (ix - x0)(y1 - iy),
 *   sw = (x1 - ix)(iy - y0), se = (ix - x0)(iy - y0);  a corner outside the level reads 0;
 *   out = fma(I_se, se, fma(I_sw, sw, fma(I_ne, ne, I_nw * nw))). */
enum { RB_SEMANTICS_REFERENCE = 0, RB_SEMANTICS_UPSTREAM = 1 };
int rb_set_semantics(int semantics);
int rb_get_semantics(void);
/* Device selection.  The library carries its own CUDA runtime instance; its per-thread current device does not follow the
 * host framework's (torch.cuda.device(...), cudaSetDevice in another runtime).  Call this when the calling thread switches
 * GPUs, before the calls that enqueue work (their stream argument 0 = "default stream of the current device").
 * One process per GPU (torchrun) never needs it. */
int rb_set_device(int device);
/* Number of kernels this library has launched on the calling thread since the last reset. */
long long rb_launch_count(void);
void rb_launch_count_reset(void);

/* Profiling aid: when buf != NULL, rb_update_step records 8 globaltimer timestamps per CTA of each of its
 * tensor-core convs into buf (int64[n_convs][4096][8], launch order); NULL switches it off. */
int rb_debug_set_buffer(void* buf);
/* Test hook: every later tensor-core conv on this thread uses the given configuration; 0 = automatic.
 * block_n in {16,32,64,96,128} (not applied to convs whose automatic width is 16, i.e. the split-K flow-head conv),
 * bw_log2 in [3,7] (pixel box 2^bw_log2 x 2^(7-bw_log2)), max_ctas >= 1 caps the persistent grid (on top of any
 * internal cta_limit), stages in [2, ring maximum of that width] (5/5/4/3/3 for 16/32/64/96/128; 6 for every width of the
 * single-pass kernel when the thread's math mode is RB_MATH_TC_FP16 at the time of this call; with block_n = 0 the request
 * is clamped to the ring of the width each conv picks).  Anything else -> RB_ERR_BAD_ARG, before any CUDA call.
 * Workspace sizes that depend on the pixel box (rb_encoder_workspace_bytes) must be queried under the same override. */
int rb_debug_conv_override(int block_n, int bw_log2, int max_ctas, int stages);
/* Configuration of the last tensor-core conv launched on this thread (for tests to assert coverage): tile width, pixel
 * box, CTAs launched, ring depth, 128-pixel x block_n tiles.  Returns the number of tensor-core convs since the last
 * rb_debug_conv_override() call that produced fused instance-norm statistics in their epilogue (an encoder conv whose
 * statistics fall back to the stand-alone pass is not counted), or RB_ERR_BAD_ARG if no conv has been launched. */
int rb_debug_conv_last(int* block_n, int* bw_log2, int* grid, int* stages, int* total_tiles);
/* wgmma per product of that conv: 3 (split operands) or 1 (the single-pass kernel of RB_MATH_TC_FP16); RB_ERR_BAD_ARG if
 * no conv has been launched on this thread. */
int rb_debug_conv_last_passes(void);
/* Test hook: the halo A operand of the tensor-core conv (one activation box of (box rows + kh - 1) rows per channel chunk
 * and kx, feeding all kh vertical taps).  mode -1: no conv uses it; 0 (default): the update-block convs that request it;
 * 1: every stride-1 conv with kh > 1 (rb_conv2d included).  Results are the same bits either way.  Anything else ->
 * RB_ERR_BAD_ARG. */
int rb_debug_conv_halo(int mode);
/* Launch log of the tensor-core convs on this thread since the last rb_debug_conv_override() call (the first 64):
 * rec[10] of launch i = {block_n, bw_log2, grid, stages (B ring depth with the halo), total_tiles, halo box rows (0: one A
 * box per tap), kh, kw, 64-channel chunks multiplied per tile, wgmma per product}.  Returns the number of launches logged,
 * or RB_ERR_BAD_ARG if i is not one of them. */
int rb_debug_conv_log(int i, int* rec);

/* ---- A4: coords_grid(batch, ht, wd)  networks/utils.py:4-11 ----------------------------------
 * coords[b,y,x,0] = x, coords[b,y,x,1] = y. */
int rb_coords_grid(float* coords, int B, int h, int w, void* stream);
/* F10 warm start (upstream RAFT.forward's flow_init): coords1 [B,h,w,2] = coords_grid + flow_init, one fp32 add per
 * element (upstream's coords1 = coords1 + flow_init); a NULL flow_init gives the bits of rb_coords_grid.
 * rb_coords_to_flow: flow_low [B,h,w,2] = coords1 - coords_grid in fp32 (upstream's coords1 - coords0).  Null pointers
 * (coords1, flow_low), B/h/w <= 0 and B*h*w >= 2^31 -> RB_ERR_* before any CUDA call. */
int rb_coords_init(float* coords1, const float* flow_init, int B, int h, int w, void* stream);
int rb_coords_to_flow(const float* coords1, float* flow_low, int B, int h, int w, void* stream);

/* ---- A1: GetCorrPyramid(fmap1, fmap2, num_levels=4)  networks/model_utils.py:199-221 ----------
 * pyramid layout: level l (dims h_l = h >> l, w_l = w >> l, floor) is a dense fp32 array
 * [B*h*w, h_l, w_l]; levels are concatenated, level l starting at rb_corr_level_offset(). */
int rb_corr_pyramid_bytes(int B, int h, int w, size_t* bytes);
int rb_corr_level_offset(int B, int h, int w, int level, size_t* offset_floats, int* hl, int* wl);
int rb_corr_workspace_bytes(int B, int h, int w, int C, size_t* bytes);
int rb_corr_build(const float* fmap1, const float* fmap2, float* pyramid, int B, int h, int w,
                  int C, void* workspace, size_t workspace_bytes, void* stream);

/* ---- A2/A3: SampleCorr(corr_pyramid, coords, num_levels=4, radius)  model_utils.py:224-249 ----
 * with bilinear_sampler / tf_grid_sample semantics of networks/utils.py:39-103 (truncation toward
 * zero, index clamping, weights from the clamped x1/y1).  out: [B,h,w,4*(2r+1)^2] fp32, channel =
 * level*(2r+1)^2 + (x_off+r)*(2r+1) + (y_off+r).
 * Coordinates: any fp32 value is accepted.  Finite coordinates with |c| < 2^62 are bit-exact with the reference sampler
 * and its 64-bit truncation (far right x0 = x1 = W_l - 1, far left x0 = x1 = 0, weights from the clamped x1/y1).  Beyond
 * that and for +-inf / NaN the values are unspecified, but no memory outside the level is read, and rb_corr_lookup and
 * rb_corr_otf_lookup (on a pyramid whose entries equal its dot products) give the same values.  Under
 * RB_SEMANTICS_UPSTREAM every coordinate, non-finite ones included, follows the rule above (ix = -100).  The same holds
 * for rb_update_lookup, rb_update_lookup_otf, rb_raft_iterate and rb_bilinear_sample (reference semantics only). */
int rb_corr_lookup(const float* pyramid, const float* coords, float* out, int B, int h, int w,
                   int radius, void* stream);

/* ---- A3 (general form): bilinear_sampler(img, coords)  networks/utils.py:101-103 ---------------
 * img [n,H,W,1], coords [n,S,2] (x,y in pixels) -> out [n,S]; tf_grid_sample semantics (:39-99). */
int rb_bilinear_sample(const float* img, const float* coords, float* out, int n, int H, int W, int S,
                       void* stream);

/* ---- A14: tensorpack Conv2D(stride 1, padding 'same', use_bias) on fp32 NHWC tensors -----------
 * x [B,h,w,cin], W_host HWIO [kh,kw,cin,cout] and b_host [cout] (host pointers; b_host nullable),
 * y [B,h,w,cout] = act(conv(x,W)+b), act = ReLU if relu != 0.  Synchronises the stream once to upload
 * the packed kernel (stand-alone / test entry; the update block keeps its weights resident). */
int rb_conv2d_workspace_bytes(int B, int h, int w, int cin, int cout, int kh, int kw, size_t* bytes);
int rb_conv2d(const float* x, const float* W_host, const float* b_host, float* y, int B, int h, int w,
              int cin, int cout, int kh, int kw, int relu, void* workspace, size_t workspace_bytes,
              void* stream);
/* Same with tensorpack's `strides` argument (1 or 2; the encoders' stride-2 layers, model_utils.py:21,39,68,92):
 * y [B, ceil(h/stride), ceil(w/stride), cout], TensorFlow 'SAME' padding (pad before = total / 2, the odd one after), or
 * PyTorch's pad before = k / 2 under RB_SEMANTICS_UPSTREAM.
 * The strided taps are read through TMA element strides -- no gathered copy of the input.  Same workspace query. */
int rb_conv2d_strided(const float* x, const float* W_host, const float* b_host, float* y, int B, int h, int w,
                      int cin, int cout, int kh, int kw, int stride, int relu, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ---- A5-A11: BasicUpdateBlock / SmallUpdateBlock  model_utils.py:110-194 ----------------------
 * Weights: rb_update_num_convs(small) convolutions in the fixed order given by
 * rb_update_conv_name(small, i) (reference variable scopes, e.g. "update_block/gru/convz1");
 * W_host[i] is the HWIO fp32 kernel [kh,kw,cin,cout], b_host[i] the bias [cout] (host pointers,
 * as loaded from the reference's .npz).  The packed blob is device memory owned by the caller. */
int rb_update_num_convs(int small);
const char* rb_update_conv_name(int small, int i);
int rb_update_conv_shape(int small, int i, int* kh, int* kw, int* cin, int* cout);
int rb_update_weights_bytes(int small, size_t* bytes);
int rb_update_weights_pack(int small, const float* const* W_host, const float* const* b_host,
                           void* blob, size_t blob_bytes, void* stream);
/* Host-only forms (no GPU needed): the same blob written to host memory, and where packed conv `id` lives inside it
 * (id 0..11: convc1, convc2, convf2, motion-encoder conv, convz|r 1, convq1, convz|r 2, convq2, flow-head conv1, conv2, mask
 * conv0, conv2; 100: the tensor-core form of convf1).  Planes are [cout_pad][kh*kw][cin_pad] fp16 (hi, lo) + fp32 bias. */
int rb_update_weights_pack_host(int small, const float* const* W_host, const float* const* b_host, void* host_blob,
                                size_t blob_bytes);
int rb_update_packed_conv(int small, int id, size_t* hi_off, size_t* lo_off, size_t* bias_off, int* kh, int* kw,
                          int* cin_pad, int* cout, int* cout_pad);

/* Workspace holding the recurrent state (net), the context features (inp) and every per-iteration
 * activation.  Must be zero-filled by the caller once before first use (cudaMemset). */
int rb_update_workspace_bytes(int small, int B, int h, int w, size_t* bytes);
/* net = tanh(cnet[..., :hidden]) and inp = relu(cnet[..., hidden:]) (RAFT.py:85-87) are supplied
 * already activated: net [B,h,w,hidden], inp [B,h,w,context].  `weights` is the packed blob: the
 * iteration-invariant contribution of `inp` to the GRU convolutions is computed here, once per pair. */
int rb_update_set_state(int small, const void* weights, void* workspace, const float* net,
                        const float* inp, int B, int h, int w, void* stream);
/* Same from the raw context-encoder output cnet [B,h,w,hidden+context]: applies the split, tanh and relu of
 * RAFT.py:85-87 itself. */
int rb_update_set_state_cnet(int small, const void* weights, void* workspace, const float* cnet,
                             int B, int h, int w, void* stream);
int rb_update_get_net(int small, const void* workspace, float* net, int B, int h, int w,
                      void* stream);
/* Lookup written straight into the workspace in the layout the first conv consumes (fast path). */
int rb_update_lookup(int small, void* workspace, const float* pyramid, const float* coords1, int B,
                     int h, int w, void* stream);
/* Same slot filled from an fp32 [B,h,w,4*(2r+1)^2] tensor (functional BasicUpdateBlock mirror). */
int rb_update_set_corr(int small, void* workspace, const float* corr, int B, int h, int w,
                       void* stream);
/* One update-block application: flow = coords1 - coords_grid (RAFT.py:95), motion encoder, GRU,
 * flow head, coords1 += delta (RAFT.py:102).  delta_out (nullable) receives delta_flow [B,h,w,2];
 * mask_out (nullable) receives 0.25*mask [B,h,w,576] (things only; model_utils.py:180-183).
 * GRU gates: z, r = sigmoid_f and q = tanh_f (SFU ex2.approx / rcp.approx, deterministic functions of the fp32
 * pre-activation, within 3e-7 of fp64: measured on an H100 at most 1.07e-7 for sigmoid and 2.02e-7 for tanh, DESIGN section 4), and h' = fma(z, q, fl32(fl32(1 - z) * h)) with one rounding in the fma, in every math
 * mode and tile configuration (tests/test_gpu_exact_gates.py holds the gates and this combine bit for bit). */
int rb_update_step(int small, const void* weights, void* workspace, float* coords1,
                   float* delta_out, float* mask_out, int B, int h, int w, void* stream);
/* ---- A12: the loop of RAFT.network_graph (RAFT.py:91-102): iters x (lookup, update). ---------- */
int rb_raft_iterate(int small, const void* weights, void* workspace, const float* pyramid,
                    float* coords1, float* mask_out, int B, int h, int w, int iters, void* stream);

/* ---- F2 (SURVEY 8(f)): volume-free correlation -- GetCorrPyramid + SampleCorr (model_utils.py:199-249) without the
 * 4*N^2-byte volume.  Level l of the pyramid equals fmap1 . pool^l(fmap2)^T / sqrt(C) (pooling is linear), so each
 * iteration evaluates only the (2r+3) x (2r+3) entries per pixel and level that the bilinear taps can touch, as fp32
 * dot products against the pooled feature maps, and applies the same tap arithmetic as rb_corr_lookup.  Results equal
 * the materialised path up to the summation order / operand rounding of the dot products (parity is on the flow, 1e-3);
 * where those dot products are exact in fp32 (e.g. small-integer feature maps), the results are bit-identical to
 * rb_corr_lookup on the pyramid fl(fmap1 . pool^l(fmap2) / fl(sqrt C)) at every coordinate (contract at rb_corr_lookup).
 * rb_corr_otf_prepare pools fmap2 once per pair into `workspace` (levels 1..3, fp32); C = 128 or 256. */
int rb_corr_otf_workspace_bytes(int B, int h, int w, int C, size_t* bytes);
int rb_corr_otf_prepare(const float* fmap2, void* workspace, size_t workspace_bytes, int B, int h, int w, int C,
                        void* stream);
int rb_corr_otf_lookup(const float* fmap1, const float* fmap2, const void* workspace, const float* coords,
                       float* out, int B, int h, int w, int C, int radius, void* stream);
/* lookup written straight into the update workspace (the volume-free counterpart of rb_update_lookup) */
int rb_update_lookup_otf(int small, void* workspace, const float* fmap1, const float* fmap2,
                         const void* otf_workspace, const float* coords1, int B, int h, int w, int C, void* stream);

/* ---- A13: RAFT.upsample_flow (RAFT.py:119-134) and upflow8 (utils.py:105-111) ----------------
 * flow = coords1 - coords_grid is formed inside; out: [B,8h,8w,2].  Convex upsampling per fine pixel: softmax weights
 * p_k = expf(v_k - max) / sum (libm expf, the sum in tap order k = 0..8, IEEE quotient), then
 * out = fma(8 f_8, p_8, ... fma(8 f_1, p_1, fma(8 f_0, p_0, 0))) with f_k = coords1 - grid of tap k (0 outside the image);
 * tests/test_gpu_exact_gates.py holds this bit for bit on exact softmax weights. */
int rb_upsample_convex(const float* coords1, const float* mask, float* out, int B, int h, int w,
                       void* stream);
/* scale = 1.0 reproduces the reference (no x8, utils.py:110); upstream RAFT would pass 8.0. */
int rb_upflow8(const float* coords1, float* out, int B, int h, int w, float scale, void* stream);
/* Cropped forms: out is [B,out_h,out_w,2] = rows [top, top+out_h) x cols [left, left+out_w) of the 8h x 8w field
 * (frames that rb_frames_prepare padded to a multiple of 8 are cropped back by the upsampling kernel itself). */
int rb_upsample_convex_crop(const float* coords1, const float* mask, float* out, int B, int h, int w,
                            int top, int left, int out_h, int out_w, void* stream);
int rb_upflow8_crop(const float* coords1, float* out, int B, int h, int w, float scale, int top, int left,
                    int out_h, int out_w, void* stream);

/* ---- F5: forward-backward consistency of a pair of full-resolution flows (Sundaram et al. 2010; UnFlow) -------
 * Both directions in one launch.  flow_fw, flow_bw: [B,H,W,2] fp32; occ_fw, occ_bw: [B,H,W] uint8:
 * 0 = consistent, 1 = inconsistent (occluded), 2 = the flow leaves the frame.  Per pixel p = (x,y) of fw (bw alike,
 * with the flows swapped): f = s*fw(p) (s = flow_scale: 8.0 for raft-small, whose upflow8 flow is in 1/8-resolution
 * units, 1.0 for raft-things), q = p + f; 2 unless 0 <= q.x <= W-1 and 0 <= q.y <= H-1 (a NaN gives 2); b = s times
 * the bilinear sample of bw at q (x0 = floor(q.x), x1 = min(x0+1, W-1), ax = q.x - x0, rows likewise,
 * ((1-ax)b00 + ax b01)(1-ay) + ((1-ax)b10 + ax b11)ay); 1 if |f+b|^2 > alpha1 (|f|^2 + |b|^2) + alpha2, else 0.  Every
 * operation is rounded on its own, left to right, without FMA contraction (bit-reproducible by an fp32 restatement).
 * Null pointers, B/H/W <= 0, flow_scale <= 0 or non-finite, negative or non-finite alphas -> RB_ERR_* before any CUDA
 * call.  UnFlow's constants are alpha1 = 0.01, alpha2 = 0.5. */
int rb_flow_fb_check(const float* flow_fw, const float* flow_bw, uint8_t* occ_fw, uint8_t* occ_bw,
                     int B, int H, int W, float flow_scale, float alpha1, float alpha2, void* stream);

/* ---- F16: point tracking -- consecutive flows chained per point, with the F5 test at every step -------------------
 * flow_fw, flow_bw: [T,H,W,2] fp32 in pair order (flow_fw[k] frame k -> k+1, flow_bw[k] k+1 -> k, as
 * forward_sequence_bidirectional returns them); the first n_steps (1 <= n_steps <= T) pairs are used.  N queries:
 * qframe [N] int32 (a global frame index) and qpos [N,2] fp32 (x, y in the flows' pixels); first_frame is the global
 * index of flow frame 0.  pos [N,2] fp32 and state [N] uint8 carry a query across calls: read for a query with
 * qframe < first_frame, and always written with the last row.  Outputs, frame-major: tracks [n_steps+1,N,2] fp32 and
 * status [n_steps+1,N] uint8, row j = frame first_frame + j.  Status: 0 consistent, 1 inconsistent (occluded), 2 left
 * the frame, 3 before the query frame.  Rows before qframe are (NaN, NaN) with 3; the row of qframe is qpos with 0; a
 * query with qframe < first_frame has row 0 = (pos, state).  Each step k -> k+1 from a position q with status 0 or 1:
 * f = s * (bilinear sample of flow_fw[k] at q), the sample and its arithmetic those of rb_flow_fb_check (s = flow_scale);
 * q' = q + f; status 2 and position NaN unless q' is inside [0, W-1] x [0, H-1] (NaN counts as outside), and status 2
 * is final; otherwise b = s * (sample of flow_bw[k] at q'), status 1 if |f+b|^2 > alpha1 (|f|^2 + |b|^2) + alpha2 else
 * 0, position q'.  Status 1 is not final: the position keeps integrating.  A qpos outside the frame leaves it at the
 * first step.  Every operation is rounded on its own, left to right (bit-reproducible by an fp32 restatement), and
 * each query is computed alone: its rows do not depend on N, the other queries or how a clip is split into calls.
 * Null pointers, T/H/W/N <= 0, n_steps outside [1, T], flow_scale <= 0 or non-finite, negative or non-finite alphas
 * -> RB_ERR_* before any CUDA call. */
int rb_track_points(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps, float flow_scale,
                    float alpha1, float alpha2, const int32_t* qframe, const float* qpos, int N, int first_frame,
                    float* pos, uint8_t* state, float* tracks, uint8_t* status, void* stream);

/* ---- F17: point tracking backward in time -- F16 from the query frame down to frame first_frame -------------------
 * Arguments, checks and outputs as rb_track_points (row j = frame first_frame + j, q0 = qframe - first_frame); the rows
 * run from n_steps down to 0.  0 <= q0 <= n_steps: row q0 = qpos with status 0.  Rows after the query frame (j > q0)
 * are not stored, so a launch after rb_track_points on the same tracks / status completes them in place and leaves the
 * rows at and after the query frame as the forward launch wrote them.  q0 > n_steps (the query frame lies in a later call
 * of a reverse sweep): row n_steps = the carried (pos, state), and the point goes on from there.  q0 < 0 (the query frame
 * lies in an earlier call's frames): nothing is stored and pos / state are left as they are.  Each step k+1 -> k from a
 * position q with status 0 or 1 is rb_track_points' step with the flows' roles swapped at pair k: f = s * (sample of
 * flow_bw[k] at q), q' = q + f, status 2 and NaN unless q' is inside the frame (final), else b = s * (sample of
 * flow_fw[k] at q') and the same test of f and b.  After the rows, pos / state = row 0 for every query with q0 >= 0.  On
 * the clip reversed (fw'[k] = flow_bw[T-1-k], bw'[k] = flow_fw[T-1-k]) this is rb_track_points from query frame T - q
 * with its rows reversed, on the rows up to q, bit for bit.  One thread per query, no atomics, every operation rounded on
 * its own left to right. */
int rb_track_points_backward(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps,
                             float flow_scale, float alpha1, float alpha2, const int32_t* qframe, const float* qpos, int N,
                             int first_frame, float* pos, uint8_t* state, float* tracks, uint8_t* status, void* stream);

/* ---- F18: flow accumulation -- per pixel of every frame, the displacement back to a keyframe ---------------------
 * flow_fw, flow_bw: [T,H,W,2] fp32 as for rb_track_points (flow_fw[j] frame j -> j+1, flow_bw[j] j+1 -> j); the first
 * n_steps (1 <= n_steps <= T) pairs are used.  acc [n_steps+1,H,W,2] fp32: row r holds, per pixel of frame r, the
 * displacement to the keyframe; status [n_steps+1,H,W] uint8: 0 consistent at every step back to the keyframe, 1
 * inconsistent (occluded) at some step, 2 entered through the frame edge at some step (the larger value wins).  Row
 * `start` (0 <= start <= n_steps) is the input state (zeros for the keyframe; the previous pass's last row for a later
 * pass).  rb_flow_accumulate writes rows start+1 .. n_steps, rb_flow_accumulate_backward rows start-1 .. 0; no other
 * row is touched.  Forward step r-1 -> r at pixel p = (x, y), s = flow_scale:
 *   f = s * flow_bw[r-1][p], q = p + f (rb_flow_fb_check's f and q);
 *   q inside [0, W-1] x [0, H-1]: d = f, step = the F5 test of f and s * (bilinear sample of flow_fw[r-1] at q);
 *   otherwise: qc = q clamped into the frame (fminf / fmaxf: NaN -> 0; replicate border), d = qc - p, step = 2;
 *   acc[r][p] = d + (bilinear sample of acc[r-1] at qc, no scale), componentwise;
 *   status[r][p] = max(step, status[r-1] at qc's nearest tap: x1 if ax > 0.5 else x0, rows likewise).
 * The backward entry is the mirror (step r+1 -> r: f from flow_fw[r], the test against flow_bw[r], row r+1 sampled):
 * on the clip reversed (fw'[k] = flow_bw[T-1-k], bw'[k] = flow_fw[T-1-k]) it is the forward entry bit for bit.  Every
 * operation is rounded on its own, left to right; one launch per step on the stream, no atomics, no allocation.  Null
 * pointers, T/H/W <= 0, H*W >= 2^31, n_steps outside [1, T], start outside [0, n_steps], flow_scale <= 0 or non-finite,
 * negative or non-finite alphas -> RB_ERR_* before any CUDA call. */
int rb_flow_accumulate(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps, float flow_scale,
                       float alpha1, float alpha2, int start, float* acc, uint8_t* status, void* stream);
int rb_flow_accumulate_backward(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps,
                                float flow_scale, float alpha1, float alpha2, int start, float* acc, uint8_t* status,
                                void* stream);

/* ---- F19: label propagation -- the keyframe's labels pulled along F18's displacements -----------------------------
 * acc [n,H,W,2] fp32 and status [n,H,W] uint8 (F18's rows) at the network size; key [Hs,Ws] uint8 the keyframe's label
 * map at the frames' own size; labels, status_out [n,Hs,Ws] uint8.  Per output pixel p = (x, y) of row i:
 *   A' = rb_flow_resize's value of acc[i] at p (cv2's float bilinear resize, a copy when H x W = Hs x Ws, then
 *        u *= fl32(Ws / W), v *= fl32(Hs / H));
 *   o  = p + A', clamped into [0, Ws-1] x [0, Hs-1];
 *   status_out = status[i] at the network pixel holding p's centre (rb_frame_synthesize_*_resized's `nearest`), 2 if
 *        the clamp moved o (or o is NaN);
 *   labels = the vote of o's four bilinear taps of key (x0 = floor(o.x), x1 = min(x0+1, Ws-1), ax = o.x - x0, rows
 *        likewise) with weights (1-ax)(1-ay), ax(1-ay), (1-ax)ay, ax ay: each distinct label scores the sum of its taps'
 *        weights in tap order 00, 01, 10, 11, the largest score wins and a tie goes to the smaller label.
 * Labels never blend into ids that do not exist, an integer displacement copies exactly, and a zero row reproduces key.
 * One thread per output pixel, blockIdx.y over the rows; no allocation.  Null pointers, n/H/W/Hs/Ws <= 0 and Hs*Ws >=
 * 2^32 -> RB_ERR_* before any CUDA call. */
int rb_labels_propagate(const float* acc, const uint8_t* status, int n, int H, int W, const uint8_t* key, int Hs, int Ws,
                        uint8_t* labels, uint8_t* status_out, void* stream);

/* ---- F21: several keyframes -- each frame's labels voted between the keyframes on either side of it ---------------
 * acc_a / acc_b [n,H,W,2] fp32 and status_a / status_b [n,H,W] uint8: row i's displacement to the keyframe before it
 * (side A, F18's forward chain) and to the keyframe after it (side B, F18's backward chain) at the network size; keys
 * [m,Hs,Ws] uint8 the keyframes' label maps at the frames' own size; rows [n,4] int32 in device memory, 16-byte aligned,
 * per row (slot_a, slot_b, w_a, w_b): the key of each side, -1 for an absent side, and the two sides' integer weights;
 * labels, status_out [n,Hs,Ws] uint8.  The C entry cannot read the device table: the kernel treats any slot outside
 * [-1, m) as absent too, so a bad table is memory-safe.  Per output pixel p of row i and per present side, exactly
 * rb_labels_propagate's work on that side's row and key: A' (rb_flow_resize's value), o = p + A' clamped, S = 2 if the
 * clamp moved o else the side's status at the network pixel holding p's centre, and o's four taps with the bilinear
 * weights (1-ax)(1-ay), ax(1-ay), (1-ax)ay, ax ay.  Then:
 *   voters  = the present sides whose S is the smallest (0 consistent beats 1 occluded beats 2 entered at the edge);
 *   one     : the vote of its four taps with its plain weights -- rb_labels_propagate's labels and status, bit for bit;
 *   two     : side A's weights times fl32(w_a), side B's times fl32(w_b) (each product rounded on its own), the eight
 *             candidates A00 A01 A10 A11 B00 B01 B10 B11 each score the sum, left to right, of the weights of the
 *             candidates carrying its label; the largest score wins, a tie goes to the smaller label;
 *   status_out = the smallest S; no present side: label 0, status 3.
 * raft_b200.video.keyframe_rows builds the table: w_a = K_j - t and w_b = t - K_i for frame t between keys K_i and
 * K_j, so the nearer key weighs more, and labels never blend into ids that do not exist.  Every operation is rounded on
 * its own, no FMA contraction.  One thread per output pixel, blockIdx.y over the rows; no allocation.  Null pointers, a
 * misaligned table, n/H/W/m/Hs/Ws <= 0 and Hs*Ws >= 2^32 -> RB_ERR_* before any CUDA call. */
int rb_labels_propagate_keys(const float* acc_a, const uint8_t* status_a, const float* acc_b, const uint8_t* status_b,
                             const int32_t* rows, int n, int H, int W, const uint8_t* keys, int m, int Hs, int Ws,
                             uint8_t* labels, uint8_t* status_out, void* stream);

/* ---- F22: global motion -- a robust similarity fit of each frame pair's camera motion to its flow -----------------
 * flow_fw [B,Hn,Wn,2] fp32 on the network grid and occ_fw [B,Hn,Wn] uint8 (rb_flow_fb_check's masks) of B pairs whose
 * frames are Hs x Ws.  In the frames' own pixels, centred on ((Ws-1)/2, (Hs-1)/2): network pixel (i, j) is the point
 * p = ((j+0.5) Ws/Wn - 0.5, (i+0.5) Hs/Hn - 0.5) - centre (cv2's pixel-centre rule) and its target q = p + flow_scale
 * (u Ws/Wn, v Hs/Hn).  The similarity M = [[a, -b, tx], [b, a, ty]] (frame k -> frame k+1) is fitted by weighted least
 * squares from the 8 sums (RB_MOTION_SUMS, in this order) S = sum w, sum w px, sum w py, sum w |p|^2,
 * sum w (px qx + py qy), sum w (px qy - py qx), sum w qx, sum w qy, solved in fp64 in closed form:
 *   a = (U S - X Qx - Y Qy) / D,  b = (V S - X Qy + Y Qx) / D,  D = P S - X^2 - Y^2,
 *   tx = (Qx - a X + b Y) / S,    ty = (Qy - b X - a Y) / S.
 * Round 0 weighs a pixel by 1 where occ == 0 and the flow is finite, else 0; rounds 1..rounds by that times the Cauchy
 * weight 1 / (1 + (r / cauchy_c)^2), r = |M p - q| of the previous round in network pixels (x divided by Ws/Wn, y by
 * Hs/Hn).  Outputs: params [B,4] fp64 (a, b, tx, ty); weight [B] fp64, round 0's S / (Hn Wn); flags [B] uint8, 1 for an
 * unreliable pair -- weight below min_weight, or a singular system in any round (S = 0 or D <= 1e-9 P S) -- which gets
 * the identity (1, 0, 0, 0); sums (nullable) [B,8] fp64, the last round's sums.  Per round, a chunk launch reduces
 * fixed 4096-pixel chunks of each pair in fp64 in a fixed tree into the workspace (rb_global_motion_workspace_bytes) and
 * a per-pair launch adds them in a fixed order and solves; the rounds stay on the device (no synchronisation), the
 * chunking depends on Hn x Wn only, so a pair's bits depend neither on B nor on its place in the batch; no allocation,
 * no atomics.  Null pointers, B/Hn/Wn/Hs/Ws <= 0, B > 65535, flow_scale or cauchy_c <= 0 or non-finite, rounds outside
 * [0, RB_MOTION_MAX_ROUNDS], min_weight outside [0, 1] and a workspace that is too small -> RB_ERR_* before any CUDA
 * call. */
#define RB_MOTION_SUMS 8
#define RB_MOTION_MAX_ROUNDS 32
int rb_global_motion_workspace_bytes(int B, int Hn, int Wn, size_t* bytes);
int rb_global_motion(const float* flow_fw, const uint8_t* occ_fw, int B, int Hn, int Wn, int Hs, int Ws, float flow_scale,
                     int rounds, double cauchy_c, double min_weight, double* params, double* weight, uint8_t* flags,
                     double* sums, void* workspace, size_t workspace_bytes, void* stream);

/* ---- F23: affine warp of uint8 frames -- the stabilized frames at their own size ----------------------------------
 * frames, out: [F,H,W,C] uint8 (C in [1, 4], any channel order), out not aliasing frames; A: [F,2,3] fp64 in device
 * memory, per frame the matrix from an output pixel (x, y) (uncentred, integer) to its source position:
 *   sx = fl64(fl64(A00 x) + fl64(A01 y)) + A02,  sy likewise with row 1 (each operation rounded on its own, no FMA),
 * rounded once to fp32, clamped into [0, W-1] x [0, H-1] (the border replicates; NaN -> 0), and sampled per channel with
 * fb_sample.cuh's bilinear taps on the byte values as fp32 (rounded on its own), then rintf and clamped to [0, 255].
 * The identity returns the frame byte for byte.  One thread per output pixel, blockIdx.y over the frames; no
 * allocation.  Null pointers, F/H/W <= 0, F > 65535, H or W >= 2^24 and C outside [1, 4] -> RB_ERR_* before any CUDA
 * call. */
int rb_frames_warp_affine(const uint8_t* frames, const double* A, int F, int H, int W, int C, uint8_t* out, void* stream);

/* ---- F24: masked fill -- the membrane (Laplace) fill of a field inside a hole --------------------------------------
 * values [B,H,W,C] fp32 (C = 2 or 3), filled in place; hole [B,H,W] uint8, non-zero = the pixel is unknown.  Each field
 * approximates the 4-neighbour discrete Laplace equation on its hole pixels with the known pixels as Dirichlet data
 * (neighbours outside the image left out of the stencil); the known pixels keep their bits.  Method, every fp32
 * operation rounded on its own, no FMA contraction (tests/inpaint_oracle.py restates it bit for bit):
 *   pyramid  level l+1 halves level l with ceil down to 1 x 1; a coarse pixel's children are (2i,2j), (2i,2j+1),
 *            (2i+1,2j), (2i+1,2j+1) (this tap order) inside level l;
 *   mean     of values v_0, v_1, ... in order: s = 0 + v_0 + v_1 + ..., s / n, clamped by comparisons into the values'
 *            [min, max];
 *   guess    a coarse pixel is known when any child is, with the mean of its known children (0 when none); from the
 *            coarsest level to level 0 each hole pixel takes its parent's value (nearest), then RB_FILL_INIT_SWEEPS
 *            red-black Gauss-Seidel sweeps (red: x + y even, first) set each hole pixel to the mean of its neighbours
 *            up, down, left, right (omega = 1);
 *   cycles   RB_FILL_CYCLES multigrid V-cycles for the correction of level 0.  Level l >= 1's unknowns are the pixels
 *            whose children are all unknowns of level l - 1 (level 0's: the hole).  Down: the right-hand side of level
 *            l + 1 is 0 + the residuals s - n e of the four children in tap order (0 for a child outside the level or off
 *            its unknowns; s = f + the neighbours' e in order, f = 0 and e = the field on level 0), its correction e
 *            starts at 0, and RB_FILL_SMOOTH red-black sweeps e_p = s / n run on it; at 1 x 1 nothing moves.  Up: each
 *            unknown adds the cell-centred bilinear value of the coarser correction (weights 1/4, 3/4 per axis, taps
 *            clamped, ((wx0 e00 + wx1 e01) wy0) + ((wx0 e10 + wx1 e11) wy1)), then RB_FILL_SMOOTH sweeps.  On level 0
 *            the sum is clamped into the field's [min, max] of known values per channel, and the sweeps are the
 *            guess's mean sweeps.
 * Every value the fill writes lies in [min, max] of the field's known values per channel, bit for bit, and a constant
 * field stays bit for bit.  A field without a known pixel becomes zeros and flags[b] = 1 (flags nullable, [B] uint8,
 * else 0).  Levels of at most 4096 pixels run their part of each V-cycle in one CTA per field.  Deterministic, no
 * atomics, no allocation (workspace: rb_masked_fill_workspace_bytes), and a field's bits depend neither on B nor on its
 * place in the batch.  The holes must stay unchanged during the call.  Null pointers, B/H/W <= 0, C not 2 or 3,
 * B > 65535, H*W >= 2^31 and a workspace that is too small -> RB_ERR_* before any CUDA call. */
#define RB_FILL_INIT_SWEEPS 4
#define RB_FILL_CYCLES 6
#define RB_FILL_SMOOTH 3
int rb_masked_fill_workspace_bytes(int B, int H, int W, int C, size_t* bytes);
int rb_masked_fill(float* values, const uint8_t* hole, int B, int H, int W, int C, uint8_t* flags, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---- F25: object removal -- the hole masks and the temporal fill from the nearest frames that see behind a hole ----
 * rb_inpaint_masks: masks [F,Hs,Ws] uint8 (label maps at the frames' own size); select [256] uint8 in device memory,
 * non-zero = that label is removed.  hole [F,Hs,Ws] uint8 (not aliasing masks) = 1 where some pixel of the
 * (2 dilate + 1)^2 square around it (clipped to the frame) has a selected label, else 0.  hole_net [F,Hn,Wn] uint8: network
 * pixel (i, j) is 1 when any frame pixel (y, x) with floor((y + 0.5) Hn / Hs) = i and floor((x + 0.5) Wn / Ws) = j
 * (64-bit integers) is a hole; a row or column that no frame pixel maps to takes the one holding its centre,
 * floor((i + 0.5) Hs / Hn).  Null pointers, F/Hs/Ws/Hn/Wn <= 0, F > 65535, a frame of >= 2^31 pixels and dilate outside
 * [0, RB_INPAINT_MAX_DILATE] -> RB_ERR_* before any CUDA call.
 * rb_inpaint_propagate: frames [F,Hs,Ws,3] uint8 and hole [F,Hs,Ws] (rb_inpaint_masks' hole) of F consecutive frames;
 * flow_fw, flow_bw [F-1,Hn,Wn,2] fp32 (flow_fw[k] frame k -> k+1, flow_bw[k] k+1 -> k, completed inside the holes by
 * rb_masked_fill); rows [n_rows,3] int32 in device memory, row r = (t, nf, nb): frame t and the steps each side may
 * take.  Outputs colour [n_rows,Hs,Ws,3] fp32 and status [n_rows,Hs,Ws] uint8.  Per pixel p = (x, y) of row r:
 *   not a hole: colour = the frame's bytes, status 0;
 *   a hole: p0 = (fl32((x + 0.5) Wn/Ws - 0.5), fl32((y + 0.5) Hn/Hs - 0.5)) in fp64 (each operation rounded), clamped
 *     into the grid (track_queries' map).  Forward side: up to min(nf, F-1-t) steps of rb_track_points' step from p0
 *     (f = s * sample of flow_fw[k] at q, q' = q + f; the side stops when q' leaves the grid or the F5 test against
 *     s * flow_bw[k] at q' fails).  After step n the position maps back to frame pixels, o = fl32((q' + 0.5) Ws/Wn -
 *     0.5) per axis in fp64, clamped into the frame; when none of o's four bilinear taps (fb_sample.cuh's) is a hole in
 *     frame t + n, the side is found at distance n_f = n with colour c_f = the bilinear sample of frame t + n's bytes at
 *     o.  Backward side: the mirror (flow_bw[k] pulls, flow_fw[k] tests, k = t - n, up to min(nb, t) steps) -- on the
 *     reversed clip it is the forward side, bit for bit.
 *     Both found: colour = fl32(fl32(n_b c_f) + fl32(n_f c_b)) / (n_f + n_b) per channel, status 1; one: its colour,
 *     status 2; none: colour 0, status 3 (left for the spatial fill).
 * A row whose t lies outside [0, F) is absent (colour 0, status 3) and nf / nb are clamped into the clip, so a bad table
 * reads nothing out of bounds.  Every fp32 operation is rounded on its own.  One thread per frame pixel, blockIdx.y over
 * the rows; no allocation.  Null pointers (the flows may be null when F = 1), F/Hs/Ws/Hn/Wn/n_rows <= 0, a frame of
 * >= 2^31 pixels, flow_scale <= 0 or non-finite and negative or non-finite alphas -> RB_ERR_* before any CUDA call. */
#define RB_INPAINT_MAX_DILATE 32
int rb_inpaint_masks(const uint8_t* masks, const uint8_t* select, int F, int Hs, int Ws, int dilate, int Hn, int Wn,
                     uint8_t* hole, uint8_t* hole_net, void* stream);
int rb_inpaint_propagate(const uint8_t* frames, const uint8_t* hole, int F, int Hs, int Ws, const float* flow_fw,
                         const float* flow_bw, int Hn, int Wn, float flow_scale, float alpha1, float alpha2,
                         const int32_t* rows, int n_rows, float* colour, uint8_t* status, void* stream);

/* ---- F26: full-frame stabilization -- flows extended past the frame edge, and the borders filled from other frames ---
 * Geometry: B flows [B,Hn,Wn,2] fp32 on the network grid of Hs x Ws frames, extended by my, mx >= 0 network pixels per
 * side onto the canvas Hc x Wc = (Hn + 2 my) x (Wn + 2 mx); canvas pixel (i, j) is network position (x, y) =
 * (j - mx, i - my).  motions [B,4] fp64 in device memory, per field the similarity (a, b, tx, ty) of F22 (for a
 * backward flow the inverse of the pair's, computed by the caller).  The global flow at (x, y), in fp64 with every
 * operation rounded on its own and rounded once to fp32:
 *   px = ((x + 0.5) Ws/Wn - 0.5) - (Ws-1)/2,  py likewise,
 *   g = ((((a px - b py) + tx) - px) / (Ws/Wn) / flow_scale,  (((b px + a py) + ty) - py) / (Hs/Hn) / flow_scale).
 * rb_flow_extend_residual: resid [B,Hc,Wc,2] fp32 = fl32(flow - g) inside the grid and 0 on the band; hole [B,Hc,Wc]
 *   uint8 = 0 inside, 1 on the band -- the input of rb_masked_fill (F24), which bends the residual, not the linear g.
 * rb_flow_extend_finish: ext [B,Hc,Wc,2] fp32 = the flow bit for bit inside the grid and fl32(resid + g) on the band;
 *   ext may alias resid.
 * One thread per canvas pixel, blockIdx.y over the fields; no allocation.  Null pointers, B/Hn/Wn/Hs/Ws <= 0, negative
 * margins, B > 65535, a canvas of >= 2^31 pixels, flow_scale <= 0 or non-finite and an output aliasing the flow ->
 * RB_ERR_* before any CUDA call.
 * rb_frames_warp_affine_fill: frames [F,Hs,Ws,3] uint8; ext_fw, ext_bw [F-1,Hc,Wc,2] fp32 (rb_flow_extend_finish's, ext_fw[k]
 * frame k -> k+1, ext_bw[k] k+1 -> k); A [n_rows,2,3] fp64 in device memory; rows [n_rows,3] int32 in device memory, row
 * r = (t, nf, nb).  Outputs colour [n_rows,Hs,Ws,3] fp32 and status [n_rows,Hs,Ws] uint8.  Per output pixel (x, y) of
 * row r, the source (sx, sy) is computed in fp64 from A[r] exactly as rb_frames_warp_affine (F23) does, then:
 *   inside: when fl32(sx), fl32(sy) lie in [0, Ws-1] x [0, Hs-1] or either is NaN, colour = F23's bilinear value of frame t
 *     before rintf, status 0 -- rounded and clamped it is rb_frames_warp_affine's byte;
 *   outside: the canvas position p = (fl32(fl64((sx + 0.5) Wn/Ws - 0.5) + mx), likewise y) (the pixel-centre rule,
 *     unclamped).  Forward side: when p lies on the canvas, up to min(nf, F-1-t) steps of rb_track_points' step on
 *     the canvas (f = flow_scale * the bilinear sample of ext_fw[k] at p, q = p + f; the side stops when q leaves the
 *     canvas or the F5 test against flow_scale * ext_bw[k] at q fails).  After step n the position maps back to frame
 *     pixels unclamped, o = fl32(((q - m) + 0.5) Ws/Wn - 0.5) per axis in fp64; the side is found at distance n_f = n
 *     at the first step where o lies in frame t + n, with colour c_f = the bilinear sample of that frame's bytes at o.
 *     Backward side: the mirror (ext_bw[k] pulls, ext_fw[k] tests, k = t - n, up to min(nb, t) steps).
 *     Both found: colour = fl32(fl32(n_b c_f) + fl32(n_f c_b)) / (n_f + n_b), status 1; one: its colour, status 2; none:
 *     colour 0, status 3 (left for the spatial fill).
 * A row whose t lies outside [0, F) is absent (colour 0, status 3) and nf / nb are clamped into the clip, as in
 * rb_inpaint_propagate.  Every operation is rounded on its own.  One thread per output pixel, blockIdx.y over the rows;
 * no allocation.  Null pointers (the flows may be null when F = 1), F/Hs/Ws/Hn/Wn/n_rows <= 0, negative margins, a
 * frame or canvas of >= 2^31 pixels, flow_scale <= 0 or non-finite and negative or non-finite alphas -> RB_ERR_* before
 * any CUDA call. */
int rb_flow_extend_residual(const float* flow, const double* motions, int B, int Hn, int Wn, int Hs, int Ws, int my,
                            int mx, float flow_scale, float* resid, uint8_t* hole, void* stream);
int rb_flow_extend_finish(const float* flow, const double* motions, int B, int Hn, int Wn, int Hs, int Ws, int my,
                          int mx, float flow_scale, const float* resid, float* ext, void* stream);
int rb_frames_warp_affine_fill(const uint8_t* frames, int F, int Hs, int Ws, const float* ext_fw, const float* ext_bw,
                               int Hn, int Wn, int my, int mx, float flow_scale, float alpha1, float alpha2,
                               const double* A, const int32_t* rows, int n_rows, float* colour, uint8_t* status,
                               void* stream);

/* ---- F27: video denoising -- each pixel merged with its patch matches along the chained flow of neighbouring frames --
 * rb_denoise_merge: frames [F,Hs,Ws,3] uint8 of F consecutive frames; flow_fw, flow_bw [F-1,Hn,Wn,2] fp32 (flow_fw[k]
 * frame k -> k+1, flow_bw[k] k+1 -> k, as for rb_inpaint_propagate); rows [n_rows,3] int32 in device memory, row r =
 * (t, nf, nb): frame t and the steps each side may take (raft_b200.inpaint.inpaint_rows' table); sigma the noise's
 * standard deviation in grey levels.  Outputs out [n_rows,Hs,Ws,3] uint8 (not aliasing frames) and support
 * [n_rows,Hs,Ws] uint8.  Per pixel p = (x, y) of row r:
 *   chain: p0 = (fl32((x + 0.5) Wn/Ws - 0.5), fl32((y + 0.5) Hn/Hs - 0.5)) in fp64 (each operation rounded), clamped into
 *     the grid.  Forward side: up to min(nf, F-1-t) steps of rb_track_points' step from p0 (f = s * sample of flow_fw[k]
 *     at q, q' = q + f; the side stops at the first step where q' leaves the grid or the F5 test against s * flow_bw[k]
 *     at q' fails).  Every passing step n is a match in frame t + n at o_n = fl32((q' + 0.5) Ws/Wn - 0.5) per axis in
 *     fp64, clamped into the frame.  Backward side: the mirror (flow_bw[k] pulls, flow_fw[k] tests, k = t - n, up to
 *     min(nb, t) steps) -- on the reversed clip it is the forward side, bit for bit.  support = the matched frames of
 *     both sides.
 *   candidates: in frame t the integer pixels p + s, in each matched frame the positions o_n + s, for the
 *     (2 RB_DENOISE_SEARCH + 1)^2 integer offsets s.  A sample at o + delta (delta integer) is the replicate-padded frame
 *     sampled there: o's bilinear weights (fb_sample.cuh's bilerp_at / bilerp1 arithmetic) on the taps x0 + delta_x,
 *     x0 + 1 + delta_x (likewise y), each clamped into the frame.  In frame t, o = p: the bytes themselves.
 *   weight: d = the mean over the (2 RB_DENOISE_PATCH + 1)^2 * 3 values of (candidate patch - frame t's patch at p)^2,
 *     summed from 0 in raster order, channel innermost, then divided by 27; x = max(d - 2 sigma^2, 0) / (RB_DENOISE_H
 *     sigma)^2 (x = 0 when the numerator is 0), w = (1 - x)^2 for x < 1, else 0 -- Tukey's biweight above the noise
 *     floor.  The centre candidate (frame t, s = 0) has d = 0 and w = 1.
 *   out = clamp(rintf(sum w c / sum w), 0, 255) per channel, c the candidate's centre sample; the sums run from 0 over
 *     frame t, then the forward matches n = 1, 2, ..., then the backward ones, each frame's offsets in raster order.
 * A row whose t lies outside [0, F) is absent (out 0, support 0); nf / nb are clamped into [0, RB_DENOISE_MAX_WINDOW] and
 * into the clip, so a bad table reads nothing out of bounds.  Every fp32 operation is rounded on its own.  One thread
 * per output pixel, blockIdx.y over the rows; no atomics, no allocation.  Null pointers (the flows may be null when
 * F = 1), F/Hs/Ws/Hn/Wn/n_rows <= 0, a frame of >= 2^31 pixels, flow_scale <= 0 or non-finite, negative or non-finite
 * alphas, sigma <= 0 or non-finite and out aliasing frames -> RB_ERR_* before any CUDA call.
 * ---- F28: the noise estimate behind sigma = "auto" ----
 * rb_noise_sums: frames [N,H,W,3] uint8; sums [N,3] int64 = sum over the interior pixels (1 <= x <= W-2, 1 <= y <= H-2)
 * of |I * M| per frame and channel, M = [[1,-2,1],[-2,4,-2],[1,-2,1]] (Immerkaer, "Fast noise variance estimation",
 * CVIU 1996).  The host takes sigma = sqrt(pi/2) S / (6 (H-2)(W-2)) per frame and channel.  Integer sums: exact and
 * deterministic with int64 atomics; one memset and one launch, no allocation.  Null pointers, N <= 0, H or W < 3,
 * N > 65535 and H*W >= 2^31 -> RB_ERR_* before any CUDA call. */
#define RB_DENOISE_SEARCH 1
#define RB_DENOISE_PATCH 1
#define RB_DENOISE_MAX_WINDOW 16
#define RB_DENOISE_H 3.0f
int rb_denoise_merge(const uint8_t* frames, int F, int Hs, int Ws, const float* flow_fw, const float* flow_bw, int Hn,
                     int Wn, float flow_scale, float alpha1, float alpha2, const int32_t* rows, int n_rows, float sigma,
                     uint8_t* out, uint8_t* support, void* stream);
int rb_noise_sums(const uint8_t* frames, int N, int H, int W, int64_t* sums, void* stream);

/* ---- F29: temporal consistency -- the per-pixel temporal term of a processed frame (Bonneel et al. 2015) ----------
 * rb_tcons_terms: frame I_t, prev_frame I_(t-1), processed P_t, prev_out O_(t-1): [Hs,Ws,3] uint8; flow_fw, flow_bw
 * [Hn,Wn,2] fp32 the pair (t-1, t) (flow_fw frame t-1 -> t, flow_bw t -> t-1); strength lambda.  Outputs c [Hs,Ws] fp32,
 * r [Hs,Ws,3] fp32 and status [Hs,Ws] uint8.  Per pixel p = (x, y), every fp32 operation rounded on its own:
 *   step: p0 = (fl32((x + 0.5) Wn/Ws - 0.5), likewise y) in fp64, clamped into the grid (fb_sample.cuh's px_remap);
 *     one step of rb_track_points' step backward: f = s * the bilinear sample of flow_bw at p0, q = p0 + f; it fails
 *     when q leaves the grid or the F5 test against s * flow_fw at q fails (status 1).  o = (fl32((q + 0.5) Ws/Wn -
 *     0.5), likewise y) in fp64, clamped into the frame -- rb_denoise_merge's first backward step, bit for bit.
 *   check: I^, O^ the bilinear samples (bilerp_at / bilerp1) of I_(t-1), O_(t-1) at o; d = (0 + e_0^2 + e_1^2 + e_2^2) / 3
 *     with e_ch = I_t(p) - I^; x = d / fl32(RB_TCONS_KAPPA^2); w = (1 - x)^2 when x < 1 (status 0), else 0 (status 2).
 *   terms: c = fl32(lambda w) + RB_TCONS_EPS; r = fl32(lambda w) (O^ - P_t(p)) per channel where status is 0, else +0.
 * prev_frame = NULL means no previous frame (frame 0, or the first frame after a scene cut): status 3, c = RB_TCONS_EPS,
 * r = 0, and only the outputs are touched.  One thread per pixel; no allocation.  Null pointers, Hs/Ws/Hn/Wn <= 0, a
 * frame of >= 2^31 pixels, flow_scale <= 0 or non-finite, negative or non-finite alphas and strength <= 0 or non-finite
 * -> RB_ERR_* before any CUDA call.  RB_TCONS_KAPPA is in grey levels, chosen on the synthetic clip of
 * tests/test_temporal.py; it is not tuned on real footage.
 * ---- F30: the screened Poisson solve of the correction D = O_t - P_t ----
 * rb_screened_poisson: c [H,W] fp32 (> 0), r [H,W,3] fp32; D [H,W,3] fp32 (not aliasing r) approximates per channel
 *   (c_p + n_p) D_p - sum_(q in N(p)) D_q = r_p,  N(p) the in-image 4-neighbours and n_p their count (Neumann boundary).
 * Method (tests/tcons_oracle.py restates it bit for bit):
 *   levels   level l+1 halves level l with ceil down to 1 x 1 (rb_masked_fill's pyramid); a coarse pixel's children are
 *            (2i,2j), (2i,2j+1), (2i+1,2j), (2i+1,2j+1) (this order) inside level l; c_(l+1) = 0 + the children's c in
 *            order.  Every level keeps the unit 4-neighbour coupling (rediscretised, not Galerkin).
 *   stencil  s = f + e_up + e_down + e_left + e_right (+0 for a neighbour outside the level), n = 0 + 1 per in-level
 *            neighbour in the same order; residual s - (n e + c e); sweep e = s / (c + n).
 *   V-cycle  V(f) from e = 0 on level 0: on each level RB_TCONS_SWEEPS red-black Gauss-Seidel sweeps (red, x + y even,
 *            first), the next level's f = 0 + the residuals of the children in order and its e = 0, down to 1 x 1 (the
 *            same sweeps there); up: each pixel adds the cell-centred bilinear value of the coarser e (weights 1/4, 3/4
 *            per axis, taps clamped, ((wxa e_aa + wxb e_ab) wya) + ((wxa e_ba + wxb e_bb) wyb)), then the sweeps.
 *   solve    flexible preconditioned conjugate gradients, per channel, from D = 0: res = r, z = V(res), p = z,
 *            rho = <res, z>; then RB_TCONS_ITERS times: q = A p, alpha = fl32(rho / <p, q>) (0 unless <p, q> > 0),
 *            D += alpha p, res' = res - alpha q, d = res' - res, res = res'; and except after the last: z = V(res),
 *            beta = fl32(<z, d> / rho) (0 unless rho > 0), rho = <res, z>, p = z + beta p.  A p = -(the residual of p
 *            with f = 0).
 *   dots     <a, b> per channel in fp64 of the exact products: blocks of 1024 pixels, thread t adds pixels t + 256 k,
 *            k = 0..3, in order from 0 (0 past the end), then the tree s[t] += s[t + h], h = 128, ..., 1; the block
 *            partials likewise by one block (thread t: partials t + 256 k in order, then the tree).
 * r = 0 gives D = 0 bit for bit.  Deterministic: no atomics and a fixed sequence of launches and device copies, 61 L + 12
 * of them at the constants below for L levels (744 for 1080 x 1920, L = 12); no allocation (workspace:
 * rb_screened_poisson_workspace_bytes, about 17 H W floats).  Null pointers, H/W <= 0, H*W >= 2^31, any overlap of D, c, r and
 * the workspace (except c with r, both read only) and a workspace that is too small -> RB_ERR_* before any CUDA call.
 * ---- F31: the warping error E_warp of a video aligned with the frames (Lai et al., ECCV 2018) ----
 * rb_warp_error: video [F,Hs,Ws,3] uint8 (F >= 2); flow_fw, flow_bw [F-1,Hn,Wn,2] fp32 of the original frames.  Per pixel
 * p of frame k < F-1: one forward step (flow_fw[k] pulls, flow_bw[k] tests; F29's map and step, mirrored); where it
 * passes, e = 0 + sum_ch (V_k(p) - V^_(k+1)(o))^2 in fp32, V^ the bilinear sample.  sums [F-1,2] fp64 = (sum e, count)
 * per pair: blocks of 4096 pixels (thread t: pixels t + 256 k, k = 0..15, in order), the fixed tree, then one block
 * per pair adds its partials in a fixed order (workspace: rb_warp_error_workspace_bytes).  The host forms E_pair =
 * sum e / (255^2 count).  Null pointers, F < 2, F - 1 > 65535, Hs/Ws/Hn/Wn <= 0, a frame of >= 2^31 pixels, bad
 * flow_scale or alphas and a workspace that is too small -> RB_ERR_* before any CUDA call. */
#define RB_TCONS_KAPPA 20.0f
#define RB_TCONS_EPS 1e-4f
#define RB_TCONS_ITERS 6
#define RB_TCONS_SWEEPS 2
int rb_tcons_terms(const uint8_t* frame, const uint8_t* prev_frame, const uint8_t* processed, const uint8_t* prev_out,
                   int Hs, int Ws, const float* flow_fw, const float* flow_bw, int Hn, int Wn, float flow_scale,
                   float alpha1, float alpha2, float strength, float* c, float* r, uint8_t* status, void* stream);
int rb_screened_poisson_workspace_bytes(int H, int W, size_t* bytes);
int rb_screened_poisson(const float* c, const float* r, int H, int W, float* D, void* workspace, size_t workspace_bytes,
                        void* stream);
int rb_warp_error_workspace_bytes(int F, int Hs, int Ws, size_t* bytes);
int rb_warp_error(const uint8_t* video, int F, int Hs, int Ws, const float* flow_fw, const float* flow_bw, int Hn,
                  int Wn, float flow_scale, float alpha1, float alpha2, double* sums, void* workspace,
                  size_t workspace_bytes, void* stream);

/* ---- F6: frame interpolation -- flow_utils.py:166-274 reverse_flow_avg_skip_static, batched, and the frame blend -----
 * rb_flow_reverse: per sample of flow01 [B,H,W,2] fp32, bit for bit with the reference under numpy >= 2:
 *  1. static(p) = every channel c has d_c < 10, d_c = uint8(bg - im0) (img_u8 = 1: wraps, like numpy's uint8) or
 *     |fl32(bg - im0)| (img_u8 = 0); bg, im0: [B,H,W,img_channels], both or neither (neither: nothing is static);
 *  2. f = fl32((static ? +inf : flow01) * time_step);
 *  3. (px, py) = (double)f + (x, y); a source with an infinite or NaN coordinate is skipped (NaN: the reference raises);
 *  4. target = (clamp(rint(px), 0, W-1), clamp(rint(py), 0, H-1)), rint rounding half to even like np.round;
 *  5. each target sums -f over its sources in fp32 from +0.0, in source raster order, and counts them;
 *  6. flow_t = fl32(sum / (double)count) where count > 0; multi = count > 1; empty = count == 0;
 *  7. each empty pixel gets the fp32 mean, summed in the order up, down, left, right from +0.0, of the nearest
 *     non-empty pixels above / below in its column and left / right in its row (+0.0 if there are none);
 *  8. empty_eroded = 5x5 minimum of empty over the window clipped to the image (cv2.erode's default border).
 * flow_t [B,H,W,2] fp32; empty, multi, empty_eroded, static_mask [B,H,W] uint8 (empty_eroded, static_mask nullable).
 * Deterministic (no float atomics): a stable radix sort orders every target's sources; a target that every source of
 * its frame hits is summed by one thread in O(H W).  The workspace (rb_flow_reverse_workspace_bytes) holds CUB's
 * temporary storage too, so the call allocates nothing and is CUDA-graph capturable.  Null pointers, only one of bg /
 * im0, non-finite time_step, B/H/W <= 0, B*H*W + 1 >= 2^32 and a workspace smaller than its fixed part -> RB_ERR_*
 * before any CUDA call (the rest of the size check queries the device). */
int rb_flow_reverse_workspace_bytes(int B, int H, int W, size_t* bytes);
int rb_flow_reverse(const float* flow01, const void* bg, const void* im0, int img_u8, int img_channels, float time_step,
                    float* flow_t, uint8_t* empty, uint8_t* multi, uint8_t* empty_eroded, uint8_t* static_mask,
                    int B, int H, int W, void* workspace, size_t workspace_bytes, void* stream);
/* rb_frame_synthesize: frames [2B,Hp,Wp,3] fp32 = [I0 | I1], read at rows [top, top+H) x cols [left, left+W);
 * flow_t0, flow_t1 [B,H,W,2] (time t -> frame 0 / frame 1, pixels), empty0, empty1 [B,H,W] uint8 (rb_flow_reverse);
 * out [B,H,W,3] fp32.  Per pixel p and frame k: q = (min(max(x + F.x, 0), W-1), likewise y; NaN -> 0), v_k = the
 * bilinear sample of I_k at q per channel (the arithmetic of rb_flow_fb_check); w0 = empty0 ? 0 : 1-t,
 * w1 = empty1 ? 0 : t, both 0 -> (1-t, t); out = (w0 v_0 + w1 v_1) / (w0 + w1).  Every operation is rounded on its own,
 * left to right, so t = 0 gives I0 and t = 1 gives I1 exactly.  t outside [0, 1], null pointers, bad shapes or a crop
 * outside the frames -> RB_ERR_* before any CUDA call. */
int rb_frame_synthesize(const float* frames, int Hp, int Wp, int top, int left, const float* flow_t0,
                        const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1, float t, float* out,
                        int B, int H, int W, void* stream);

/* ---- F13: every time step of frame interpolation in one launch (frame sequences and many t per pair) --------------
 * rb_flow_reverse_multi: the reversal of one flow01 [B,H,W,2] fp32 by n_steps time steps at once.  time_steps is a host
 * array of n_steps finite values, copied into the kernel parameters (no host-to-device copy, no allocation, CUDA-graph
 * capturable).  flow_t [n_steps,B,H,W,2] fp32, empty and multi [n_steps,B,H,W] uint8: sample (i, b) is bit for bit
 * rb_flow_reverse(flow01[b], time_steps[i]) without bg / im0 (steps 1-7 above; no static mask, no eroded mask).  The
 * n_steps * B samples share one key sort (keys up to n_steps*B*H*W) and one hole fill with n_steps*B*W column and
 * n_steps*B*H row threads.  rb_flow_reverse is the n_steps = 1 case of the same kernels.  The workspace
 * (rb_flow_reverse_multi_workspace_bytes; rb_flow_reverse_workspace_bytes is its n_steps = 1 value) holds CUB's
 * temporary storage too.  Null pointers, n_steps < 1 or > RB_INTERP_MAX_STEPS, a non-finite step, B/H/W <= 0,
 * n_steps*B*H*W + 1 >= 2^32 and a workspace smaller than its fixed part -> RB_ERR_* before any CUDA call. */
#define RB_INTERP_MAX_STEPS 64
int rb_flow_reverse_multi_workspace_bytes(int n_steps, int B, int H, int W, size_t* bytes);
int rb_flow_reverse_multi(const float* flow01, const float* time_steps, int n_steps, float* flow_t, uint8_t* empty,
                          uint8_t* multi, int B, int H, int W, void* workspace, size_t workspace_bytes, void* stream);
/* rb_frame_synthesize_pairs: rb_frame_synthesize's blend for n_t times at once, with the two frames of every pair given
 * apart: frames0, frames1 [B,Hp,Wp,3] fp32 (pair b blends frames0[b] and frames1[b]; for T consecutive pairs of T + 1
 * frames these are images[:T] and images[1:], for B independent pairs the halves of [I0 | I1]).  ts: a host array of n_t
 * times in [0, 1], copied into the kernel parameters; flow_t0, flow_t1 [n_t,B,H,W,2] and empty0, empty1 [n_t,B,H,W]
 * (rb_flow_reverse_multi's outputs for the steps t and 1 - t); out [n_t,B,H,W,3]: fp32 (out_u8 = 0), the values of
 * rb_frame_synthesize at each t, or uint8 (out_u8 = 1), each value quantised as rb_frame_metrics does,
 * min(max(rintf(fl32(255 v)), 0), 255) with NaN -> 0 -- the CLI's np.clip(np.rint(255 v), 0, 255) for every finite v.
 * bgr = 1 writes the channels in reverse order (RGB <-> BGR).  rb_frame_synthesize is this call with
 * frames1 = frames + B*Hp*Wp*3, one t and fp32 output.  Null pointers, n_t < 1 or > RB_INTERP_MAX_STEPS, out_u8 or bgr
 * not 0 / 1, a t outside [0, 1] (or NaN), bad shapes or a crop outside the frames -> RB_ERR_* before any CUDA call. */
int rb_frame_synthesize_pairs(const float* frames0, const float* frames1, int Hp, int Wp, int top, int left,
                              const float* flow_t0, const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1,
                              const float* ts, int n_t, void* out, int out_u8, int bgr, int B, int H, int W,
                              void* stream);

/* ---- F14: per-item reversal and blend (frame-rate conversion: every pair its own times) ----------------------------
 * An item is one (sample, time) of its own, so a call does only the work its items need, whatever times the other
 * samples want.  item_sample (int32) and item_step / item_t (fp32) are host arrays of n_items entries, copied into the
 * kernel parameters like rb_flow_reverse_multi's steps (no copy, no allocation, CUDA-graph capturable).  Both entries run
 * the kernels of the multi-step entries above, whose sample -> (time, row) map takes the item table instead.
 * rb_flow_reverse_items: item i reverses flow01[item_sample[i]] (flow01 [B,H,W,2] fp32) by item_step[i] into flow_t
 * [n_items,H,W,2] fp32 and empty, multi [n_items,H,W] uint8; item i is bit for bit
 * rb_flow_reverse_multi(flow01[item_sample[i]], {item_step[i]}, 1, ..., B = 1): the same keys, the same stable sort, the
 * same raster-order sums and the same hole fill, whichever other items share the call (samples may repeat and come in
 * any order).  The workspace is rb_flow_reverse_multi_workspace_bytes(n_items, 1, H, W).  Null pointers, n_items < 1 or
 * > RB_INTERP_MAX_STEPS, B/H/W <= 0, n_items*H*W + 1 >= 2^32, a sample outside [0, B), a non-finite step and a
 * workspace smaller than its fixed part -> RB_ERR_* before any CUDA call (the rest of the size check queries the
 * device).
 * rb_frame_synthesize_items: item i blends frames0[item_sample[i]] and frames1[item_sample[i]] ([B,Hp,Wp,3] fp32, crop
 * as in rb_frame_synthesize_pairs) at item_t[i] with flow_t0, flow_t1 [n_items,H,W,2] and empty0, empty1 [n_items,H,W]
 * (rb_flow_reverse_items' outputs for the steps s t and s (1 - t)) into out [n_items,H,W,3]: fp32 (out_u8 = 0) or uint8
 * (out_u8 = 1) with bgr, each item bit for bit rb_frame_synthesize_pairs of that sample at that t.  Null pointers,
 * n_items < 1 or > RB_INTERP_MAX_STEPS, out_u8 or bgr not 0 / 1, a t outside [0, 1] (or NaN), B/H/W <= 0, a sample
 * outside [0, B) and a crop outside the frames -> RB_ERR_* before any CUDA call. */
int rb_flow_reverse_items(const float* flow01, int B, const int32_t* item_sample, const float* item_step, int n_items,
                          float* flow_t, uint8_t* empty, uint8_t* multi, int H, int W, void* workspace,
                          size_t workspace_bytes, void* stream);
int rb_frame_synthesize_items(const float* frames0, const float* frames1, int Hp, int Wp, int top, int left,
                              const float* flow_t0, const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1,
                              const int32_t* item_sample, const float* item_t, int n_items, void* out, int out_u8,
                              int bgr, int B, int H, int W, void* stream);

/* ---- F16: the blend at the frames' own size from flows at the network size ----------------------------------------
 * The network runs at H x W (an engine's input_size); the frames have their own Hs x Ws.  The reversal stays at H x W
 * (flow_t0, flow_t1 [n,H,W,2] fp32 and empty0, empty1 [n,H,W] uint8 from rb_flow_reverse_multi / _items), and output
 * pixel p = (x, y) of Hs x Ws of sample i is, bit for bit,
 *   rb_frame_synthesize_*(prepare(frames0), prepare(frames1), Hs, Ws, 0, 0, resize_flow(flow_t0), resize_flow(flow_t1),
 *                         nearest(empty0), nearest(empty1), ...)
 * without any Hs x Ws fp32 intermediate, where
 *   resize_flow = rb_flow_resize(flow_t[i], Hs, Ws): cv2's float bilinear resize (copy / OpenCV / IPP as there), then
 *                 u *= fl32(Ws / W), v *= fl32(Hs / H) -- the flow in the frames' pixels;
 *   nearest     = empty[i][ys][xs], ys = ((2y+1) H) div (2 Hs), xs = ((2x+1) W) div (2 Ws) in 64-bit integers: the network
 *                 pixel whose area holds p's centre.  This is neither cv2's INTER_NEAREST nor INTER_NEAREST_EXACT (both
 *                 pick other pixels at 432x1024 -> 1080x1920);
 *   prepare     = uint8 frames (frames_u8 = 1) divided as rb_frames_prepare does (np.float32(u) / 255), fp32 frames
 *                 (frames_u8 = 0) as they are.
 * frames0, frames1 [B,Hs,Ws,3], unpadded (an engine's staging buffer of raw frames); out as rb_frame_synthesize_pairs /
 * _items at Hs x Ws, fp32 (out_u8 = 0) or quantised uint8 (out_u8 = 1, bgr = 1 reverses the channels).  Hs x Ws = H x W
 * is the existing blend bit for bit, and t = 0 with uint8 frames and uint8 output returns frames0 byte for byte.
 * One thread per output pixel; the low-resolution flows and masks are read through the read-only path, uint8 frames as
 * bytes.  No allocation, no synchronisation, graph-capturable.
 * rb_frame_synthesize_pairs_resized: ts, n_t, pair b of time i as rb_frame_synthesize_pairs; out [n_t,B,Hs,Ws,3].
 * rb_frame_synthesize_items_resized: item i blends frames0[item_sample[i]] and frames1[item_sample[i]] at item_t[i] as
 * rb_frame_synthesize_items; out [n_items,Hs,Ws,3].
 * Null pointers, frames_u8 / out_u8 / bgr not 0 or 1, n < 1 or > RB_INTERP_MAX_STEPS, a t outside [0, 1] (or NaN), a
 * sample outside [0, B), B/H/W/Hs/Ws <= 0 and Hs*Ws >= 2^32 -> RB_ERR_* before any CUDA call. */
int rb_frame_synthesize_pairs_resized(const void* frames0, const void* frames1, int frames_u8, int Hs, int Ws,
                                      const float* flow_t0, const float* flow_t1, const uint8_t* empty0,
                                      const uint8_t* empty1, int H, int W, const float* ts, int n_t, void* out,
                                      int out_u8, int bgr, int B, void* stream);
int rb_frame_synthesize_items_resized(const void* frames0, const void* frames1, int frames_u8, int Hs, int Ws,
                                      const float* flow_t0, const float* flow_t1, const uint8_t* empty0,
                                      const uint8_t* empty1, int H, int W, const int32_t* item_sample,
                                      const float* item_t, int n_items, void* out, int out_u8, int bgr, int B,
                                      void* stream);

/* ---- F32: a camera shutter for frame-rate conversion -- each output frame the mean of sub-frames over its exposure --
 * Times are in input frames (input frame i sits at time i).  Output frame n of a conversion from rate `in` to rate `out`
 * sits at s = n in/out; with shutter angle A in (0, 360] its exposure is [s - e/2, s + e/2], e = (A/360) in/out, and with
 * `density` D >= 1 samples per input-frame interval it is sampled at m = max(1, ceil(D e)) times
 * u_j = s - e/2 + (j + 1/2) e/m (the midpoint rule), each clamped into the frames [a, b] of the shot holding s (a scene
 * cut is a shot boundary; a frame inside a cut pair k belongs to the shot of raft_b200.video.cut_copy).  A non-integer
 * u_j is the item (k, t) = (floor(u_j), fl32(u_j - k)) -- rb_frame_synthesize_items' (or _items_resized') fp32 value --
 * and an integer u_j is input frame u_j as prepared (the blend's value at t = 0 exactly).  The output frame is acc / m,
 * acc the fp32 sum from +0.0 of the m values in sample order, each add rounded on its own, quantised as rb_frame_metrics
 * does: min(max(rintf(fl32(255 v)), 0), 255), NaN -> 0.  m = 1 is the conversion without a shutter byte for byte.
 * (Brooks & Barron, CVPR 2019: interpolate, then average; it is how Nah et al., CVPR 2017, made the GoPro blur.)
 *
 * rb_frame_expose_items runs a table of rows, each one output frame's run of samples, copied into the kernel parameters
 * like rb_frame_synthesize_items' items (no copy, no allocation, no atomics, CUDA-graph capturable):
 *   entries[i]  = (slot, sample, t): slot >= 0 is the blend of frames[sample] and frames[sample + 1] at t with slot
 *                 `slot` of flow_t0, flow_t1 [n_slots,H,W,2] and empty0, empty1 [n_slots,H,W] (rb_flow_reverse_items'
 *                 outputs for the steps s t and s (1 - t)); slot = RB_EXPOSE_FRAME is input frame `sample` itself;
 *   rows[r]     = (first, count, m, acc, out, flags): entries first .. first + count - 1 in order.  flags
 *                 RB_EXPOSE_OPEN starts the sum from +0.0, else from acc[acc]; RB_EXPOSE_CLOSE writes the quantised
 *                 acc / m to out[out] (bgr = 1: channels reversed), else stores the sum in acc[acc].
 * So a frame's samples may be split over calls (and over passes of a video): the fp32 sum carries through acc, and the
 * bytes do not depend on where the calls split.  One thread per (row, pixel) adds its row's entries in order.
 * frames [B+1,Hp,Wp,3] fp32 padded, read at the crop (top, left) + H x W as in rb_frame_synthesize_pairs; acc
 * [n_acc,H,W,3] fp32; out [n_out,H,W,3] uint8.  Null pointers (the flows and masks may be null when n_slots = 0, acc
 * when no row reads or stores it, out when none closes), n_entries < 1 or > RB_INTERP_MAX_STEPS, n_rows < 1 or > n_entries, bgr not 0 / 1, bad shapes or
 * crop, a row's entries outside the table or count < 1, m < 1 or > 2^24, unknown flags, an acc or out index outside
 * [0, n_acc) / [0, n_out), two rows of the call on one acc or out index, a slot outside [-1, n_slots), a sample outside
 * [0, B) (a blend) or [0, B] (a frame) and a t outside [0, 1] (or NaN) -> RB_ERR_* before any CUDA call.
 * rb_frame_expose_items_resized is the same at the frames' own Hs x Ws from flows at H x W (F16's blend, and frames as
 * there: uint8 with frames_u8 = 1, read as np.float32(u) / 255, or fp32 as they are); frames [B+1,Hs,Ws,3] unpadded, acc
 * [n_acc,Hs,Ws,3], out [n_out,Hs,Ws,3]. */
#define RB_EXPOSE_FRAME (-1)
#define RB_EXPOSE_OPEN 1
#define RB_EXPOSE_CLOSE 2
typedef struct {
  int32_t slot, sample;
  float t;
} rb_expose_entry;
typedef struct {
  int32_t first, count, m, acc, out, flags;
} rb_expose_row;
int rb_frame_expose_items(const float* frames, int Hp, int Wp, int top, int left, const float* flow_t0,
                          const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1, int n_slots,
                          const rb_expose_entry* entries, int n_entries, const rb_expose_row* rows, int n_rows,
                          float* acc, int n_acc, uint8_t* out, int n_out, int bgr, int B, int H, int W, void* stream);
int rb_frame_expose_items_resized(const void* frames, int frames_u8, int Hs, int Ws, const float* flow_t0,
                                  const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1, int H, int W,
                                  int n_slots, const rb_expose_entry* entries, int n_entries, const rb_expose_row* rows,
                                  int n_rows, float* acc, int n_acc, uint8_t* out, int n_out, int bgr, int B,
                                  void* stream);

/* ---- F34: camera homography -- a robust homography fit of each frame pair's camera motion to its flow --------------
 * flow [B,Hn,Wn,2] fp32 and occ [B,Hn,Wn] uint8 of B fields (forward or backward) whose frames are Hs x Ws; sim_params
 * [B,4] fp64 and sim_flags [B] uint8, rb_global_motion's outputs for the same fields.  Points as in F22: network pixel
 * (i, j) is p = ((j+0.5) Ws/Wn - 0.5, (i+0.5) Hs/Hn - 0.5) - ((Ws-1)/2, (Hs-1)/2) and its target q = p + flow_scale
 * (u Ws/Wn, v Hs/Hn), both divided by L = max(Ws, Hs) / 2: (x, y) and (qx, qy).  The model H = [[h1, h2, h3], [h4, h5,
 * h6], [h7, h8, 1]] maps (x, y) to pi(H (x, y, 1)), pi(X, Y, z) = (X/z, Y/z).  Each point gives the DLT rows
 * a_x = (x, y, 1, 0, 0, 0, -x qx, -y qx) with right-hand side qx and a_y = (0, 0, 0, x, y, 1, -x qy, -y qy) with qy.
 * Each of `rounds` rounds forms the 45 fp64 sums (RB_HOMOGRAPHY_SUMS, in this order) S = sum w, the upper triangle of
 * sum w (a_x a_x^T + a_y a_y^T) row by row ((0,0), (0,1), ..., (0,7), (1,1), ..., (7,7)), and the 8 entries of
 * sum w (a_x qx + a_y qy), and solves the 8 x 8 system by Cholesky in fp64 in thread 0 of the pair's block, in a fixed
 * order.  A pixel counts where occ == 0 and its flow is finite, with w = 1 / (1 + (r / cauchy_c)^2) / z^2: r = |q -
 * pi(H p)| under the previous round's H in network pixels (x scaled by Wn/Ws, y by Hn/Hs, as F22), z = h7 x + h8 y + 1
 * (the iteratively reweighted DLT); z <= 0 or a non-finite residual gives w = 0.  Round 0's previous H is the
 * similarity [[a, -b, tx/L], [b, a, ty/L], [0, 0, 1]].  The reciprocals of z and of the Cauchy term are the hardware's
 * approximate reciprocal refined by two Newton steps (within an ulp).  Outputs H [B,9] fp64 row-major in the normalised
 * coordinates (h33 = 1) and flags [B] uint8: 0 homography; 1 singular in some round (S = 0, a Cholesky pivot <= 1e-12 x
 * its diagonal entry, or a non-finite solution), the field keeps the initial similarity from then on; 2 the similarity
 * was flagged unreliable, H is the identity.  sums (nullable) [B,45] fp64, the last round's.  Reduction as F22: fixed
 * 4096-pixel chunks (a shuffle tree per warp, then the warps in order) into the workspace
 * (rb_homography_motion_workspace_bytes), then one per-pair launch that adds the chunks in order, so a field's bits
 * depend neither on B nor on its place in the batch; no allocation, no atomics.  Null pointers (sums excepted),
 * B/Hn/Wn/Hs/Ws <= 0, B > 65535, flow_scale or cauchy_c <= 0 or non-finite, rounds outside [1,
 * RB_HOMOGRAPHY_MAX_ROUNDS] and a workspace that is too small -> RB_ERR_* before any CUDA call.
 * ---- F35: motion evidence and segmentation ----
 * rb_motion_evidence: T frame pairs of F = T + 1 frames; flow_fw, flow_bw [T,Hn,Wn,2] fp32 (flow_fw[k] frame k -> k+1,
 * flow_bw[k] k+1 -> k), occ_fw, occ_bw [T,Hn,Wn] uint8; H [2T,9] and flags [2T] F34's fit of the 2T fields as one batch,
 * the forward fields first; cuts (nullable) [T] uint8, non-zero for a scene-cut pair.  evidence [F,Hn,Wn,2] fp32 = (N, C)
 * per frame and network pixel: from +0, the forward field of pair t, then the backward field of pair t - 1, each where
 * occ == 0, the flow is finite, the field's flag <= 1 and the pair is not a cut, adds e = r^2 / (r^2 + tau^2) to N and 1
 * to C.  r is F34's residual under the field's H in network pixels, in fp64 with every operation rounded on its own
 * (cv2's pixel centre, (p * (1/L)), X = (h1 x + h2 y) + h3, X / z, ((X/z - qx) L) Wn/Ws ...), r^2 = dx^2 + dy^2 rounded
 * once to fp32; e = 1 where z <= 0 or r^2 is not finite.  e >= 0.5 exactly when r >= tau.  One thread per network pixel.
 * rb_motion_segment: evidence [F,Hn,Wn,2] as above; flow_fw, flow_bw [F-1,Hn,Wn,2]; rows [n_rows,3] int32 in device
 * memory, row r = (t, nf, nb) (raft_b200.inpaint.inpaint_rows' table).  Per frame pixel (x, y) of row r: p0 =
 * rb_denoise_merge's pixel-centre map; (num, den) = the bilinear sample (fb_sample.cuh's bilerp_at / bilerp1) of
 * (N, C) of frame t at p0; the forward side then takes up to min(nf, F-1-t) steps of rb_denoise_merge's chain, stopping
 * at the first step that leaves the grid or fails the F5 test, and each passing step adds the bilinear samples of the
 * frame reached at the position reached; the backward side mirrors it (up to min(nb, t) steps).  Order: frame t, the
 * forward steps, the backward steps.  mask [n_rows,Hs,Ws] uint8 = 1 where den > 0 and 2 num >= den, else 0; status
 * [n_rows,Hs,Ws] uint8 = 0, or 1 where den = 0 (no evidence).  A row whose t lies outside [0, F) is absent (mask 0,
 * status 1); nf / nb are clamped into [0, RB_MOTION_SEG_MAX_WINDOW] and the clip.  Every fp32 operation is rounded on
 * its own; no atomics, no allocation.  Null pointers (cuts excepted; the flows of rb_motion_segment may be null when
 * F = 1), non-positive shapes, a frame of >= 2^31 pixels, flow_scale or tau <= 0 or non-finite and negative or
 * non-finite alphas -> RB_ERR_* before any CUDA call. */
#define RB_HOMOGRAPHY_SUMS 45
#define RB_HOMOGRAPHY_MAX_ROUNDS 32
#define RB_MOTION_SEG_TAU 1.0f
#define RB_MOTION_SEG_MAX_WINDOW 16
int rb_homography_motion_workspace_bytes(int B, int Hn, int Wn, size_t* bytes);
int rb_homography_motion(const float* flow, const uint8_t* occ, int B, int Hn, int Wn, int Hs, int Ws, float flow_scale,
                         const double* sim_params, const uint8_t* sim_flags, int rounds, double cauchy_c, double* H,
                         uint8_t* flags, double* sums, void* workspace, size_t workspace_bytes, void* stream);
int rb_motion_evidence(const float* flow_fw, const float* flow_bw, const uint8_t* occ_fw, const uint8_t* occ_bw,
                       const double* H, const uint8_t* flags, const uint8_t* cuts, int T, int Hn, int Wn, int Hs, int Ws,
                       float flow_scale, float tau, float* evidence, void* stream);
int rb_motion_segment(const float* evidence, int F, int Hn, int Wn, const float* flow_fw, const float* flow_bw, int Hs,
                      int Ws, float flow_scale, float alpha1, float alpha2, const int32_t* rows, int n_rows,
                      uint8_t* mask, uint8_t* status, void* stream);

/* ---- F9: end-point-error metrics (upstream RAFT's evaluate.py validate_sintel / validate_kitti) ---------------------
 * flow, gt: [B,H,W,2] fp32; valid: [B,H,W] uint8, nonzero = the pixel counts (NULL: every pixel counts).  Per pixel,
 * every operation rounded on its own (no FMA contraction), so the values equal upstream's torch expressions bit for bit:
 *   d = flow_scale * flow - gt,  e = sqrt(d.x*d.x + d.y*d.y),  m = sqrt(gt.x*gt.x + gt.y*gt.y),
 *   outlier = e > 3.0f && e / m > 0.05f  (KITTI's F1 rule; IEEE semantics for m = 0).
 * flow_scale as in rb_flow_fb_check: 8.0 for raft-small's reference-semantics flow (1/8-resolution units; x8 is exact),
 * 1.0 otherwise.  epe (nullable): [B,H,W] fp32, written for every pixel, counted or not.  stats: [B][RB_FLOW_STATS] fp64,
 * over the counted pixels of sample b: {n, sum e, #(e < 1), #(e < 3), #(e < 5), #outliers}; the counts are exact and a NaN
 * flow propagates into the sum.  The reduction is deterministic and independent of B: each sample's pixels are split
 * into fixed chunks, each reduced by one block in a fixed tree into the workspace (rb_flow_metrics_workspace_bytes), and a
 * second launch adds each sample's partials in a fixed order -- a batch gives the per-sample bits, no allocation, no
 * float atomics, graph-capturable.  Null pointers, B/H/W <= 0, flow_scale <= 0 or non-finite, B > 65535 and a workspace
 * that is too small -> RB_ERR_* before any CUDA call. */
#define RB_FLOW_STATS 6
int rb_flow_metrics_workspace_bytes(int B, int H, int W, size_t* bytes);
int rb_flow_metrics(const float* flow, float flow_scale, const float* gt, const uint8_t* valid, int B, int H, int W,
                    float* epe, double* stats, void* workspace, size_t workspace_bytes, void* stream);

/* ---- F10: warm start -- upstream RAFT's forward_interpolate (core/utils/utils.py), batched, on the GPU -------------
 * flow, out: [B,h,w,2] fp32 NHWC; each sample on its own.  Source pixel (x, y) with (dx, dy) = flow[b,y,x] lands at
 * x1 = (double)x + dx, y1 = (double)y + dy (exact, like numpy's int64 + float32); it is valid iff 0 < x1 < w and
 * 0 < y1 < h (strict; a NaN is invalid).  out[b,qy,qx] = the (dx, dy) of the valid source of sample b with the smallest
 * d = fl64(fl64((qx - x1)^2) + fl64((qy - y1)^2)) (no FMA contraction: cKDTree's float64 squared distance), copied bit for
 * bit; equal d -> the lower source index y*w + x.  scipy breaks such ties in kd-tree order, so the result equals upstream's
 * griddata(method='nearest') wherever the nearest source is unique.  A sample without a valid source gives zeros
 * (upstream's griddata raises on the empty point set).
 * Valid sources are bucketed by integer cell (floor(x1), floor(y1)) with integer atomics, a per-sample scan and a placement
 * pass; one thread per grid point scans rings of cells outward until no closer source can exist: O(B h w) for a flow
 * whose sources land near the grid points (a few valid sources far from most grid points degrade to every cell).  No float
 * atomics, the same bits for every B, no allocation (workspace: rb_flow_forward_interpolate_workspace_bytes), CUDA-graph
 * capturable.  Null pointers, B/h/w <= 0, B*h*w >= 2^31 and a workspace that is too small -> RB_ERR_* before any CUDA call. */
int rb_flow_forward_interpolate_workspace_bytes(int B, int h, int w, size_t* bytes);
int rb_flow_forward_interpolate(const float* flow, float* out, int B, int h, int w, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ---- F11: flow colour coding -- flow_utils.flow_to_color (the reference's flow_utils.py:95-121), batched ----------
 * flow: [B,H,W,2] fp32; out: [B,H,W,3] uint8, RGB, or BGR with convert_to_bgr.  Each sample on its own: with clip,
 * (u, v) = min(max((u, v), 0), clip_flow) first (the reference's np.clip(flow, 0, clip): negative components become 0).
 * Per pixel, each operation rounded on its own (no FMA contraction), in numpy's types for a float32 flow:
 *   fp32  rad = sqrt(u^2 + v^2); den = fl32(max_b rad + 1e-5f); u' = u / den, v' = v / den; r = sqrt(u'^2 + v'^2);
 *         a = fl32(atan2((double)-v', (double)-u')) / fl32(pi); fk = ((a + 1) / 2) * 54 + 1;
 *         k0 = min(floor(fk), 53), k1 = k0 + 1 (55 -> 1);
 *   fp64  f = fk - k0; col = (1 - f) * (wheel[k0] / 255.0) + f * (wheel[k1] / 255.0);
 *         col = r <= 1 ? 1 - r * (1 - col) : col * 0.75; out = floor(255 * col).
 * wheel is make_colorwheel() (55 rows).  The one difference from numpy is arctan2, computed in fp64 and rounded once to
 * fp32 (numpy's float32 arctan2 is not correctly rounded and depends on the machine).  Indices are clamped into the
 * wheel, so non-finite flows read nothing out of bounds (their colours are unspecified).  The maximum radius is reduced
 * per sample in fixed chunks into the workspace (rb_flow_to_color_workspace_bytes) by a first launch; a batch gives the
 * per-sample bits, no allocation, no synchronisation, graph-capturable.  Null pointers, B/H/W <= 0, a non-finite
 * clip_flow with clip, B > 65535 and a workspace that is too small -> RB_ERR_* before any CUDA call. */
int rb_flow_to_color_workspace_bytes(int B, int H, int W, size_t* bytes);
int rb_flow_to_color(const float* flow, int B, int H, int W, int clip, float clip_flow, int convert_to_bgr, uint8_t* out,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- F12: frame metrics -- PSNR / SSIM of interpolated frames (the Vimeo-90K triplet protocol) --------------------
 * pred: [B,H,W,3], fp32 (pred_is_u8 = 0) or uint8 (1); gt: [B,H,W,3] uint8.  An fp32 value x is quantised as
 * infer_raft.py --interpolate writes its PNGs, np.clip(np.rint(fl32(255 * x)), 0, 255): q = rintf(__fmul_rn(255.f, x))
 * (ties to even), clamped to [0, 255]; a NaN becomes 0.  So the scores describe the 8-bit frame a user would write.
 * stats: [B][RB_FRAME_STATS] fp64 per sample b:
 *   stats[b][0] = SSE = sum over the H*W*3 values of (q - gt)^2, summed in integers: exact;
 *   stats[b][1] = SSIM = the mean over the 3 channels of skimage's structural_similarity(gt_c, q_c,
 *     gaussian_weights=True, sigma=1.5, use_sample_covariance=False, data_range=255), in fp64: with the 11-tap window
 *     w_k = exp(-k^2 / (2 * 1.5^2)) / sum_j exp(-j^2 / (2 * 1.5^2)), k = -5..5 (scipy's gaussian_filter, truncate 3.5),
 *     mx, my, Exx, Eyy, Exy the separable 11x11 weighted means, vx = Exx - mx^2, vy = Eyy - my^2, vxy = Exy - mx*my,
 *     C1 = (0.01*255)^2, C2 = (0.03*255)^2, S = (2 mx my + C1)(2 vxy + C2) / ((mx^2 + my^2 + C1)(vx + vy + C2)), and SSIM
 *     the mean of S over the crop [5, H-5) x [5, W-5) -- exactly the pixels whose window stays inside the frame, so
 *     skimage's reflect padding never reaches a counted pixel.
 * PSNR = 10 log10(255^2 * 3HW / SSE) follows on the host.  Each block reduces one fixed tile of one sample into the
 * workspace (rb_frame_metrics_workspace_bytes) and a second launch adds each sample's partials in a fixed order: a sample's
 * bits do not depend on B or its place in the batch; no allocation, no float atomics, graph-capturable.  Null pointers,
 * pred_is_u8 not 0 or 1, B/H/W <= 0, H or W < 11 (skimage refuses a window larger than the image), B > 65535 and a
 * workspace that is too small -> RB_ERR_* before any CUDA call. */
#define RB_FRAME_STATS 2
int rb_frame_metrics_workspace_bytes(int B, int H, int W, size_t* bytes);
int rb_frame_metrics(const void* pred, int pred_is_u8, const uint8_t* gt, int B, int H, int W, double* stats,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- F20: label metrics -- DAVIS-2017's J (region) and F (boundary) as integer counts ----------------------------
 * pred, gt: [n,H,W] uint8 label maps.  counts: [n][n_objects][RB_LABEL_STATS] int64, zeroed by the call on the stream.
 * For frame i and object o = 1..n_objects, with P = (pred == o) and G = (gt == o):
 *   {|P and G|, |P or G|, #boundary(P), #boundary(G), #(boundary(P) with a boundary(G) pixel in the disk),
 *    #(boundary(G) with a boundary(P) pixel in the disk)}.
 * boundary is davis2017-evaluation's _seg2bmap at the map's own size: b = (m ^ e) | (m ^ s) | (m ^ se), e / s / se the
 * right / down / down-right neighbours (0 outside the image), the last row m ^ e, the last column m ^ s, the last pixel
 * 0.  The disk is skimage.morphology.disk(bound_pix), the offsets with dx^2 + dy^2 <= bound_pix^2; pixels outside the
 * image never match (cv2.dilate's default border).  Tiles of 32 x 32 pixels with a halo of bound_pix + 1 in shared
 * memory; block counts reach global memory through 64-bit integer atomics, so they are exact and deterministic.  Null
 * pointers, n/H/W <= 0, n > 65535, n_objects outside [1, 255] and bound_pix outside [1, 32] -> RB_ERR_* before any CUDA
 * call.  DAVIS's bound_pix = ceil(0.008 * hypot(H, W)): 8 at 480p, 18 at 1080p. */
#define RB_LABEL_STATS 6
int rb_label_metrics(const uint8_t* pred, const uint8_t* gt, int n, int H, int W, int n_objects, int bound_pix,
                     int64_t* counts, void* stream);

/* ---- F15: scene-cut scores -- where frame-rate conversion and warm-started video flow stop ------------------------
 * frames: [N,H,W,3] uint8, the decoded frames at their own size (any channel order: the bins are symmetric in it).
 * hist: [N][RB_SCENE_BINS] int32, frame n's joint colour histogram, pixel (c0, c1, c2) in bin
 *   (c0 >> 5) * 64 + (c1 >> 5) * 8 + (c2 >> 5) (8 levels per channel), each pixel counted once; zeroed by the call.
 * scores: [N-1] fp32, scores[k] = fl32((double)(H*W - sum_b min(hist[k][b], hist[k+1][b])) / (double)(H*W)): one minus
 *   the histogram intersection of frames k and k + 1, in [0, 1] -- 0 for frames with one histogram, 1 for frames that
 *   share no bin.
 * Counts are integers (warp-aggregated shared-memory atomics, then one global atomic per block and nonzero bin), so both
 * outputs are exact and independent of the launch order.  A memset and two launches on the stream; no allocation, no
 * synchronisation, graph-capturable.  Null pointers, N < 2, H/W <= 0, H*W >= 2^31 and N frames that exceed one grid ->
 * RB_ERR_* before any CUDA call. */
#define RB_SCENE_BINS 512
int rb_scene_cut_scores(const uint8_t* frames, int N, int H, int W, int32_t* hist, float* scores, void* stream);

/* ---- F3 (input edge): dataflow/test_dataflow.py:56-61,96-97 + the SURVEY 8(d) shape policy ------------------
 * src: [B,H,W,3] device frames, BGR like cv2.imdecode -- fp32 in [0,1] (src_is_u8 = 0) or uint8 in [0,255]
 * (src_is_u8 = 1: x/255.0f, the reference's np.float32(x)/255.0, bit for bit).  dst: [B,H+pt+pb,W+pl+pr,3] fp32
 * in [0,1], replicate-padded (upstream InputPadder; the caller chooses the split).  The 2x-1 of
 * RAFT.input_preprocess (RAFT.py:53-59) is applied inside rb_encoder_forward. */
int rb_frames_prepare(const void* src, int src_is_u8, float* dst, int B, int H, int W, int pad_top,
                      int pad_bottom, int pad_left, int pad_right, void* stream);
/* rb_frames_resize: the reference's cv2.resize of every frame to the network size (test_dataflow.py:85-87), bit for
 * bit with OpenCV 4.13's bilinear resize, then (uint8) the /255 of rb_frames_prepare and the replicate pad.
 * src [B,H,W,3] uint8 or fp32, any H, W >= 1; dst [B,Ho+pad_top+pad_bottom,Wo+pad_left+pad_right,3] fp32.  One thread
 * per output pixel, coefficients computed in-kernel (tests/resize_oracle.py restates both of cv2's algorithms).
 * Null pointers, B/H/W/Ho/Wo <= 0, negative pads -> RB_ERR_* before any CUDA call; no allocation, no synchronisation. */
int rb_frames_resize(const void* src, int src_is_u8, float* dst, int B, int H, int W, int Ho, int Wo, int pad_top,
                     int pad_bottom, int pad_left, int pad_right, void* stream);
/* rb_flow_resize: flow_utils.py:277-284 resize_flow for a batch: flow [B,H,W,2] fp32 -> dst [B,Ho,Wo,2], each channel
 * resized like cv2's float bilinear resize, then u *= fl32(Wo / W) and v *= fl32(Ho / H) (numpy >= 2 float32 multiply).
 * Argument errors as rb_frames_resize. */
int rb_flow_resize(const float* flow, float* dst, int B, int H, int W, int Ho, int Wo, void* stream);

/* ---- F1: BasicEncoder / SmallEncoder  networks/model_utils.py:61-105 (+ input_preprocess RAFT.py:53-59) --
 * norm: 0 = 'none', 1 = 'instance' (fnet), 2 = 'batch' (cnet of raft-things; folded into the convs at pack
 * time from inference statistics).  Convs are enumerated in execution order; names are relative to the
 * encoder scope ("conv1", "layer2/0/downsample.0", ...), rb_encoder_norm_name gives the scope of the norm
 * that follows conv i ("" = none).  W_host[i] HWIO fp32, b_host[i] [cout]; bn_host[i] (norm == 2 only) is
 * [gamma | beta | mean/EMA | variance/EMA], 4*cout floats.  image: [B,H,W,3] fp32 in [0,1] (2x-1 is applied
 * inside); out: [B,ceil(H/8),ceil(W/8),out_dim] fp32.  The workspace must be zero-filled once before first use. */
int rb_encoder_num_convs(int small);
const char* rb_encoder_conv_name(int small, int i);
const char* rb_encoder_norm_name(int small, int i);
int rb_encoder_conv_shape(int small, int i, int out_dim, int* k, int* stride, int* cin, int* cout);
int rb_encoder_weights_bytes(int small, int out_dim, size_t* bytes);
int rb_encoder_weights_pack(int small, int norm, int out_dim, const float* const* W_host,
                            const float* const* b_host, const float* const* bn_host, void* blob,
                            size_t blob_bytes, void* stream);
/* Host-only forms (no GPU needed), as for the update block; conv index i as in rb_encoder_conv_name.  The stem is packed
 * as a 4x1 conv over the space-to-depth view (csrc/encoder.cu), batch norm is folded into weights and bias. */
int rb_encoder_weights_pack_host(int small, int norm, int out_dim, const float* const* W_host, const float* const* b_host,
                                 const float* const* bn_host, void* host_blob, size_t blob_bytes);
int rb_encoder_packed_conv(int small, int out_dim, int i, size_t* hi_off, size_t* lo_off, size_t* bias_off, int* kh, int* kw,
                           int* cin_pad, int* cout_pad);
int rb_encoder_workspace_bytes(int small, int B, int H, int W, size_t* bytes);
int rb_encoder_forward(int small, int norm, const void* weights, const float* image, float* out, int B,
                       int H, int W, int out_dim, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RAFT_B200_H_ */
