/*
 * td_b200.h -- C-ABI of the H100-native tiled-diffusion / tiled-VAE hot path.
 *
 * The reference (pkuliyi2015/multidiffusion-upscaler-for-automatic1111 @ 22798f6)
 * has NO FFI boundary: its hot path is eager PyTorch inside Python classes
 * (SURVEY.md section 8(b)).  This header is the boundary our Python host classes
 * (same names / arguments as the reference's tile-method + VAEHook surface) bind
 * with ctypes; INTEGRATION.md shows the binding a reference maintainer would add.
 * Each entry point cites the reference code it replaces (file:line relative to
 * the reference root).
 *
 * Conventions
 *   - plain C types only: pointers, sizes, a cudaStream_t passed as void*;
 *   - DEVICE pointers are `tensor.data_ptr()`; the caller (PyTorch) owns all memory;
 *   - no allocation, no host<->device sync, no exceptions: every function returns
 *     TD_OK (0) or a negative td_status, and td_last_error() gives the message;
 *   - all work is enqueued on the given stream (reference: "current stream").
 */
#ifndef TD_B200_H
#define TD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TD_ABI_VERSION 13

typedef enum td_status {
    TD_OK = 0,
    TD_ERR_INVALID_ARG = -1, /* null pointer, negative size, out-of-range index */
    TD_ERR_UNSUPPORTED = -2, /* legal in the reference but not on this path (e.g. >256 grid rows) */
    TD_ERR_CUDA = -3,        /* launch / driver error; see td_last_error() */
    TD_ERR_CAPACITY = -4     /* caller-provided output array too small */
} td_status;

typedef enum td_dtype { TD_F16 = 0, TD_BF16 = 1, TD_F32 = 2 } td_dtype;

/* blend flags */
#define TD_FLAG_FORCE_GENERIC 1u /* use the scalar any-alignment kernel (test / fallback path) */
#define TD_FLAG_NO_TMA 2u        /* use the register-staged vector kernels (no smem staging): scatter_vec_kernel
                                    instead of the row-block scatter, the register-staged blends */
#define TD_FLAG_TMA 4u           /* blend: use the TMA-staged kernel instead of the cp.async one   */
#define TD_FLAG_PIPELINE 8u      /* blend: persistent software-pipelined cp.async form (measured slower) */
#define TD_FLAG_PEER_ASYNC 16u   /* peer blend: stage peer tiles with cp.async instead of direct 128-bit loads */
#define TD_FLAG_NO_PDL 32u       /* launch without the programmatic-dependent-launch attribute (A/B measurement) */
#define TD_FLAG_ONE_PLANE 64u    /* cp.async blend: one (n, c) plane per CTA (the default of a TD_AS_PPC=1 build) */
#define TD_FLAG_STRIP 128u       /* MultiDiffusion blend: strip CTAs (8 rows x full width), opt-in, see csrc/td_strip.cu */
#define TD_FLAG_DBG_NO_TILES 0x100u /* measurement aid: skip all tile visits (launch + epilogue floor) */
#define TD_FLAG_ROWS 0x400u      /* row-block form (csrc/td_rows.cu: one persistent CTA per SM, bulk-copy staging), bit-identical:
                                    the scatter's default; opt-in for the blends, whose defaults stay many small co-resident
                                    CTAs (DESIGN.md section 4) */

#define TD_MAX_GRID_DIM 256   /* max tile rows / cols of a grid plan            */
#define TD_MAX_BATCH_PTRS 128 /* max UNet output batch tensors per blend launch */
#define TD_MAX_PEERS 16       /* max ranks of a tile-sharded step (one process per GPU) */
#define TD_IPC_HANDLE_BYTES 64

const char* td_last_error(void);
int td_abi_version(void);
/* measurement aid: an empty kernel launch (launch-latency floor of the bench harness) */
int td_debug_launch_empty(int blocks, int threads, void* stream);
/* measurement / test aid: counts (16-bit numerator, integer w <= max_w) pairs where the fast divide differs from IEEE */
int td_debug_check_fast_div(int dtype, int max_w, unsigned long long* mismatches_dev, void* stream);

/* ------------------------------------------------------------------------- *
 *  Host bookkeeping (integer-exact; Python float64 semantics reproduced with
 *  C double).  No GPU needed.
 * ------------------------------------------------------------------------- */

/* split_bboxes -- tile_utils/utils.py:160-177.
 * Writes up to `cap` tiles as (x, y, w, h) int32 quadruples in row-major order
 * (row outer, col inner).  Returns the tile count T (>= 1) or a td_status.
 * out_cols / out_rows may be NULL. */
int td_split_bboxes(int w, int h, int tile_w, int tile_h, int overlap,
                    int32_t* out_xywh, int cap, int* out_cols, int* out_rows);

/* splitable -- tile_utils/utils.py:151-158 (w, h in IMAGE pixels). Returns 0/1. */
int td_splitable(int w, int h, int tile_w, int tile_h, int overlap);

/* gaussian_weights -- tile_utils/utils.py:180-194.  out: fp32 [tile_h*tile_w]. */
int td_gaussian_weights(int tile_w, int tile_h, float* out);

/* feather_mask -- tile_utils/utils.py:196-214 (region prompt control, FOREGROUND boxes).
 * out: fp32 [h*w]; 1 inside, (dist/radius)^2 towards the border, radius = int(min(w//2, h//2) * ratio). */
int td_feather_mask(int w, int h, double ratio, float* out);

/* Region rectangle in latent units from the UI's relative (x, y, w, h) --
 * tile_methods/abstractdiffusion.py:206-215: x = max(0, int(x*W)), w = min(W - x, ceil(w*W)), same for y / h.
 * Returns 1 and writes out_xywh, or 0 if the reference skips the box (x > 1, y > 1, w <= 0 or h <= 0). */
int td_custom_bbox_rect(double x, double y, double w, double h, int canvas_w, int canvas_h, int32_t* out_xywh);

/* Grid plan = what init_grid_bbox leaves on the delegate
 * (tile_methods/abstractdiffusion.py:172-186): clamped tile size and overlap,
 * separable tile origins, tile count and re-balanced tile batch size, and the
 * axes on which the canvas is periodic (seamless tiling). */
#define TD_WRAP_X 1u /* td_grid.wrap: the canvas is periodic in x */
#define TD_WRAP_Y 2u /* td_grid.wrap: the canvas is periodic in y */
typedef struct td_grid {
    int32_t H, W;           /* latent canvas, abstractdiffusion.py:25-26           */
    int32_t tile_h, tile_w; /* min(tile, canvas), :176-177                         */
    int32_t overlap;        /* clamped with the UNclamped tile args, :178          */
    int32_t rows, cols;     /* utils.py:161-162                                    */
    int32_t num_tiles;      /* rows*cols                                           */
    int32_t num_batches;    /* ceil(T / tile_bs), :184                             */
    int32_t tile_bs;        /* ceil(T / num_batches), :185                         */
    int32_t wrap;           /* TD_WRAP_X | TD_WRAP_Y: periodic axes (new)          */
    int32_t ys[TD_MAX_GRID_DIM]; /* tile-row origins, utils.py:169                 */
    int32_t xs[TD_MAX_GRID_DIM]; /* tile-col origins, utils.py:171                 */
} td_grid;

/* init_grid_bbox -- abstractdiffusion.py:172-186.  w, h are LATENT sizes.  Returns T or a td_status.
 * `wrap` (TD_WRAP_X | TD_WRAP_Y, stored in g->wrap) tiles those axes as a circle -- seamless tiling, new: the reference
 * has no periodic plan.  A wrapped axis of length L with (clamped) tile t has one tile at 0 when t == L, else
 * n = ceil(L / (t - overlap)) tiles at floor(k * (L / n)) (float64): origins lie in [0, L), a tile may run past L and
 * continue at 0, and cyclic neighbours -- the last and the first included -- overlap by at least `overlap`.  A bounded
 * axis, the clamps, the tile order, num_batches and tile_bs follow the reference. */
int td_grid_init(td_grid* g, int w, int h, int tile_w, int tile_h, int overlap, int tile_bs, int wrap);

/* Weight canvas of split_bboxes -- utils.py:167,175: fp32 [H*W] zeros, then
 * `+= init_weight` per tile in list order.  tile_weights NULL => 1.0
 * (abstractdiffusion.py:188-190), else fp32 [tile_h*tile_w]
 * (mixtureofdiffusers.py:38-43).  HOST arrays.  On an axis whose g->wrap bit is set
 * the placement is modular: tile (r, c) adds at ((ys[r]+v) mod H, (xs[c]+u) mod W).
 * Rejects (TD_ERR_INVALID_ARG) a tile that leaves the canvas on a bounded axis. */
int td_grid_weights(const td_grid* g, const float* tile_weights, float* out_weights);

/* rescale_factor = 1 / weights -- mixtureofdiffusers.py:32 (fp32 IEEE divide). */
int td_rescale_factor(const float* weights, float* out, int64_t n);

/* ------------------------------------------------------------------------- *
 *  Device kernels: per-sampler-step hot path.
 * ------------------------------------------------------------------------- */

/* Scatter -- multidiffusion.py:155, mixtureofdiffusers.py:88,104:
 *   tiles[(t - tile_begin)*N + n, c, v, u] = x[n, c, ys[t/cols] + v, xs[t%cols] + u]
 * for t in [tile_begin, tile_end): ONE launch for the whole step (the reference
 * issues one torch.cat per tile batch).  x: [N,C,H,W] contiguous; tiles:
 * [(tile_end-tile_begin)*N, C, tile_h, tile_w] contiguous; same dtype. */
int td_scatter_tiles(const td_grid* g, const void* x, void* tiles, int N, int C, int dtype,
                     int tile_begin, int tile_end, uint32_t flags, void* stream);
/* Every grid entry below (and td_scatter_tiles) rejects with TD_ERR_INVALID_ARG a plan whose tiles leave the canvas
 * (origin < 0, origin + tile > extent) on an axis whose g->wrap bit is clear.  With the bit set, coverage on
 * that axis is modular: canvas pixel x is covered by tile column c when (x - xs[c]) mod W < tile_w, and the tile
 * element is taken at that residue (the same in y).  The arithmetic -- tile order, per-add rounding, the MultiDiffusion
 * normalisation and the Mixture of Diffusers products -- is unchanged. */

/* Blend + normalise, MultiDiffusion -- multidiffusion.py:166-167 + :208 fused,
 * gather form, one launch per step:
 *   acc = 0 (acc_dtype);  for covering tiles t ascending: acc = round_acc(float(acc) + float(tile_t))
 *   x_out = weights > 1 ? float(acc) / weights : float(acc)          (fp32, IEEE divide)
 * which is bit-identical to the reference's sequential `x_buffer[slicer] +=`.
 * batch_ptrs: HOST array of `num_batches` DEVICE pointers, batch b holding tiles
 * [b*tile_bs, min((b+1)*tile_bs, T)) as [.*N, C, tile_h, tile_w] contiguous
 * (the UNet's output tensors; peer-GPU pointers are allowed).
 * weights: fp32 [H*W] device.  x_out: fp32 [N,C,H,W].  x_buffer (acc_dtype,
 * [N,C,H,W]) is optional (NULL = do not materialise abstractdiffusion.py:24).
 * rcp_weights: optional fp32 [H*W] = correctly rounded 1/weights (td_rescale_factor).  Pass it
 * ONLY when every weight is an integer <= 4096 (MultiDiffusion's always are) and the canvas is
 * fp16/bf16: the divide then runs as q=a*rcp; r=fma(-q,w,a); q+=r*rcp, which is the correctly
 * rounded quotient on that domain (exhaustively verified by td_debug_check_fast_div). */
int td_blend_multidiffusion(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs,
                            int N, int C, int tile_dtype, int acc_dtype, const float* weights,
                            const float* rcp_weights, float* x_out, void* x_buffer, uint32_t flags,
                            void* stream);

/* Blend, Mixture of Diffusers -- mixtureofdiffusers.py:122-126, returns x_buffer (:169):
 *   w   = tile_weights[v,u] * rescale[y,x]                       (fp32 product)
 *   acc = round_acc(float(acc) + float(tile_t) * w)              (separate mul / add roundings)
 * tile_weights: fp32 [tile_h*tile_w]; rescale: fp32 [H*W]; x_buffer: acc_dtype [N,C,H,W]. */
int td_blend_mixture(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs,
                     int N, int C, int tile_dtype, int acc_dtype, const float* tile_weights,
                     const float* rescale, void* x_buffer, uint32_t flags, void* stream);

/* ------------------------------------------------------------------------- *
 *  Tiled VAE (scripts/tilevae.py of the reference).
 * ------------------------------------------------------------------------- */

/* get_best_tile_size -- tilevae.py:390-403. */
int td_vae_best_tile_size(int lowerbound, int upperbound);

/* split_tiles -- tilevae.py:405-462.  Writes T input and T output bboxes as int32
 * [x1, x2, y1, y2] quadruples (input bbox already expanded by `pad` and clipped;
 * output bbox snapped to the borders and scaled x8 (decoder) or //8 (encoder)).
 * Pass NULL arrays to query T.  Returns T or a td_status.
 * `wrap` (TD_WRAP_X | TD_WRAP_Y; 0 = the reference's split) splits those axes as a circle -- seamless tiling, new.
 * A wrapped axis of length L gets n = max(ceil(L / tile_size), 1) tiles cut at b_k = m * floor(k * L / (n * m)), b_n = L
 * (m = 8 for the encoder, 1 for the decoder); output bbox [b_k, b_{k+1}) (x8 decoder, /8 encoder), input bbox
 * [b_k - pad, b_{k+1} + pad) in UNwrapped coordinates: it may be negative or exceed L, the tile load reads it modulo L
 * (td_nchw_to_nhwc_wrap, or td_copy_region per piece). */
int td_vae_split_tiles(int h, int w, int tile_size, int pad, int is_decoder, int wrap,
                       int32_t* in_bboxes, int32_t* out_bboxes, int cap);

/* Statistics of `nseg` contiguous segments of `seg_len` elements each, ONE read:
 * get_var_mean -- tilevae.py:207-215 with nseg = B*32, seg_len = (C/32)*H*W (the
 * channels of a group are adjacent in NCHW); also the per-channel std_mean of the
 * fast-mode prelude (tilevae.py:553-554, nseg = B*C, seg_len = H*W, unbiased = 1) and
 * z.min()/z.max() (:559) through the optional seg_min / seg_max outputs.
 * mean, var (biased unless `unbiased`), seg_min, seg_max: fp32 [nseg] device.
 * workspace: device scratch of td_gn_stats_workspace_bytes() bytes. */
int64_t td_gn_stats_workspace_bytes(int64_t nseg, int64_t seg_len, int dtype);
int td_gn_stats(const void* x, int64_t nseg, int64_t seg_len, int dtype, int unbiased,
                void* workspace, int64_t workspace_bytes, float* mean, float* var,
                float* seg_min, float* seg_max, void* stream);

/* custom_group_norm (+ SiLU) -- tilevae.py:218-245 (+ :102-104), fused, one read and one
 * write:  y = act(((x - mean[g]) / sqrt(var[g] + eps)) * gamma[c] + beta[c]).
 * x, y: [B, C, HW] of `dtype` (y may alias x).  mean / var: fp32 [groups] shared by the
 * batch (stats_per_batch = 0: the reference's merged / estimated statistics) or
 * [B*groups] (stats_per_batch = 1).  gamma / beta: fp32 [C] or NULL.  act: 0 none, 1 SiLU. */
int td_gn_apply(const void* x, void* y, int B, int C, int64_t HW, int dtype, int groups,
                const float* mean, const float* var, int stats_per_batch, const float* gamma,
                const float* beta, float eps, int act, void* stream);

/* Strided 3-D region copy dst[p, r, c] = src[p, r, c]: the tile crop (tilevae.py:532-535,
 * which the reference stages through host RAM) and crop_valid_region + paste
 * (tilevae.py:248-259, :632).  Pointers are already offset to the region origin; strides
 * and pitches are in elements. */
int td_copy_region(const void* src, void* dst, int planes, int rows, int cols,
                   int64_t src_plane_stride, int64_t src_pitch, int64_t dst_plane_stride,
                   int64_t dst_pitch, int dtype, void* stream);

/* Fast-mode estimator input -- tilevae.py:545-559.
 * td_resample_nearest: out[p, i, j] = in[p, src_y[i], src_x[j]] (F.interpolate
 * nearest-exact; the index tables are computed on the host with ATen's float32 rule).
 * td_affine_clamp: x = clamp((x - mean_new[c]) / std_new[c] * std_old[c] + mean_old[c],
 * lo[0], hi[0]) in place, every step rounded through `dtype` like the eager ops. */
int td_resample_nearest(const void* in, void* out, int planes, int H, int W, int oh, int ow,
                        const int32_t* src_y, const int32_t* src_x, int dtype, void* stream);
int td_affine_clamp(void* x, int B, int C, int64_t HW, int dtype, const float* mean_new,
                    const float* std_new, const float* mean_old, const float* std_old,
                    const float* lo, const float* hi, void* stream);

/* ------------------------------------------------------------------------- *
 *  Multi-GPU tile shard (new: the reference is single-device, SURVEY.md section 5).
 *  One process per GPU; rank r denoises a contiguous chunk of the tile list into an
 *  exchange buffer that its peers map through CUDA IPC; td_peer_signal publishes a
 *  step counter into every peer's flag array; td_blend_multidiffusion_peer waits for
 *  all ranks' counters and blends, reading peer tile outputs over NVLink in the same
 *  kernel (batch_ptrs[b] = rank b's buffer).  Deterministic tile order => the latent is
 *  bit-identical on every rank and to a single-GPU run.
 * ------------------------------------------------------------------------- */
int td_dev_alloc(int64_t bytes, void** out);   /* cudaMalloc'd (IPC-exportable), zero-filled */
int td_dev_free(void* ptr);
int td_ipc_get_handle(const void* dev_ptr, void* handle_out /* TD_IPC_HANDLE_BYTES */);
int td_ipc_open(const void* handle, void** dev_ptr_out);
int td_ipc_close(void* dev_ptr);
/* flag_ptrs: HOST array [world] of DEVICE pointers to each rank's uint32[world] flag array
 * (own array for i == rank, IPC-mapped for peers).  Bumps this rank's device-side *step_counter
 * and stores the new value into slot `rank` of every array (CUDA-graph replayable: no host-side
 * step number). */
int td_peer_signal(void* const* flag_ptrs, int world, int rank, uint32_t* step_counter, void* stream);
/* As td_blend_multidiffusion, preceded in-kernel by: wait until wait_flags[i] >= *wait_value for
 * all i < world (acquire, system scope).  wait_flags: this rank's own uint32[world] array;
 * wait_value: this rank's step counter (the one td_peer_signal bumps). */
int td_blend_multidiffusion_peer(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs,
                                 int N, int C, int tile_dtype, int acc_dtype, const float* weights,
                                 float* x_out, void* x_buffer, const uint32_t* wait_flags, int world,
                                 const uint32_t* wait_value, uint32_t flags, void* stream);

/* Row-strip tile shard: td_blend_multidiffusion restricted to canvas rows [row_begin, row_end) (multiples of 8, or H),
 * preceded in-kernel by the acquire wait of td_blend_multidiffusion_peer on wait_flags[0 .. wait_count) (wait_count 0: no
 * wait).  A rank blends only the rows it owns; batch_ptrs has one entry per tile ROW (tile_bs = cols): the rank's own tile
 * outputs or the halo buffer its neighbours pushed the overlapping tile rows into (entries of tile rows that do not
 * touch the range are never dereferenced).  Same arithmetic, same tile order: bit-identical to the whole-canvas blend.
 * own_band_begin / own_band_end: tile rows whose batch_ptrs entries are LOCAL outputs -- CTAs that read only those skip the
 * wait and are scheduled ahead of the ones that need a neighbour's halo (begin == end: every CTA waits).  A build whose
 * blend patches are taller than 8 rows (TD_AS_ROWS) refuses a window not aligned to them with TD_ERR_UNSUPPORTED. */
int td_blend_multidiffusion_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs,
                                 int N, int C, int tile_dtype, int acc_dtype, const float* weights,
                                 const float* rcp_weights, float* x_out, void* x_buffer, int row_begin, int row_end,
                                 const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                                 int own_band_begin, int own_band_end, uint32_t flags, void* stream);
/* Row-strip tile shard, Mixture of Diffusers: td_blend_mixture restricted to canvas rows [row_begin, row_end) of x_buffer
 * (whole-canvas, acc_dtype; the other rows are not written), with the row window, the per-tile-row batch_ptrs, the halo wait
 * and the own bands of td_blend_multidiffusion_rows, and the same refusals.  Same arithmetic, same tile order: the union of
 * the strips is bit-identical to td_blend_mixture over the whole canvas.  Needs the vector path (tile_dtype == acc_dtype,
 * W and tile_w multiples of the vector, 16-byte aligned tile_weights / rescale / x_buffer) and tile_w % 8 == 0, else
 * TD_ERR_UNSUPPORTED. */
int td_blend_mixture_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs,
                          int N, int C, int tile_dtype, int acc_dtype, const float* tile_weights,
                          const float* rescale, void* x_buffer, int row_begin, int row_end,
                          const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                          int own_band_begin, int own_band_end, uint32_t flags, void* stream);
/* Row-strip tile shard on a periodic plan (g->wrap != 0, seamless tiling): td_blend_multidiffusion / td_blend_mixture of the
 * canvas rows [row_begin, row_end) only, with the per-tile-row batch_ptrs (tile_bs = cols), the in-kernel halo wait and the
 * own bands of td_blend_multidiffusion_rows.  Coverage is modular: under TD_WRAP_Y a row near the top of the canvas is also
 * covered by the last tile row(s), and a CTA waits when any of its rows is covered by a tile row outside the own bands.
 * wait_flags[0 .. wait_count) may run past the world size (mirrored flag slots), never past TD_MAX_PEERS entries.  Same
 * arithmetic and tile order as the whole-canvas wrap blend: every row gets its bits.  Needs the vector path (tile_dtype ==
 * acc_dtype, W and tile_w multiples of the vector, 16-byte aligned buffers), else TD_ERR_UNSUPPORTED; a bounded plan
 * (wrap == 0) returns TD_ERR_UNSUPPORTED (it takes the rows entries above).  An empty window launches nothing. */
int td_blend_multidiffusion_wrap_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                      int tile_dtype, int acc_dtype, const float* weights, float* x_out, void* x_buffer,
                                      int row_begin, int row_end, const uint32_t* wait_flags, int wait_count,
                                      const uint32_t* wait_value, int own_band_begin, int own_band_end, uint32_t flags, void* stream);
int td_blend_mixture_wrap_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                               int tile_dtype, int acc_dtype, const float* tile_weights, const float* rescale, void* x_buffer,
                               int row_begin, int row_end, const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                               int own_band_begin, int own_band_end, uint32_t flags, void* stream);
/* One warp spins (acquire, system scope, bounded) until flags[i] >= *value for i < count: stream-ordered work after it
 * sees what the signalling ranks wrote before their td_peer_signal. */
int td_peer_wait(const uint32_t* flags, int count, const uint32_t* value, void* stream);

/* Halo push of the row-strip shard in one launch of TD_PUSH_CTAS CTAs: copies up to TD_MAX_PUSH_REGIONS strided 2-D regions
 * (16-byte aligned pointers / pitches / row lengths; dst usually IPC-mapped peer memory); every CTA then adds 1 (release,
 * system scope) to each target_slots[i] -- DEVICE pointers to slot `rank` of the targets' flag arrays -- so a slot advances by
 * TD_PUSH_CTAS per push and "slot >= expect" means the whole push has landed (one NVLink round trip for data + signal).
 * expect_own (NULL: untouched): this rank's expect counter of the set, advanced by TD_PUSH_CTAS when the launch starts; with
 * wait_count > 0 the launch then waits until wait_flags[i] >= *expect_own for i < wait_count (as td_peer_wait).
 * bump_next (NULL: none): a second expect counter advanced by TD_PUSH_CTAS at the end of the launch -- the tile-halo set's,
 * by the latent-halo push that closes a step, so that the next step's blend (td_blend_multidiffusion_rows: wait_value) reads a
 * value written on ITS stream while the tile-halo push itself may run on a side stream.  Expect counters of a set that is
 * only ever waited on through bump_next start at TD_PUSH_CTAS.  n_regions 0 is a signal-only push: the slots still advance
 * by TD_PUSH_CTAS (a rank inside a waiter's range that has no rows for it). */
#define TD_MAX_PUSH_REGIONS 8
#define TD_PUSH_CTAS 32
typedef struct td_push_region {
    const void* src;
    void* dst;
    int32_t planes, rows;
    int64_t row_bytes, src_plane_bytes, src_pitch_bytes, dst_plane_bytes, dst_pitch_bytes;
} td_push_region;
int td_push_regions(const td_push_region* regions, int n_regions, void* const* target_slots, int n_targets,
                    uint32_t* expect_own, const uint32_t* wait_flags, int wait_count, uint32_t* bump_next, void* stream);

/* Region prompt control (custom bboxes): everything after the regions' denoiser calls in ONE launch --
 * multidiffusion.py:187-216 / mixtureofdiffusers.py:145-175.  x_buffer: the grid accumulator [N,C,H,W] of `dtype`
 * (zeros when the background layer is off).  Regions in list order; mode 0 = BACKGROUND (added into the accumulator,
 * multiplied by the fp32 [h*w] `aux` when given: Mixture of Diffusers' custom_weights), mode 1 = FOREGROUND (`aux` =
 * fp32 [h*w] feather mask: averaged over overlapping regions and laid over the normalised background).
 * weights: fp32 [H*W] divide-where->1 canvas (MultiDiffusion) or NULL (Mixture of Diffusers).  out: fp32 [N,C,H,W].
 * Every rounding of the reference's tensor expressions is reproduced (see csrc/td_region.cu). */
#define TD_MAX_REGIONS 32
typedef struct td_region {
    int32_t x, y, w, h;
    int32_t mode;
    const void* out;     /* region denoiser output [N, C, h, w] of `dtype`, device */
    const float* aux;
} td_region;
int td_region_composite(const void* x_buffer, const float* weights, const td_region* regions, int n_regions,
                        int N, int C, int H, int W, int dtype, float* out, void* stream);
/* td_region_composite limited to canvas rows [row_begin, row_end) (0 <= row_begin <= row_end <= H): the same per-pixel
 * arithmetic, only those rows of `out` are written (x_buffer, weights and out are still whole-canvas pointers).  Regions keep
 * canvas coordinates; a region may also be given clipped to the window -- y and h narrowed to the rows it covers there,
 * `out` holding just those rows as [N, C, h, w] and `aux` pointing at the first of them -- and reads the same values. */
int td_region_composite_rows(const void* x_buffer, const float* weights, const td_region* regions, int n_regions,
                             int N, int C, int H, int W, int dtype, float* out, int row_begin, int row_end, void* stream);

/* ------------------------------------------------------------------------- *
 *  DemoFusion extras (tile_methods/demofusion.py).
 * ------------------------------------------------------------------------- */

/* Dilated global views -- demofusion.py:283-308: out[(v*N+n), c, i, j] = src_v[n, c, by_v + i*s, bx_v + j*s],
 * src_v = x1 where view_second[v] (mixture mode: the blurred latent) else x0.  Host int arrays of n_views,
 * 1 <= n_views <= 64 per launch.  Any offsets with 0 <= bx, bx + (out_w - 1) * s < W and 0 <= by,
 * by + (out_h - 1) * s < H are gathered; others are refused with TD_ERR_INVALID_ARG. */
int td_dilated_gather(const void* x0, const void* x1, void* out, int N, int C, int H, int W, int s,
                      int out_h, int out_w, const int32_t* view_bx, const int32_t* view_by,
                      const int32_t* view_second, int n_views, int dtype, void* stream);

/* demofusion.py:296-322 fused: strided `x_global[:, :, by::s, bx::s] += view` in view order (each add
 * rounded through dtype), `/ 2` in mixture mode, and out = x_local*(1-c2) + x_global*c2 (each product and
 * the sum rounded through dtype).  view_batch_ptrs: HOST array of DEVICE pointers, batch b holding
 * views [b*views_per_batch, ...) as [.*N, C, out_h, out_w].  Pixels with y >= end_y or x >= end_x get
 * x_global = 0 (the reference's `end = W - jitter_range` slice bound, demofusion.py:280).  Refused with
 * TD_ERR_INVALID_ARG before any launch: s <= 0, a non-positive size, end_y > H, end_x > W, and views that
 * do not cover [0, end_y) x [0, end_x), i.e. (end_y - 1) / s >= out_h or (end_x - 1) / s >= out_w. */
int td_demofusion_combine(const void* x_local, const void* const* view_batch_ptrs, int num_batches,
                          int views_per_batch, int n_views, void* out, int N, int C, int H, int W, int s,
                          int out_h, int out_w, int end_y, int end_x, int mixture, float c2,
                          float one_minus_c2, int dtype, void* stream);

/* Random-jitter mode (demofusion.py:101-139): the local windows carry individual random offsets on the zero-padded
 * latent, i.e. an arbitrary window LIST instead of the separable td_grid.  origins_dev: DEVICE int32 [n_tiles][2]
 * (x, y) in canvas coordinates; origins_host: the same values on the host for bounds validation (may be NULL).
 *
 * td_scatter_bboxes: tiles[(t*N+n), c, v, u] = x[n, c, y_t+v, x_t+u]                       (demofusion.py:256)
 * td_blend_bboxes:   out fp32 [N,C,H,W] = acc / max(count, 1): the windows covering a pixel are added in list
 *   order, each add rounded through dtype; count = number of covering windows           (demofusion.py:259-264).
 *   batch_ptrs as in td_blend_multidiffusion (batch b holds windows [b*tile_bs, ...)). */
int td_scatter_bboxes(const void* x, void* tiles, const int32_t* origins_dev, const int32_t* origins_host, int n_tiles,
                      int N, int C, int H, int W, int tile_h, int tile_w, int dtype, void* stream);
int td_blend_bboxes(const void* const* batch_ptrs, int num_batches, int tile_bs, const int32_t* origins_dev,
                    const int32_t* origins_host, int n_tiles, int N, int C, int H, int W, int tile_h, int tile_w,
                    int dtype, float* out, void* stream);

/* td_demofusion_combine with the dilated views starting at offset + (by, bx) (offset = jitter_range,
 * demofusion.py:279-310): pixels with y < offset, x < offset, y >= end_y or x >= end_x get x_global = 0. */
int td_demofusion_combine_offset(const void* x_local, const void* const* view_batch_ptrs, int num_batches,
                                 int views_per_batch, int n_views, void* out, int N, int C, int H, int W, int s,
                                 int out_h, int out_w, int offset, int end_y, int end_x, int mixture, float c2,
                                 float one_minus_c2, int dtype, void* stream);

/* gaussian_filter -- demofusion.py:173-178: depthwise k x k convolution, zero padding k/2, fp32
 * accumulate, result rounded to dtype.  kernel_host: k*k fp32 values (already rounded through dtype). */
int td_depthwise_conv2d(const void* in, void* out, int planes, int H, int W, const float* kernel_host,
                        int k, int dtype, void* stream);

/* Seamless DemoFusion (new: the reference has no periodic canvas).  `wrap` = TD_WRAP_X | TD_WRAP_Y names the periodic
 * axes; unknown bits are refused with TD_ERR_INVALID_ARG.
 *
 * td_depthwise_conv2d_wrap: td_depthwise_conv2d with circular indexing on the wrapped axes and zero padding on the
 *   bounded ones; the same taps, tap order and fp32 fmaf accumulation.  Refused: k/2 > L on a wrapped axis of length L.
 *   wrap = 0 runs the kernel of td_depthwise_conv2d.
 * td_scatter_bboxes_wrap / td_blend_bboxes_wrap: td_scatter_bboxes / td_blend_bboxes on a window list whose origins
 *   (canvas coordinates, no padding) may cross the canvas edge.  A window covers rows (y_t + v) mod H on a wrapped y axis
 *   and y_t + v on a bounded one, where the scatter reads 0 outside [0, H) and the blend drops those pixels (the
 *   reference's zero pad, slice and crop without materialising the pad); the same in x.  origins_host is REQUIRED.
 *   Refused before any launch: on a wrapped axis an origin outside [0, L) or tile > L; on a bounded axis an origin
 *   outside [-(tile - 1), L - 1]. */
int td_depthwise_conv2d_wrap(const void* in, void* out, int planes, int H, int W, const float* kernel_host,
                             int k, int wrap, int dtype, void* stream);
int td_scatter_bboxes_wrap(const void* x, void* tiles, const int32_t* origins_dev, const int32_t* origins_host,
                           int n_tiles, int N, int C, int H, int W, int tile_h, int tile_w, int wrap, int dtype,
                           void* stream);
int td_blend_bboxes_wrap(const void* const* batch_ptrs, int num_batches, int tile_bs, const int32_t* origins_dev,
                         const int32_t* origins_host, int n_tiles, int N, int C, int H, int W, int tile_h, int tile_w,
                         int wrap, int dtype, float* out, void* stream);

/* ------------------------------------------------------------------------- *
 *  Tiled-VAE dense contractions on the tensor cores (wgmma, fp32 accumulators in registers).
 *  The reference executes its conv / attention tasks at scripts/tilevae.py:618 through third-party
 *  ldm modules (queue built at :107-204; attention tile_utils/attn.py:49-72).
 * ------------------------------------------------------------------------- */

/* One convolution (or GEMM) over NHWC activations:
 *   y[n, oy, ox, co] = alpha * sum_{ky, kx, ci} x[n, oy*stride + ky - pad_top, ox*stride + kx - pad_left, ci] * w[ky*kw + kx][co][ci]
 *                      + bias (+ residual[n, oy, ox, co])
 * out-of-range input pixels read as zero (the conv's zero padding; pad(0,1,0,1) + stride 2 is pad_top = pad_left = 0).
 * x: [N, H, W, x_pitch >= Cin], w: [kh*kw][Cout][w_pitch >= Cin], y / residual: [N, OH, OW, pitch >= Cout]; fp16 or bf16;
 * Cin % 8 == 0 (zero-pad narrower inputs; K is walked in chunks of 64, a partial last chunk reads zeros), pitches in
 * elements and multiples of 8; fp32 accumulation.
 * bias: fp32 [Cout] (bias_per_row = 0) or fp32 [N*OH*OW] (bias_per_row = 1: per output pixel = per GEMM row), or NULL.
 * A GEMM D[M, Nc] = A[M, K] B[Nc, K]^T is N = H = OH = 1, W = OW = M, Cin = K, Cout = Nc, kh = kw = 1. */
typedef struct td_conv_desc {
    int32_t N, H, W, Cin, Cout;
    int32_t kh, kw, stride, pad_top, pad_left;
    int32_t OH, OW;
    int32_t dtype;          /* TD_F16 or TD_BF16 */
    int32_t bias_per_row;
    float alpha;
    int64_t x_pitch, w_pitch, y_pitch, res_pitch;
    /* optional epilogue stage: y = act(y * post_scale[co] + post_shift[co]) (fp32 [Cout] each, device; act 1 = SiLU) --
     * the GroupNorm (+ SiLU) that follows the convolution when its statistics are already known (fast mode) */
    const float* post_scale;
    const float* post_shift;
    int32_t post_act;
    /* optional second output (NULL: none): with y2 set, y receives the result BEFORE the post stage (what the next
     * ResnetBlock adds back as its shortcut) and y2 [N, OH, OW, y2_pitch >= Cout] the result after it (that block's
     * normalised + activated input): the GroupNorm pass over the activation disappears */
    void* y2;
    int64_t y2_pitch;
} td_conv_desc;
int td_conv2d_nhwc(const td_conv_desc* d, const void* x, const void* w, const float* bias, const void* residual,
                   void* y, void* stream);

/* ldm's Upsample block -- F.interpolate(scale_factor=2, mode="nearest") then a 3x3 / pad 1 convolution ('upsample' task +
 * the 'conv' that follows it, tilevae.py:163-166) -- WITHOUT materialising the upsampled tensor: output pixel (2i+py, 2j+px)
 * only ever sees the 2x2 low-resolution neighbourhood {i-1+py, i+py} x {j-1+px, j+px}, so the block is four 2x2
 * convolutions of the low-resolution image, one per output parity, with the 3x3 taps that fall on the same source pixel
 * summed (4/9 of the multiply-adds, no 4x intermediate in HBM).  `d` describes the block as the reference sees it:
 * H x W input, OH = 2H, OW = 2W, kh = kw = 3, stride 1, pad 1; w16: folded taps [16 = (py*2+px)*4 + ty*2 + tx][Cout][w_pitch]
 * (fold in fp32, round once: vae_ops.fold_upsample_weight); no residual; the post_scale / post_shift stage applies. */
int td_upconv2x_nhwc(const td_conv_desc* d, const void* x, const void* w16, const float* bias, void* y, void* stream);

/* The mid-block's single-head attention core (tile_utils/attn.py:49-72: q·kᵀ scaled by alpha, softmax over the keys,
 * times v) fused into one kernel with an online softmax (csrc/td_attn.cu):
 *   o[t, :] = softmax_s(alpha * sum_c q[t, c] k[s, c]) v[s, :]      t, s < T
 * q / k / v / o: token-major [T, pitch >= C] fp16 or bf16 (pitches in elements, multiples of 8; 16-byte aligned);
 * fp32 accumulation; C % 64 == 0 and C <= 512 (else TD_ERR_UNSUPPORTED); any T >= 1.  Nothing of size T x T is
 * written: the call needs no memory beyond its four operands.  One rounding of o to the storage dtype. */
int td_attention(const void* q, const void* k, const void* v, void* o, int T, int C, int64_t q_pitch, int64_t k_pitch,
                 int64_t v_pitch, int64_t o_pitch, float alpha, int dtype, void* stream);

/* Channels-last (NHWC) streaming kernels around the tensor-core convolutions (csrc/td_nhwc.cu).  fp16 / bf16.
 *
 * td_nchw_to_nhwc: tile crop (tilevae.py:532-535) + layout change + channel zero-padding:
 *   y[n, i, j, c] = c < C ? x[n*x_img_stride + c*x_plane_stride + i*x_pitch + j] : 0,  y: [N, rows, cols, Cpad] contiguous.
 * td_nhwc_to_nchw_region: crop_valid_region + paste (tilevae.py:248-259, :632) + layout change back:
 *   y[n*y_img_stride + c*y_plane_stride + i*y_pitch + j] = x[n*x_img_stride + (i*x_width + j)*x_pitch + c], c < C
 *   (x / y already offset to the region origins; strides and pitches in elements).
 * td_upsample2x_nhwc: F.interpolate(scale_factor=2, mode="nearest") of ldm's Upsample ('upsample' task, tilevae.py:163).
 * td_gn_stats_nhwc: get_var_mean (tilevae.py:207-215) of ONE image x: [pixels, C]; mean / var: fp32 [groups], biased.
 * td_gn_apply_nhwc: custom_group_norm (+ SiLU when act = 1) (tilevae.py:218-245, :102-104); y may alias x.
 * td_softmax_rows: y[r, :cols] = softmax(x[r, :cols]) (tile_utils/attn.py:58-60), y[r, cols:pitch] = 0. */
int td_nchw_to_nhwc(const void* x, void* y, int N, int C, int rows, int cols, int64_t x_img_stride,
                    int64_t x_plane_stride, int64_t x_pitch, int Cpad, int dtype, void* stream);
/* td_nchw_to_nhwc of a tile of a periodic canvas: y[n, i, j, c] = x[n, c, (row0 + i) mod H, (col0 + j) mod W] (c < C, else 0);
 * x points at the canvas origin of image 0, row0 / col0 may be negative or run past the canvas (seamless tiling). */
int td_nchw_to_nhwc_wrap(const void* x, void* y, int N, int C, int rows, int cols, int row0, int col0, int H, int W,
                         int64_t x_img_stride, int64_t x_plane_stride, int64_t x_pitch, int Cpad, int dtype, void* stream);
int td_nhwc_to_nchw_region(const void* x, void* y, int N, int C, int rows, int cols, int64_t x_img_stride,
                           int x_width, int64_t x_pitch, int64_t y_img_stride, int64_t y_plane_stride,
                           int64_t y_pitch, int dtype, void* stream);
int td_upsample2x_nhwc(const void* x, void* y, int N, int H, int W, int C, int dtype, void* stream);
int64_t td_gn_stats_nhwc_workspace_bytes(int64_t pixels, int C, int groups);
int td_gn_stats_nhwc(const void* x, int64_t pixels, int C, int groups, int dtype, void* workspace,
                     int64_t workspace_bytes, float* mean, float* var, void* stream);
int td_gn_apply_nhwc(const void* x, void* y, int64_t pixels, int C, int groups, int dtype, const float* mean,
                     const float* var, const float* gamma, const float* beta, float eps, int act, void* stream);
int td_softmax_rows(const void* x, void* y, int rows, int cols, int64_t pitch, int dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TD_B200_H */
