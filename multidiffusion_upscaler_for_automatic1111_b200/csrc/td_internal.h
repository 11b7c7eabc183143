// Internal helpers shared by the translation units of libtd_b200.so.
#pragma once
#include <stdint.h>

void td_set_error(const char* fmt, ...);

static inline int td_dtype_size(int dtype) { return dtype == 2 /*TD_F32*/ ? 4 : ((dtype == 0 || dtype == 1) ? 2 : 0); }

// td_strip.cu: strip form of the MultiDiffusion blend (TD_FLAG_STRIP).  TD_OK launched, 1 not applicable, < 0 error.
struct td_grid;
int td_strip_try_launch(const struct td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                        const float* weights, const float* rcp_weights, float* x_out, void* x_buffer, int pdl, int max_ppc, void* stream);
int td_strip_try_launch_mod(const struct td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                            const float* tile_weights, const float* rescale, void* x_buffer, int pdl, void* stream);

// td_rows.cu: row-block form (one persistent CTA per SM, bulk-copy staging) of scatter / blend.  TD_OK launched, 1 not
// applicable (caller falls back to td_diffusion.cu), < 0 error.
int td_rows_try_launch_md(const struct td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                          const float* weights, const float* rcp_weights, float* x_out, void* x_buffer, int pdl, int dbg_no_tiles,
                          void* stream);
int td_rows_try_launch_mod(const struct td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                           const float* tile_weights, const float* rescale, void* x_buffer, int pdl, void* stream);
int td_rows_try_launch_scatter(const struct td_grid* g, const void* x, void* tiles, int N, int C, int dtype, int tile_begin, int tile_end,
                               int pdl, void* stream);

// td_wrap.cu: scatter / blends on a periodic canvas (g->wrap != 0).  Called by the C-ABI entries of td_diffusion.cu after
// they validated the grid and the batch table; `vec`: their vector-path test passed (else one element per thread, any
// width, alignment or dtype pair).  mixture: 0 MultiDiffusion, 1 Mixture of Diffusers.
int td_wrap_scatter(const struct td_grid* g, const void* x, void* tiles, int N, int C, int dtype, int tile_begin, int tile_end,
                    bool vec, bool pdl, void* stream);
int td_wrap_blend(const struct td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype,
                  int acc_dtype, int mixture, const float* weights, const float* tile_weights, const float* rescale, float* x_out,
                  void* x_buffer, bool vec, bool pdl, void* stream);
// Row-strip shard on a periodic canvas (td_blend_*_wrap_rows, vector path only, arguments validated by the caller): the blend
// of the canvas rows [row_begin, row_end) (non-empty), waiting in-kernel for the halo bands.
int td_wrap_blend_rows(const struct td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype,
                       int mixture, const float* weights, const float* tile_weights, const float* rescale, float* x_out, void* x_buffer,
                       int row_begin, int row_end, const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                       int own_band_begin, int own_band_end, bool pdl, void* stream);
