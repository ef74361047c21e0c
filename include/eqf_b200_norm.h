/* eqf_b200_norm.h - C ABI of libeqf_b200_norm.so: the per-graph equivariant norms.
 *
 * EquivariantGraphNorm (reference nets/graph_norm.py:9-134) and EquivariantInstanceNorm (nets/instance_norm.py:9-134)
 * normalise every irreps entry over the nodes of each graph of the batch.  Per entry [N][2l+1][mul] (planar, as in
 * eqf_b200.h) and per graph g with nodes ptr[g] .. ptr[g+1]-1, channel c:
 *
 *   0e entries:   m[g][c] = mean_i x[i][0][c],   z = x - shift[c] * m[g][c]   (shift = 1 for the instance norm)
 *   other ones:   z = x
 *   every entry:  v[g][c] = mean_i (mean or sum over the 2l+1 components of z^2),  r = (v + eps)^-1/2
 *                 y = z * r * w[c]  (+ b[c] on 0e entries)
 *
 * The statistics are fixed-order segmented reductions (no atomics): runs are bitwise reproducible.  A graph without
 * nodes gets m = 0, v = 0 and writes nothing.  Conventions as in eqf_b200.h: device pointers, fp32 data, int64 indices,
 * `stream` is a cudaStream_t, 0 = ok, negative = error with a message from eqf_last_error().
 */
#ifndef EQF_B200_NORM_H_
#define EQF_B200_NORM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EQF_NORM_MAX_ENTRIES 8

/* One per norm module.  Channel offsets are prefix sums of mul: w_off over all entries (affine_weight),
 * s_off over the 0e entries (affine_bias and the [G][n_s] mean columns).  The mean shift of a 0e entry is read at
 * shift[c], c < mul, for every 0e entry: nets/graph_norm.py:90 never advances its offset. */
typedef struct {
  int32_t n_entries;
  int32_t mul[EQF_NORM_MAX_ENTRIES];
  int32_t d[EQF_NORM_MAX_ENTRIES];          /* 2l+1 */
  int32_t is_scalar[EQF_NORM_MAX_ENTRIES];  /* 1: 0e entry (centred, biased) */
  int32_t w_off[EQF_NORM_MAX_ENTRIES];
  int32_t s_off[EQF_NORM_MAX_ENTRIES];      /* -1 for entries that are not 0e */
  int32_t n_w;                              /* sum of mul */
  int32_t n_s;                              /* sum of mul over 0e entries */
  int32_t component;                        /* 1: 'component' (mean over 2l+1), 0: 'norm' (sum) */
  float eps;
} EqfSegNormLayout;

const char* eqf_last_error(void);

/* graph_ptr[g] = first node i with batch[i] >= g, g = 0 .. n_graphs (batch ascending, [N]) */
int eqf_norm_graph_ptr(const int64_t* batch, int64_t N, int64_t n_graphs, int64_t* graph_ptr, void* stream);

/* Forward: y blocks as x; mean [G][n_s], rstd [G][n_w] saved for the backward.  shift may be NULL (instance norm). */
int eqf_norm_fwd(const EqfSegNormLayout* lay, const float* const* x_blocks, const int64_t* graph_ptr, int64_t n_graphs,
                 const float* shift, const float* w, const float* b, float* const* y_blocks, float* mean, float* rstd,
                 void* stream);

/* Backward: gx blocks, and per-graph parameter partials part[G][n_w + 2 n_s] = d w | d b | d shift, which
 * eqf_norm_param_reduce sums over the graphs in ascending order into out[n_w + 2 n_s]. */
int eqf_norm_bwd(const EqfSegNormLayout* lay, const float* const* x_blocks, const float* const* gy_blocks,
                 const int64_t* graph_ptr, int64_t n_graphs, const float* shift, const float* w, const float* mean,
                 const float* rstd, float* const* gx_blocks, float* part, void* stream);
int eqf_norm_param_reduce(const float* part, int64_t n_graphs, int32_t cols, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
