/* eqf_b200.h - C ABI of libeqf_b200.so, the sm_90a edge kernels behind the Equiformer hot path.
 *
 * The reference (atomicarchitects/equiformer) has no FFI layer of its own: the boundary is the
 * Python nn.Module surface of nets/tensor_product_rescale.py and nets/graph_attention_transformer.py
 * (SURVEY.md section 8b).  This library sits *under* the drop-in modules in equiformer_b200/nets and
 * is bound with ctypes (equiformer_b200/_lib.py).  Each entry point names the reference code whose
 * GPU work it replaces.  Conventions:
 *
 *   - every pointer is a DEVICE pointer unless marked "host"; tensors are fp32, index arrays int64;
 *   - "planar" layout: an irrep block (mul x degree l) of R rows is stored as [R][2l+1][mul]
 *     (component-major, channel innermost), one buffer per block; this is the e3nn layout
 *     [R][mul][2l+1] transposed per row, chosen so that lanes = channels gives coalesced access and
 *     the per-degree channel-mixing linears that follow are plain row-major GEMMs;
 *   - `stream` is a cudaStream_t passed as void*; launches are asynchronous on it;
 *   - return value 0 = ok, negative = error; eqf_last_error() returns a thread-local message;
 *   - no global state except immutable plans owned by the caller.
 */
#ifndef EQF_B200_H_
#define EQF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EQF_MAX_BLOCKS 8   /* max irrep blocks per operand (in1 blocks / output groups / value groups) */
#define EQF_MAX_HEADS 16

#define EQF_OK 0
#define EQF_ERR_INVALID (-1)
#define EQF_ERR_CUDA (-2)
#define EQF_ERR_UNSUPPORTED (-3)

typedef struct EqfPlan EqfPlan;

/* One Clebsch-Gordan path of a depth-wise ('uvu', mul(in2)=1) tensor product:
 * reference instruction (i_in1, i_in2, i_out, 'uvu', True) built at
 * nets/graph_attention_transformer.py:166-172 and executed by o3.TensorProduct inside
 * TensorProductRescale (nets/tensor_product_rescale.py:33-37, :126). */
typedef struct {
  int32_t l1, l2, l3;      /* degrees of in1 block, in2 (edge SH) irrep, output irrep            */
  int32_t mul;             /* channels u of the in1 block                                         */
  int32_t in1_block;       /* index into the in1 block list                                      */
  int32_t in2_off;         /* float offset of the degree-l2 SH inside one edge_attr row          */
  int32_t out_group;       /* index of the output group (all paths with equal (l3,p3), sorted)   */
  int32_t out_chan_off;    /* first channel of this path inside its output group                 */
  int32_t w_off;           /* float offset of this path's [mul] weights in a weight row          */
  int32_t cg_off;          /* float offset into `cg`: dense [2l1+1][2l2+1][2l3+1], path weight folded in */
} EqfPathDesc;

/* Operand bundle shared by the four contraction kernels.  Unused members are NULL. */
typedef struct {
  const float* x[EQF_MAX_BLOCKS];    /* in1 blocks, planar [Rx][2l1+1][mul]                        */
  const float* x2[EQF_MAX_BLOCKS];   /* optional second table added to x (gathered by `dst`)      */
  const int64_t* src;                /* optional: row of x used by edge e (NULL: row e)           */
  const int64_t* dst;                /* row of x2 used by edge e (required iff x2[0] != NULL)     */
  const float* y;                    /* edge_attr (SH), [E][d_y]                                  */
  const float* w;                    /* per-edge weights [E][W] or shared [W]                     */
  int32_t w_shared;                  /* 1: w is [W] (internal weights), 0: [E][W]                 */
  const float* g[EQF_MAX_BLOCKS];    /* output-group tensors (cotangents), planar [E][2l3+1][K]   */
  const float* w_offset;             /* optional [W]: the kernels use w[e] + w_offset (RadialProfile's offset,
                                        nets/radial_func.py:45-49, folded into the weight load); may be NULL.
                                        Only the plan-specialised kernels take it (EQF_ERR_UNSUPPORTED otherwise) */
} EqfEdgeOperands;

int eqf_version(void);
const char* eqf_last_error(void);
int eqf_device_sm_count(void);

/* Build the immutable device tables for one depth-wise tensor product
 * (DepthwiseTensorProduct, nets/graph_attention_transformer.py:157-183).  All arrays are host. */
int eqf_plan_create(const EqfPathDesc* paths, int32_t n_paths,
                    const int32_t* in1_l, const int32_t* in1_mul, int32_t n_in1,
                    const int32_t* out_l, const int32_t* out_mul, int32_t n_out,
                    int32_t d_y, int32_t weight_numel,
                    const float* cg, int32_t cg_len, EqfPlan** plan_out);
void eqf_plan_destroy(EqfPlan* plan);
/* host-side introspection: out[0..n) = {n_paths, m_size, n_wtasks, n_xtasks, tile_edges, smem_bytes, blob_words,
 * weight_numel, vec_ok, n_vwtasks, n_vxtasks, smem_bytes_vec_fwd, has_generated_kernels} */
int eqf_plan_info(const EqfPlan* plan, int32_t* out, int32_t n);
/* number of CTAs eqf_dtp_grad_w launches (rows of the shared-weight partial buffer) */
int eqf_plan_partial_rows(const EqfPlan* plan, int64_t n_edges);

/* out[g][e,k,koff+u] = w[e,p,u] * sum_ij cg_p[i,j,k] x[e,i,u] y[e,j]
 * == TensorProductRescale.forward(x, y, weight) for the DTP (tensor_product_rescale.py:139-141),
 * optionally with the gather+add of graph_attention_transformer.py:487 folded into the x load. */
int eqf_dtp_forward(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                    float* const* out_groups /* host array[n_out] of device ptrs */, void* stream);

/* d/dx of <g, forward>: gx[b][e,i,u] (what autograd derives for the e3nn TP in the reference). */
int eqf_dtp_grad_x(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                   float* const* gx_blocks /* host array[n_in1] */, void* stream);

/* d/dw: per-edge gw[E][W], or for shared weights per-CTA partial sums gw[partial_rows][W]
 * (caller reduces over rows; deterministic). */
int eqf_dtp_grad_w(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                   float* gw, void* stream);

/* d/dy: gy[E][d_y] (needed for MD17 forces, graph_attention_transformer_md17.py:318-325).  x is read per edge: op->src
 * must be NULL (EQF_ERR_UNSUPPORTED otherwise). */
int eqf_dtp_grad_y(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                   float* gy, void* stream);

/* gx and gw in one pass over g (first-order training path). gw as in eqf_dtp_grad_w. */
int eqf_dtp_grad_xw(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                    float* const* gx_blocks, float* gw, void* stream);

/* ---- attention softmax + aggregation over destination-sorted edges ------------------------------
 * Value tensors are `n_groups` planar buffers [rows][d[g]][C[g]]; head h owns channels
 * [h*C/H, (h+1)*C/H) of every group (Vec2AttnHeads, graph_attention_transformer.py:252-285).      */
typedef struct {
  int32_t n_groups;
  int32_t d[EQF_MAX_BLOCKS];
  int32_t C[EQF_MAX_BLOCKS];
  int32_t n_heads;
} EqfHeadLayout;

/* alpha[e,h] = exp(z[e,h]-max_seg)/(sum_seg exp + 1e-16): torch_geometric.utils.softmax(alpha, edge_dst)
 * at graph_attention_transformer.py:508 (PyG 2.0.3 semantics).  row_ptr is the CSR of edge_dst.   */
int eqf_seg_softmax(const float* z, const int64_t* row_ptr, int64_t n_nodes, int32_t n_heads,
                    float* alpha, void* stream);
/* its backward: gz[e,h] = alpha[e,h] (ga'[e,h] - sum_{f -> dst(e)} alpha[f,h] ga'[f,h]) with ga' = ga * keep, where
 * keep [E][H] (may be NULL: ga' = ga) is the attention-dropout mask that followed the softmax (:509).           */
int eqf_seg_softmax_bwd(const float* alpha, const float* ga, const float* keep, const int64_t* row_ptr, int64_t n_nodes,
                        int32_t n_heads, float* gz, void* stream);

/* out[g][t,j] = sum_{e in seg(t)} alpha[e,head(j)] * V[g][e,j]   (alpha NULL: plain segment sum)
 * == value*alpha followed by torch_scatter.scatter(..., edge_dst) (:512-513).
 * perm (optional, NULL = identity): segment position -> edge id, for segments of an index the edge list is not
 * sorted by (the transpose of `message_src[edge_src]`, :487, in the backward pass).                */
int eqf_attn_aggregate(const EqfHeadLayout* lay, const float* alpha, const float* const* V,
                       const int64_t* row_ptr, const int64_t* perm, int64_t n_nodes, float* const* out, void* stream);
/* K2 - the PyG segment softmax (nets/graph_attention_transformer.py:508) and the attention-weighted scatter (:512-513)
 * in ONE kernel over the destination-sorted edge list: out[g][t] = sum_{e->t} softmax_t(z)[e, head] V[g][e], one warp per
 * (node, 128 columns), no atomics; alpha [E][H] (the softmax itself) is written once for the backward.  Needs the float4
 * layout and a leading 0e group (EQF_ERR_UNSUPPORTED otherwise - callers fall back to eqf_seg_softmax + eqf_attn_aggregate). */
/* keep [E][H] (may be NULL) is the attention-dropout mask (:509), entries 0 or 1/(1-p): the sum then runs over
 * softmax * keep * V, while alpha is still written without the mask (the softmax backward needs it).                */
int eqf_attn_softmax_aggregate(const EqfHeadLayout* lay, const float* z, const float* keep, const float* const* V,
                               const int64_t* row_ptr, int64_t n_nodes, float* const* out, float* alpha, void* stream);

/* Dot-product attention (nets/dp_attention_transformer.py:145-151) in ONE kernel over the destination-sorted edge list:
 * z[e,h] = sum_{j in head h} q[g][dst e, j] k[g][e, j] over all groups, alpha = the PyG segment softmax of z (+1e-16),
 * out[g][t] = sum_{e->t} alpha[e, head] keep[e, head] v[g][e].  `lay` is the q / out layout [N][d_g][C_g]; the keys and
 * values are read from the key / value blocks kv[g] [E][d_g][2 C_g] (keys in channels [0, C_g), values in [C_g, 2 C_g)).
 * keep [E][H] (may be NULL) is the attention-dropout mask (entries 0 or 1/(1-p)); alpha [E][H] is written unmasked for
 * the backward.  One warp per node, no atomics, deterministic; zero-in-degree nodes get zeros.  Needs channels per head
 * % 4 == 0, at most 1024 channels per node row and 1 / 2 / 4 / 8 / 16 heads (EQF_ERR_UNSUPPORTED otherwise).      */
int eqf_attn_dot_softmax_aggregate(const EqfHeadLayout* lay, const float* const* q, const float* const* kv,
                                   const float* keep, const int64_t* row_ptr, int64_t n_nodes, float* const* out,
                                   float* alpha, void* stream);
/* its first-order backward, G[g] = d L / d out [N][d_g][C_g]: with ga = v . G[t] per head and s_t = sum alpha keep ga,
 * gz = alpha (keep ga - s_t); gkv[g] [E][d_g][2 C_g] gets gk = gz q[t] in the key channels and gv = alpha keep G[t] in
 * the value channels, gq[g] [N][d_g][C_g] = sum_e gz k.  work [E][H] is scratch (it ends up holding ga).  Same layout
 * rules; no atomics.                                                                                                */
int eqf_attn_dot_softmax_aggregate_bwd(const EqfHeadLayout* lay, const float* const* G, const float* const* q,
                                       const float* const* kv, const float* alpha, const float* keep,
                                       const int64_t* row_ptr, int64_t n_nodes, float* const* gq, float* const* gkv,
                                       float* work, void* stream);

/* Linear-message graph attention (nets/graph_attention_transformer.py:497-513, nonlinear_message=False) in ONE kernel
 * over the destination-sorted edge list, from the 0e output of sep.lin (bias included) read in place: t0 [E][H (A+R)],
 * head h owning the alpha pre-activations [h(A+R), h(A+R)+A) and the value scalars [h(A+R)+A, (h+1)(A+R)) (Vec2AttnHeads).
 *   z[e,h] = sum_k c_slr SLR(t0[e, h(A+R)+k]) alpha_dot[h,k],  SLR(x) = (1+s)/2 x + (1-s)/2 x (2 sigmoid(x) - 1), s = slope;
 *   alpha  = the PyG segment softmax of z (+1e-16);
 *   out[g][t] = sum_{e->t} alpha[e, head] keep[e, head] v[g][e], v[0] = the value scalars, v[g >= 1] = V[g-1].
 * `lay` is the output layout: group 0 [N][1][H R], groups g >= 1 [N][d_g][H C_g]; V holds the n_groups - 1 blocks
 * [E][d_g][H C_g] of the l >= 1 values.  alpha_dot [H][A]; keep [E][H] (may be NULL) is the attention-dropout mask
 * (entries 0 or 1/(1-p)); alpha [E][H] is written unmasked for the backward.  One warp per node in a grid of
 * eqf_attn_mlp_rows(n_nodes) CTAs, no atomics, deterministic; zero-in-degree nodes get zeros.  Needs 2 / 4 / 8 heads, A,
 * R and every C_g multiples of 4, at most 128 alpha and 512 value channels per edge with 2 or 4 heads (256 and 640 with
 * 8), 16-byte aligned operands (EQF_ERR_UNSUPPORTED / EQF_ERR_INVALID otherwise).                                     */
int eqf_attn_mlp_rows(int64_t n_nodes);
int eqf_attn_mlp_softmax_aggregate(const EqfHeadLayout* lay, int32_t n_alpha, float c_slr, float slope, const float* t0,
                                   const float* const* V, const float* alpha_dot, const float* keep,
                                   const int64_t* row_ptr, int64_t n_nodes, float* const* out, float* alpha, void* stream);
/* its first-order backward, G[g] = d L / d out [N][d_g][H C_g]: with ga = v . G[t] per head, s_t = sum alpha keep ga
 * and gz = alpha (keep ga - s_t), gt0 [E][H (A+R)] gets gz alpha_dot c_slr SLR'(t0) in the alpha channels and
 * alpha keep G[0][t] in the value channels (every channel written), gV[g-1] = alpha keep G[g][t], and
 * gdot_part [eqf_attn_mlp_rows(n_nodes)][H A] the per-CTA partial sums of d L / d alpha_dot = sum_e gz c_slr SLR(t0)
 * (reduce the rows with eqf_colsum).  work [E][H] is scratch.  Same layout rules; no atomics: bitwise repeatable.      */
int eqf_attn_mlp_softmax_aggregate_bwd(const EqfHeadLayout* lay, int32_t n_alpha, float c_slr, float slope,
                                       const float* const* G, const float* t0, const float* const* V,
                                       const float* alpha_dot, const float* alpha, const float* keep,
                                       const int64_t* row_ptr, int64_t n_nodes, float* gt0, float* const* gV,
                                       float* work, float* gdot_part, void* stream);

/* galpha[e,h] = sum_{j in head h} V[g][e,j] * G[g][dst[e],j]       (transpose of aggregate w.r.t. alpha) */
int eqf_attn_edge_dot(const EqfHeadLayout* lay, const float* const* V, const float* const* G,
                      const int64_t* dst, int64_t n_edges, float* galpha, void* stream);

/* out[g][e,j] = alpha[e,head(j)] * keep[e,head(j)] * G[g][dst[e],j]  (transpose w.r.t. V; alpha NULL: gather;
 * keep NULL: no mask; keep needs alpha)                                                                              */
int eqf_attn_edge_scale(const EqfHeadLayout* lay, const float* alpha, const float* keep, const float* const* G,
                        const int64_t* dst, int64_t n_edges, float* const* out, void* stream);

/* ---- fused pointwise kernels around the GEMMs -------------------------------------------------------------------
 * y = silu(LayerNorm(x + bias)) on [R, C] rows (C <= 256): Linear bias + LayerNorm + SiLU of the hidden layers of
 * RadialProfile (nets/radial_func.py:24-35); bias may be NULL.  The backward writes gx (= gradient of x and of the
 * broadcast bias) and per-CTA partial sums part[eqf_pointwise_rows(R)][3C] = d gamma | d beta | d bias.          */
int eqf_pointwise_rows(int64_t rows);
int eqf_ln_silu_fwd(const float* x, const float* bias, const float* gamma, const float* beta, float eps, int64_t R,
                    int32_t C, float* y, float* mean, float* rstd, void* stream);
int eqf_ln_silu_bwd(const float* x, const float* bias, const float* gamma, const float* beta, const float* mean,
                    const float* rstd, const float* gy, int64_t R, int32_t C, float* gx, float* part, void* stream);

/* Hand-written wgmma GEMM (3xTF32, fp32-level accuracy) for the tall per-degree linears: C[M, N] = A[M, K] x W, all
 * row-major fp32.  W is given as Bt[N, K] (b_is_kn = 0, data gradient: W = Bt^T) or as B[K, N] (b_is_kn = 1, forward);
 * `split` = device scratch of 2*N*K floats (hi / lo planes of the weights).  Replaces the e3nn 'uvw' einsum -> cuBLAS
 * SGEMM of LinearRS (nets/tensor_product_rescale.py:165-174). */
int eqf_gemm_tf32x3(const float* A, const float* Bt, float* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                    int64_t ldb, int64_t ldc, int32_t b_is_kn, float* split, void* stream);
/* Weight gradient of the same linears, W[K1, N] = A[R, K1]^T G[R, N] (what autograd derives for the 'uvw' einsum of
 * LinearRS): the R rows are cut into eqf_gemm_tf32x3_wgrad_slices(R, K1, N) slices, every CTA reduces one slice into a
 * register accumulator and writes partial[slice][K1][N]; the caller sums the partials over slices (eqf_colsum). */
int64_t eqf_gemm_tf32x3_wgrad_slices(int64_t R, int64_t K1, int64_t N);
int eqf_gemm_tf32x3_wgrad(const float* A, const float* G, float* partial, int64_t R, int64_t K1, int64_t N, int64_t lda,
                          int64_t ldg, void* stream);
/* same product written straight into W[K1, N]: W is zeroed, the slices add into it with fp32 atomics (order not fixed -
 * last-bit differences between runs, like the reference's atomic scatter) */
int eqf_gemm_tf32x3_wgrad_accumulate(const float* A, const float* G, float* W, int64_t R, int64_t K1, int64_t N,
                                     int64_t lda, int64_t ldg, void* stream);

/* K1 - the depth-wise tensor product fused into the per-degree linear that consumes it (the reference's
 * nets/graph_attention_transformer.py:487-496: dtp(message, edge_attr, weight) -> sep_alpha / lin; :725-733 for the
 * edge-degree embedding): for output group `group` of the plan
 *   C[(e, k), :N] = DTP_group(x, y; w)[(e, k), :K] @ Wt[:K, :N]
 * with the [E * (2 l3 + 1), K] tensor-product block produced ON CHIP as the register A operand of a wgmma 3xTF32
 * GEMM (csrc/eqf_fused.cu) - it never reaches HBM.  Operands as for eqf_dtp_forward (x gathered as x[src] + x2[dst] when
 * op->src is set; w per edge [E][W] (+ w_offset) or shared [W]).  Wt row-major [K][N], row stride ldw; C
 * [E * (2 l3 + 1)][N], row stride ldc; `split` = device scratch of 2 * N * K floats (hi / lo planes of Wt).
 * eqf_dtp_linear_supported: 1 when the group qualifies (path multiplicities % 32 == 0, tables fit shared memory). */
int eqf_dtp_linear_supported(const EqfPlan* plan, int32_t group);
/* debugging aid: device buffer of 6 * 2048 int64 receiving CTA 0's clock64 timeline of later fused launches (NULL = off) */
void eqf_fused_set_timeline(long long* device_buffer);
/* out[e][k][:K] = DTP_group(x, y; w): ONE output group of the product written to HBM, planar [E][2 l3 + 1][K] - the
 * operand of a linear too wide to fuse (N > 128 columns; e.g. the 224-channel 0e group in front of sep_alpha | lin). */
int eqf_dtp_group_forward(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, int32_t group, float* out,
                          void* stream);
int eqf_dtp_linear_fwd(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, int32_t group,
                       const float* Wt, int64_t N, int64_t ldw, float* C, int64_t ldc, float* split, void* stream);

/* Edge geometry in one kernel (nets/graph_attention_transformer.py:866-870; ..._oc20.py:283-296 with `offsets`):
 * vec = pos[src] - pos[dst] (+ offsets), len = |vec|, sh = real spherical harmonics of vec / |vec| up to lmax <= 4 in e3nn's
 * convention ('component' normalisation, y polar), [E][(lmax + 1)^2].  a1 [5][3][3], a2 [7][3][5], a3 [9][3][7]: coupling
 * tensors of the recurrence Y_{l+1} = A_l . (x (x) Y_l) (host: equiformer_b200/o3/sh.py; A_l may be NULL when l >= lmax).
 * _bwd: g_vec [E][3] from g_sh / g_len (either may be NULL); the scatter of g_vec to the positions is two segment sums
 * (eqf_attn_aggregate). */
int eqf_edge_geom_fwd(const float* pos, const int64_t* src, const int64_t* dst, const float* offsets, const float* a1,
                      const float* a2, const float* a3, int64_t E, int32_t lmax, float* vec, float* len, float* sh,
                      void* stream);
int eqf_edge_geom_bwd(const float* vec, const float* a1, const float* a2, const float* a3, int64_t E, int32_t lmax,
                      const float* g_sh, const float* g_len, float* g_vec, void* stream);
/* ExpNormalSmearing of the MD17 models (nets/expnorm_rbf.py:73-78 with CosineCutoff(0, cutoff_upper) :11-33):
 * out[e][b] = cutoff(d_e) exp(-betas[b] (exp(-alpha d_e) - means[b])^2); _bwd returns d/d d_e of <g, out>. */
int eqf_expnorm_fwd(const float* dist, const float* means, const float* betas, float alpha, float cutoff_upper, int64_t E,
                    int32_t B, float* out, void* stream);
int eqf_expnorm_bwd(const float* dist, const float* means, const float* betas, float alpha, float cutoff_upper, int64_t E,
                    int32_t B, const float* g, float* g_dist, void* stream);
/* Spherical Bessel radial basis of the Bessel configurations: ocpmodels 0.0.3 RadialBasis(B, cutoff,
 * rbf={'name': 'spherical_bessel'}) with its default polynomial envelope (p = 5), built at
 * nets/graph_attention_transformer.py:785-787, nets/graph_attention_transformer_md17.py:178-180 and
 * nets/equiformer_md17_dens.py:122-124.  With x = d_e / cutoff:
 * out[e][k] = env(x) sqrt(2 / cutoff^3) sin(freq[k] x) / x,  env(x) = 1 - 21 x^5 + 35 x^6 - 15 x^7 (x < 1, else 0).
 * B is a multiple of 4 in 4..128.  _bwd writes g_dist[E] = d <g, out> / d d_e (skipped when g_dist is NULL) and
 * per-CTA partial sums part[eqf_pointwise_rows(E)][B] of d <g, out> / d freq[k] (reduce with eqf_colsum). */
int eqf_bessel_fwd(const float* dist, const float* freq, float cutoff, int64_t E, int32_t B, float* out, void* stream);
int eqf_bessel_bwd(const float* dist, const float* freq, float cutoff, const float* g, int64_t E, int32_t B, float* g_dist,
                   float* part, void* stream);

/* Neighbour list of the batched molecules: edge (j -> i) iff same graph, j != i (unless loop), |pos_j - pos_i| < r, at
 * most max_neighbors per centre (the first ones in index order); sorted by centre, neighbours ascending - what
 * torch_cluster.radius_graph(pos, r, batch, max_num_neighbors) returns at nets/graph_attention_transformer.py:866-867.
 * count -> caller scans deg into row_ptr[n + 1] -> fill. */
int eqf_radius_graph_count(const float* pos, const int64_t* batch, int64_t n, float r_squared, int32_t loop,
                           int64_t max_neighbors, int64_t* deg, void* stream);
int eqf_radius_graph_fill(const float* pos, const int64_t* batch, int64_t n, float r_squared, int32_t loop,
                          int64_t max_neighbors, const int64_t* row_ptr, int64_t* src, int64_t* dst, void* stream);

/* Neighbour list under periodic boundary conditions - ocpmodels' radius_graph_pbc + the cell offsets get_pbc_distances
 * turns into edge vectors, as the OC20 model uses them (nets/graph_attention_transformer_oc20.py:267-302): edge
 * (j, image c) -> i iff same frame and 1e-4 < |pos_j + c . cell[frame] - pos_i|^2 <= r^2, images c in [-rep, rep] per lattice
 * vector; sorted by centre i, then atom j, then image.  cell [n_frames][3][3] (rows = lattice vectors), frame_ptr
 * [n_frames + 1] = first atom of each frame (batch ascending).  count -> scan -> fill (also returns the squared
 * distances, for the nearest-`max_neighbors` cut the caller applies when a centre exceeds it). */
int eqf_radius_graph_pbc_count(const float* pos, const int64_t* batch, const int64_t* frame_ptr, const float* cell,
                               int64_t n, float r_squared, int32_t rep_a, int32_t rep_b, int32_t rep_c, int64_t* deg,
                               void* stream);
int eqf_radius_graph_pbc_fill(const float* pos, const int64_t* batch, const int64_t* frame_ptr, const float* cell,
                              int64_t n, float r_squared, int32_t rep_a, int32_t rep_b, int32_t rep_c,
                              const int64_t* row_ptr, int64_t* src, int64_t* dst, int32_t* cell_offsets, float* dist2,
                              void* stream);

/* GaussianRadialBasisLayer with 128 basis functions (nets/gaussian_rbf.py:5-40): out[e, k] = exp(-z^2/2) / (a s_k),
 * z = (weight * dist_e / cutoff + bias - mean_k) / s_k, s_k = |std_k| + 1e-5, a = sqrt(2 * 3.14159); weight and bias
 * are one-element device tensors.  The backward
 * returns g_dist[E] and per-CTA partial sums part[eqf_pointwise_rows(E)][258] = d mean | d std | d weight | d bias. */
int eqf_rbf_fwd(const float* dist, const float* mean, const float* std, const float* weight, const float* bias,
                float cutoff, int64_t n_edges, float* out, void* stream);
int eqf_rbf_bwd(const float* dist, const float* mean, const float* std, const float* weight, const float* bias,
                float cutoff, const float* g, int64_t n_edges, float* g_dist, float* part, void* stream);

/* Column sums out[c] = sum_r x[r, c] (row stride ld): the bias / radial-offset gradients the reference gets from
 * autograd's broadcast reduction (nets/tensor_product_rescale.py:120-134, radial_func.py:45-49), and the final
 * reduction of per-CTA partial rows.  Deterministic (fixed summation order). */
#define EQF_COLSUM_COUNTERS 16384
int64_t eqf_colsum_scratch_floats(int64_t rows, int64_t cols);
int eqf_colsum(const float* x, int64_t rows, int64_t cols, int64_t ld, float* out, float* part, uint32_t* counters,
               void* stream);

/* Grouped fp32 GEMM for the SMALL products of the path: all degrees of a node-level linear (reference
 * nets/tensor_product_rescale.py:LinearRS -> e3nn 'uvw' with a scalar second operand = one [rows * (2l+1), mul_in] x
 * [mul_in, mul_out] product per degree; nets/graph_attention_transformer.py:430-431, :515, FeedForwardNetwork) - forward,
 * data gradients and weight gradients - in ONE launch of warp-MMA 3xTF32 tiles (replaces the per-degree cuBLAS calls).
 * Problem i: C[M, N] = alpha * op(A) op(B); mode 0: A[M, K] B[K, N], 1: A[M, K] B[N, K]^T, 2: A[K, M]^T B[K, N];
 * accumulate != 0: the reduction is split across CTAs and ADDED into C with fp32 atomics (C holds the initial value).
 * 16-byte aligned pointers; leading dimensions and every contiguous extent multiples of 4. */
#define EQF_GROUP_MAX 8
typedef struct {
  const float* A;
  const float* B;
  float* C;
  int64_t M, N, K, lda, ldb, ldc;
  int32_t mode;
  int32_t accumulate;
  float alpha;
  int32_t pad;
} EqfGemmProblem;
int eqf_gemm_grouped(const EqfGemmProblem* problems, int32_t n, void* stream);

/* EquivariantLayerNormV2 ('component' normalisation, affine; nets/layer_norm.py:89-152) on e3nn-layout rows:
 * one fused kernel forward, one backward (per-CTA partial sums of the affine gradients:
 * part[eqf_eln_rows(N)][n_weight + n_bias] = d weight | d bias). */
typedef struct {
  int32_t n_entries;
  int32_t mul[EQF_MAX_BLOCKS];
  int32_t d[EQF_MAX_BLOCKS];
  int32_t is_scalar[EQF_MAX_BLOCKS];   /* 0e entries: mean-centred, carry the affine bias */
  float eps;
} EqfNormLayout;
int eqf_eln_rows(const EqfNormLayout* lay, int64_t rows);   /* CTAs of a backward launch = rows of `part` */
int eqf_eln_fwd(const EqfNormLayout* lay, const float* x, const float* w, const float* b, int64_t N, float* y,
                float* rstd, void* stream);
int eqf_eln_bwd(const EqfNormLayout* lay, const float* x, const float* w, const float* rstd, const float* gy,
                int64_t N, float* gx, float* part, void* stream);

/* the same on planar node features: entry t is a packed [N, d_t, mul_t] buffer (host arrays of device pointers) */
int eqf_eln_fwd_planar(const EqfNormLayout* lay, const float* const* x_blocks, const float* w, const float* b, int64_t N,
                       float* const* y_blocks, float* rstd, void* stream);
int eqf_eln_bwd_planar(const EqfNormLayout* lay, const float* const* x_blocks, const float* w, const float* rstd,
                       const float* const* gy_blocks, int64_t N, float* const* gx_blocks, float* part, void* stream);

/* Gate + attention logits of GraphAttention.forward (graph_attention_transformer.py:492-495, 506-507) in one pass:
 *   t0[e] = [alpha | scalars | gates] pre-activations (+ optional bias), gated[b] planar blocks [E, d, C];
 *   z[e,h] = sum_k c_slr * SmoothLeakyReLU(alpha[e,h,k]) * alpha_dot[h,k];  v0 = c_silu * silu(scalars);
 *   vout[b][e,i,c] = gated[b][e,i,c] * c_sigmoid * sigmoid(gate[c]).  Constants are e3nn's normalize2mom factors. */
typedef struct {
  int32_t n_gated;
  int32_t d[EQF_MAX_BLOCKS];
  int32_t C[EQF_MAX_BLOCKS];
  int32_t n_alpha, n_scalars, n_heads;
  float c_silu, c_sigmoid, c_slr, slr_slope;
} EqfGateLayout;
int eqf_gate_logits_fwd(const EqfGateLayout* lay, const float* t0, const float* bias, const float* const* gated,
                        const float* alpha_dot, int64_t n_edges, float* z, float* v0, float* const* vout, void* stream);
int eqf_gate_logits_bwd(const EqfGateLayout* lay, const float* t0, const float* bias, const float* const* gated,
                        const float* alpha_dot, const float* gz, const float* gv0, const float* const* gvout,
                        int64_t n_edges, float* gt0, float* const* ggated, float* gdot_part, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EQF_B200_H_ */
