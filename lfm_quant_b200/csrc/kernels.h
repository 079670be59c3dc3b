// Host-callable launchers of the lfmq kernels.  All return 0 or LFMQ_ERR_CUDA (message in g_err).
#pragma once
#include "common.cuh"

namespace lfmq {

// ---- fp32 SIMT building blocks (kernels_simt.cu) ---------------------------------------------
// C[M,N] (row-major, ldc) = A*B + beta*C with A(m,k) = A[m*sAm + k*sAk], B(k,n) = B[k*sBk + n*sBn].
// `scratch` (>= scratch_elems floats) is used for deterministic split-K partials.
int sgemm(cudaStream_t s, int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBk,
          long sBn, float* C, long ldc, float beta, float* scratch, size_t scratch_elems);
// C[M,N] = sum_z partial[z][M][N] (in z order) + beta*C: the reduction of a deterministic split-K product
int splitk_reduce(cudaStream_t s, int M, int N, int S, const float* partial, float* C, long ldc, float beta);
// sgemm's contract on sm_90a wgmma with tf32 operands (cvt.rna) and fp32 accumulation (tf32_gemm.cu): the GEMMs of a
// LFMQ_PREC_TF32 handle
int tf32_gemm(cudaStream_t s, int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBk,
              long sBn, float* C, long ldc, float beta, float* scratch, size_t scratch_elems);

int lstm_pointwise_fwd(cudaStream_t s, int B, int T, int H, int t, const float* z, const float* bias, float* gates,
                       float* c, float* h, const float* rmask, float* hm);
int lstm_pointwise_bwd(cudaStream_t s, int B, int T, int H, int t, const float* gates, const float* c,
                       const float* dh_out, const float* dh_rec, const float* rmask, float* dc, float* dz);
int gru_pointwise_fwd(cudaStream_t s, int B, int T, int H, int t, const float* zx, const float* zh, const float* bias,
                      float* gates, float* h, const float* rmask, float* hm);
int gru_pointwise_bwd(cudaStream_t s, int B, int T, int H, int t, const float* gates, const float* h,
                      const float* dh_out, const float* dh_rec, const float* rmask, float* dcarry, float* dxz,
                      float* dhz);
int gen_row_mask(cudaStream_t s, int B, int H, DropoutKey key, int64_t row0, float* rmask);
int shift_mask(cudaStream_t s, int B, int T, int H, const float* h, const float* rmask, float* hp);
int bn_dropout_fwd(cudaStream_t s, int B, int T, int H, const float* h, const float* gamma, const float* beta,
                   const float* mean, const float* var, float eps, bool use_dropout, DropoutKey key, int64_t row0,
                   float* y);
// dgamma == nullptr: dh_out only (no dgamma / dbeta, no scratch)
int bn_dropout_bwd(cudaStream_t s, int B, int T, int H, const float* dy, const float* h, const float* gamma,
                   const float* mean, const float* var, float eps, bool use_dropout, DropoutKey key, int64_t row0,
                   float* dh_out, float* dgamma, float* dbeta, float* scratch, size_t scratch_elems);
int add_bias_rows(cudaStream_t s, long rows, int N, float* C, const float* bias);
int colsum(cudaStream_t s, long rows, int N, const float* A, float* out, float* scratch, size_t scratch_elems);
int softplus_floor(cudaStream_t s, long n, const float* a, float* var);
int mask_count(cudaStream_t s, int B, int T, int O, const float* y, float* out2, unsigned int* tickets);
// out2 = {loss, mse_0}; maskout2 (nullable) = {B, mask_count_local}; dpred may be NULL (validation);
// denom (nullable) = device {B_global, mask_count_global}, or their weighted sums when rw (nullable, the batch's row
// weights, common.cuh row_weight) is given: then denom is required.
// lfmq_row_weights (include/lfmq.h)
int row_weights(cudaStream_t s, const double* table, int n_cols, const int* inp_idx, int B, int weight_col,
                int date_col, double halflife, int ref_month, float* w);
int loss_grad(cudaStream_t s, int B, int T, int O, const float* pred, const float* y, const float* denom,
              const float* rw, int target_idx, float p1, float p2, float* dpred, float* out2, float* maskout2,
              float* scratch);
// scalars[0] = ||g||, scalars[1] = clip scale (1 when clip <= 0)
int grad_norm_scale(cudaStream_t s, long n, const float* g, float clip, float* scalars, float* scratch,
                    unsigned int* ticket);
int opt_update(cudaStream_t s, int opt, long n, float* p, const float* g, float* slot0, float* slot1,
               const float* scalars, float lr, float c1, float c2, float momentum);
int maxnorm_cols(cudaStream_t s, int I, int N, float* W, float max_norm);
int fill(cudaStream_t s, float* p, long n, float v);

// forecast_steps > 1 (rnn_point_estimate.py:109-150): glue between the stage handles
constexpr int LFMQ_MAX_STAGES = 8;
struct ChainPtrs { float* p[LFMQ_MAX_STAGES]; };
struct ChainWeights { float w[LFMQ_MAX_STAGES]; };
struct ChainCPtrs { const float* p[LFMQ_MAX_STAGES]; };
int chain_next_input(cudaStream_t s, int B, int T, int F, int O, const float* prev, const float* pred, const float* x0,
                     float* next);
int scale_inplace(cudaStream_t s, long n, float* p, float w);
int chain_scatter_dx(cudaStream_t s, int B, int T, int F, int O, int stage, const float* dx, const ChainPtrs& dpred);
int chain_combine(cudaStream_t s, int S, const ChainPtrs& scalars, float clip, const ChainPtrs& loss2,
                  const ChainWeights& w, float* out2);
// Monte-Carlo dropout samples of a uq model: sample s of window b is row s * B + b of the batch tiled `samples` times.
// mc_replicate: xrep = rows [r0, r0 + n) of that tiled batch (row_elems floats per row).
int mc_replicate(cudaStream_t s, int B, int64_t r0, int n, long row_elems, const float* x, float* xrep);
// mc_moments: folds every stage's sampled pred / var [n, T, O] of tiled rows [r0, r0 + n) into the per-element moments
// [B, T, O] of the samples; chunks must arrive in increasing r0 and cover [0, samples * B) without gaps.  After the last
// one, mean_pred / mean_var hold the sample means and var_pred / var_var the population variances.
struct McMoments { ChainPtrs pred, var, mean_pred, mean_var, var_pred, var_var; };
int mc_moments(cudaStream_t s, int n_stages, int B, int TO, int64_t r0, int n, int samples, const McMoments& m);
// Predictive distributions of those samples (predictive.cu, lfmq_chain_forward_uq_dist).  dist_gather: the samples'
// (pred, var) at element `off` of the [T, O] rows of tiled rows [r0, r0 + n) into mu.p[s] / v.p[s] [B][samples].
// mixture_dist: per window and stage the mixture's quantiles at the host levels[n_levels] into quantiles.p[s] [B][Q]
// and, where y.p[s] is not null, {crps, nll, pit} of the target y.p[s][b * y_stride + y_off] into scores.p[s] [B][3].
constexpr int LFMQ_DIST_MAX_LEVELS = 32;
int dist_gather(cudaStream_t s, int n_stages, int B, int TO, long off, int64_t r0, int n, int samples,
                const ChainPtrs& pred, const ChainPtrs& var, const ChainPtrs& mu, const ChainPtrs& v);
int mixture_dist(cudaStream_t s, int n_stages, int B, int samples, const float* levels, int n_levels,
                 const ChainPtrs& mu, const ChainPtrs& v, const ChainCPtrs& y, long y_stride, long y_off,
                 const ChainPtrs& quantiles, const ChainPtrs& scores);
// Integrated gradients (lfmq_integrated_gradients): interpolant k of window b is row k * B + b of the batch tiled M
// times, with input alpha_k * x[b], alpha_k = (k + 1/2) / M.
// ig_scale_inputs: xs = rows [r0, r0 + n) of that tiled batch, each scaled by its alpha_k (row_elems = T * F).
int ig_scale_inputs(cudaStream_t s, int B, int M, int64_t r0, int n, long row_elems, const float* x, float* xs);
// ig_seed: dpred [n, T, O] = 1 at [T-1, target_idx] of every row, 0 elsewhere.
int ig_seed(cudaStream_t s, int n, int T, int O, int target_idx, float* dpred);
// ig_pick: out[i] = preds[i mod n_src, T-1, target_idx] for i < n_out.
int ig_pick(cudaStream_t s, int n_out, int n_src, int T, int O, int target_idx, const float* preds, float* out);
// ig_fold: adds the input gradients dx [n, T, F] of tiled rows [r0, r0 + n) into attr [B, T, F] in increasing k; the
// last interpolant multiplies the sum by x / M.  Launches must arrive in increasing r0 and cover [0, M * B).
int ig_fold(cudaStream_t s, int B, int M, int64_t r0, int n, long row_elems, const float* dx, const float* x,
            float* attr);
// Permutation importance and Shapley attributions (importance.cu, lfmq_chain_permutation_importance,
// lfmq_chain_shapley): perm_index is the bijection pi_{seed,key,rep} of [0, N) (a 4-round Philox Feistel network on
// [0, 2^m), cycle-walked into [0, N)); perm_importance_gather writes rows [a, a + n) of a copy of x [N, row_elems] to
// out [n, row_elems]: columns c with rank[col_group[c]] >= k (device int32 [row_elems] and [G]) come from window
// pi_{seed,key,rep}(i), the others from window i.
__host__ __device__ uint32_t perm_index(int32_t N, uint64_t seed, int32_t group, int32_t repeat, uint32_t i);
int perm_importance_gather(cudaStream_t s, const float* x, int N, long row_elems, const int32_t* col_group,
                           const int32_t* rank, int k, uint64_t seed, int key, int rep, int a, int n, float* out);
// shapley_fold: folds the K explained outputs of windows [a, a + n), src.p[o][i * stride + off] for output o of launch
// row i, of coalition copy k (0..G) of one sample into the sums of lfmq_chain_shapley: f_bg at k = 0, f_x at k = G, and
// for k > 0 the difference to the window's previous copy (prev [N][K]) into phi [N][K][G] at group order[k - 1], all
// three sums in fp64.  shapley_finish: out[j] = (float)(sum[j] / samples) for j < n.
struct ShapleySrc { const float* p[2 * LFMQ_MAX_STAGES]; };
int shapley_fold(cudaStream_t s, const ShapleySrc& src, int K, long stride, long off, int a, int n, int k, int G,
                 const int32_t* order, float* prev, double* phi, double* f_x, double* f_bg);
int shapley_finish(cudaStream_t s, long n, const double* sum, int samples, float* out);
// Accumulated local effects (ale.cu, lfmq_chain_ale).  ale_sort_bytes: the temp storage of the segmented radix sort of
// G segments of N (value, window) pairs.  ale_bins: the values x[i, cols[g]] sorted per feature into skey / sval, the
// edges, counts and n_bins outputs, the sorted bin ends ends [G][K+1] and every window's bin bin_of [G][N] (0: none).
constexpr int LFMQ_ALE_MAX_BINS = 1024;
struct AleSort {
  float *key, *skey;
  int32_t *val, *sval, *off, *ends, *bin_of;
};
int ale_sort_bytes(int N, int G, size_t* bytes);
int ale_bins(cudaStream_t s, const float* x, int N, long row_elems, const int32_t* cols, int G, int K, void* temp,
             size_t temp_bytes, const AleSort& w, int32_t* n_bins, float* edges, int32_t* counts);
// ale_gather: rows [a, a + n) of x [N, row_elems] into out with column col at edge[bin_of[i] - 1 + upper].
int ale_gather(cudaStream_t s, const float* x, long row_elems, int col, const int32_t* bin_of, const float* edge,
               int upper, int a, int n, float* out);
// ale_pick: the J explained outputs of windows [a, a + n) (as shapley_fold reads them) into d [N][J] on the upper copy,
// subtracted from it on the lower one.
int ale_pick(cudaStream_t s, const ShapleySrc& src, int J, long stride, long off, int a, int n, int upper, float* d);
// ale_fold: feature g's per-bin mean and population sd of d over each bin's sorted run, then ale = the centred prefix
// sums of the means; mean [K][J] is fp64 scratch.
int ale_fold(cudaStream_t s, const AleSort& w, const int32_t* n_bins, int g, int N, int K, int J, const float* d,
             double* mean, float* ale, float* local_mean, float* local_sd);
// Training-window attributions (influence.cu, lfmq_influence_*).  influence_grad: u [J][ldu][D + 1] rows [r0, r0 + n)
// from the head inputs a [n][Ta][D] and the launch's pred / var / pre / y [n][Ta][O] (mode 0 point, 1 uq, 2 dense with
// Ta = 1).  influence_query: aout [..][D + 1] and s [J][lds] rows from r0.
int influence_grad(cudaStream_t s, int n, int mode, int Ta, int D, int O, int tidx, float p1, float p2, int huber,
                   float delta, const float* a, const float* pred, const float* var, const float* pre, const float* y,
                   long r0, long ldu, float* u);
int influence_query(cudaStream_t s, int n, int Ta, int D, int O, int tidx, int uq, const float* a, const float* pre,
                    long r0, long lds, float* aout, float* sout);
// The pool split of one influence_topk call (a function of the shapes alone) and the sizes of its scratch.
struct InfluencePlan {
  int P, tiles_per_slice, n_sum;
  size_t list_elems, part_elems, usum_elems;
};
constexpr int LFMQ_INFLUENCE_MAX_K = 64;
InfluencePlan influence_plan(int Nq, int Nt, int D1, int J, int K);
int influence_topk(cudaStream_t s, const InfluencePlan& pl, const float* a, const float* u, const float* sc, int Nq,
                   int Nt, int D1, int J, int K, float* lscore, int* lidx, double* part, double* usum, int* pos_idx,
                   float* pos_score, int* neg_idx, float* neg_score, float* total);
// influence_topk's second mode (lfmq_nearest_topk): the K pool rows b [Nt][D1] nearest to each query a [Nq][D1].
// nearest_norms: the rows' squared norms nf [R] (fp64 sums in a fixed order, rounded to fp32).  The GEMM shortlists
// nearest_candidates(K) rows per query by the score 2 a.b - |b|^2 (bn [Nt] the pool's norms; pl planned for that many
// candidates); their exact fp64 distances pick idx / d2 [Nq][K] and, with value [Nt], mean [Nq].
constexpr int LFMQ_NEAREST_MAX_CAND = 80;
__host__ __device__ constexpr int nearest_candidates(int K) { return K + 16; }
int nearest_norms(cudaStream_t s, const float* p, int R, int D1, float* nf);
int nearest_topk(cudaStream_t s, const InfluencePlan& pl, const float* a, const float* b, const float* bn,
                 const float* value, int Nq, int Nt, int D1, int K, float* lscore, int* lidx, int32_t* idx, float* d2,
                 float* mean);
// Split-conformal intervals (conformal.cu, lfmq_conformal_*).  conformal_sort_bytes: the temp storage of the radix sort
// of S * Nc 64-bit (step, score) keys.  conformal_scores: r [n] of pred / y / scale [n] (scale nullable).
// conformal_calibrate: key / skey [S * Nc] scratch; n_valid [S], sorted [S][Nc], qhat [S][Q] of the host levels [Q].
// conformal_apply: lower / upper [S][N][Q] and pvalue [S][N] (y nullable: NaN p-values).
constexpr int LFMQ_CONFORMAL_MAX_LEVELS = 32;
int conformal_sort_bytes(int S, int Nc, size_t* bytes);
int conformal_scores(cudaStream_t s, long n, const float* pred, const float* y, const float* scale, float* r);
int conformal_calibrate(cudaStream_t s, int S, int Nc, const float* pred, const float* y, const float* scale,
                        const double* levels, int Q, void* temp, size_t temp_bytes, uint64_t* key, uint64_t* skey,
                        int32_t* n_valid, float* sorted, float* qhat);
int conformal_apply(cudaStream_t s, int S, int N, int Nc, int Q, const float* pred, const float* y, const float* scale,
                    const float* sorted, const int32_t* n_valid, const float* qhat, float* lower, float* upper,
                    float* pvalue);
// Lookahead factor backtests (factor.cu, lfmq_factor_eval).  FactorWork: the scratch the call carves (k0 / k1 / v0 / v1
// / d0 / d1 / pos [N] sort buffers; base_row [N] the (date, company) order; seg_off [D + 1] the date segments; pred [N] each row's
// predecessor at date index d - 1; mkey / mrow [M][N] the measures sorted within the dates; gkey / grow [N] one factor
// sorted; bq [N] its buckets; flag [N], pcg [M][N + 1] and pcm [N + 1] pair-row counts; yr [M][N] doubled measure
// ranks; temp of factor_temp_bytes).  FactorOut: the caller's outputs, as lfmq.h lays them out.
constexpr int LFMQ_FACTOR_MAX_G = 8;
constexpr int LFMQ_FACTOR_MAX_M = 4;
constexpr int LFMQ_FACTOR_MAX_Q = 100;
struct FactorWork {
  uint64_t *k0, *k1, *mkey, *gkey;
  int32_t *v0, *v1, *pos, *base_row, *seg_off, *pred, *mrow, *grow, *flag, *pcg, *pcm;
  uint32_t *d0, *d1, *yr;
  uint8_t* bq;
  char* temp;
};
struct FactorOut {
  int32_t *n, *bucket_n, *n_pair;
  double *ic, *bucket_mean, *spread, *turnover;
};
int factor_temp_bytes(int N, int D, size_t* bytes);
int factor_eval(cudaStream_t s, const int32_t* date, const int32_t* company, int N, int D, const double* score, int G,
                const double* measure, int M, int Q, const FactorWork& w, size_t temp_bytes, FactorOut o);
// The uq loss of RNNUqRangeEstimate, one stage (S = 1, w = 1) or a forecast chain: every stage's loss rows in one launch,
// then one reduction launch.
// pred.p[s] == nullptr: counts only, into counts.p[s].  Otherwise per stage {loss, uq0, mse0}.p[s] (each nullable) and
// out3 (nullable) = the weighted sums {uq_loss, uq_loss_last_tar, mse}; counts_in = 1 takes the counts from counts.p[s]
// (required with dpred), else the pass counts its own rows.  dpred / da (nullable) = w_s * dLoss_s / d(pred, apre).
// rw.p[s] (nullable): stage s's row weights; its counts are then {sum of weights, weighted unmasked rows, weighted
// unmasked last-step rows}.
struct ChainUqArgs {
  ChainPtrs pred, var, apre, y, dpred, da, counts, loss, uq0, mse0;
  ChainCPtrs rw;
  ChainWeights w;
  int counts_in;
};
int chain_uq_loss_grad(cudaStream_t s, int S, int B, int T, int O, const ChainUqArgs& a, int target_idx, float p1,
                       float p2, float* out3, float* scratch);
// Data parallelism: every stage's gradient buffer g[s] (16-byte aligned) holds n[s] gradients and then its tail; the
// flat vector holds, from off[s], the n[s] gradients and the ntail reduced tail entries: {loss, mse_0} (ntail = 2) or
// {uq_loss, mse_0, uq_loss_last_tar} (ntail = 3, tail indices 0, 1, 4).  One launch copies all stages (unpack: flat ->
// buffers).  On unpack, loss_out (nullable) = sum_s w_s of the tails: {loss, mse} or {uq_loss, uq_loss_last_tar, mse}.
struct GradPack {
  float* g[LFMQ_MAX_STAGES];
  long n[LFMQ_MAX_STAGES];
  long off[LFMQ_MAX_STAGES];
  int ntail;
};
int grad_pack(cudaStream_t s, int S, const GradPack& p, float* flat, bool unpack, const ChainWeights& w,
              float* loss_out);

struct GatherArgs {
  int n_rows, n_cols, B, T, F, O, stride, seq_norm_col, log_squasher, aux_masking;
  const double* table;
  const int32_t* inp_idx;
  const int32_t* tar_idx;
  const int32_t* inp_cols;
  const int32_t* fin_cols;
  const double* center;
  const double* scale;
  const uint8_t* scale_flag;
  const uint8_t* aux_flag;
  float* x;
  float* y;
  double* seq_norm;
};
int gather_batch(cudaStream_t s, const GatherArgs& a);

// window index on the device (data_processing.py:170-305); work: 4 * ceil(n / 1024) + n ints
struct WindowIndexArgs {
  int n, train, stride, forecast_n, min_steps, max_steps;
  int32_t start_date, end_date, last_train_date;
  const int32_t* key;
  const uint8_t* active;
  const int32_t* date;
};
int window_index(cudaStream_t s, const WindowIndexArgs& a, int cap, int32_t* inp, int32_t* tar, int32_t* rows,
                 int32_t* count, int* work);
int unscale(cudaStream_t s, const float* in, float* out, long n_rows, int O, const double* scale, const double* center,
            int log_squasher);

}  // namespace lfmq
