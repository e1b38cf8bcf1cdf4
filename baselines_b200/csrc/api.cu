// extern "C" surface of libb200rl (declared in include/b200rl.h): thin forwarding layer, no torch types.
#include <stdarg.h>
#include <stdio.h>

#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int gemm_f16_impl(const void*, const void*, void*, const float*, const void*, int, int, int, long long, long long,
                  long long, long long, int, int, int, float, int, int, int, int, int, const void*, cudaStream_t);
int conv_shift_fwd_impl(const void*, long long, int, int, int, const void*, long long, int, int, const int*, int, int,
                        void*, const long long*, const long long*, const float*, int, int, float,
                        const void*, const long long*, int, int, int, int, void*, const void*, cudaStream_t);
int conv_shift_wgrad_impl(const void*, long long, int, const void*, int, int, const int*, float*, long long, float,
                          float*, float, int, const void*, const long long*, int, int, int, int, int, cudaStream_t);
int conv_gemm_impl(const void*, long long, int, int, int, int, int, int, int, int, int, int, int, const void*,
                   long long, void*, long long, const float*, const void*, long long, int, int, int, int, float, int,
                   int, int, int, int, cudaStream_t);
int dgrad_weights_impl(const float*, void*, int, int, int, int, int, long long, cudaStream_t);
int gae_scan_impl(const float*, const float*, const uint8_t*, const float*, const uint8_t*, float*, float*, int, int,
                  double, double, int, cudaStream_t);
int im2col_impl(const void*, int, const long long*, void*, long long, int, int, int, int, int, int, cudaStream_t);
int s2d_gather_impl(const void*, const long long*, void*, long long, int, int, int, int, cudaStream_t);
int frame_stack_impl(const void*, const void*, const void*, void*, long long, long long, int, int, cudaStream_t);
int col2im_impl(const void*, const void*, void*, long long, int, int, int, int, int, int, int, cudaStream_t);
int colsum_impl(const void*, float*, long long, int, long long, float, cudaStream_t);
int cat_step_impl(const float*, long long, int, const int*, int, const float*, long long, const float*,
                  unsigned long long, unsigned long long, const unsigned long long*, long long*, float*, float*,
                  long long, cudaStream_t);
int bern_step_impl(const float*, long long, int, const float*, long long, const float*, unsigned long long,
                   unsigned long long, const unsigned long long*, float*, float*, float*, long long, cudaStream_t);
int gauss_step_impl(const float*, long long, const float*, int, const float*, long long, const float*,
                    unsigned long long, unsigned long long, const unsigned long long*, float*, float*, float*,
                    long long, cudaStream_t);
int set_scalars_impl(float*, int, float, float, float, float, cudaStream_t);
int shuffle_indices_impl(long long*, long long, unsigned long long, long long, long long, cudaStream_t);
int counter_add_impl(unsigned long long*, unsigned long long, cudaStream_t);
int adv_stats_impl(const float*, const float*, const long long*, long long, double*, cudaStream_t);
int cat_loss_impl(const float*, long long, int, const int*, int, const float*, long long, const long long*,
                  const long long*, const float*, const float*, const float*, const double*, float, float, float, void*,
                  long long, void*, long long, double*, long long, const float*, cudaStream_t);
int bern_loss_impl(const float*, long long, int, const float*, long long, const float*, const long long*, const float*,
                   const float*, const float*, const double*, float, float, float, void*, long long, void*, long long,
                   double*, long long, const float*, cudaStream_t);
int gauss_loss_impl(const float*, long long, const float*, int, const float*, long long, const float*,
                    const long long*, const float*, const float*, const float*, const double*, float, float, float,
                    void*, long long, void*, long long, float*, float, double*, long long, const float*, cudaStream_t);
int sumsq_impl(const float*, long long, double*, cudaStream_t);
int seg_sumsq_impl(const float*, const long long*, int, double*, cudaStream_t);
int clip_adam_impl(float*, const float*, float*, float*, long long, float, float, float, float, float, const double*,
                   const long long*, int, const float*, cudaStream_t);
int clip_accumulate_impl(const float*, float*, long long, float, float, const double*, cudaStream_t);
int cast_transpose_impl(const float*, int, int, void*, long long, void*, long long, float, cudaStream_t);
int cast_f32_f16_impl(const float*, void*, long long, int, long long, long long, float, cudaStream_t);
int cast_transpose_batch_impl(const void*, int, int, int, cudaStream_t);
int obs_encode_impl(const float*, const long long*, long long, int, int, int, const float*, const float*, float, float,
                    int, const int*, int, void*, int*, cudaStream_t);
int tree_set_impl(double*, double*, long long, const long long*, const double*, int, cudaStream_t);
int tree_range_sum_impl(const double*, long long, long long, long long, double*, cudaStream_t);
int per_sample_impl(const double*, const double*, long long, long long, const double*, int, double, long long*,
                    double*, float*, int*, cudaStream_t);
int per_priorities_impl(const float*, int, double, double, double*, double*, int*, cudaStream_t);
int per_pow_impl(const double*, int, double, double*, cudaStream_t);
int dqn_td_impl(const float*, long long, const float*, long long, const float*, long long, const float*, long long,
                const float*, long long, const float*, long long, int, const long long*, const long long*,
                const float*, const float*, const float*, float, int, float*, void*, long long, void*, long long,
                double*, int, cudaStream_t);
int dqn_act_impl(const float*, long long, const float*, long long, int, float, unsigned long long,
                 unsigned long long, const float*, const unsigned long long*, long long*, int, cudaStream_t);
int lstm_seq_fwd_impl(const float*, long long, const void*, const uint8_t*, const long long*, const float*,
                      const long long*, float*, void*, long long, void*, float*, float*, int, int, int, cudaStream_t);
int lstm_seq_bwd_impl(const void*, long long, const float*, const float*, const uint8_t*, const long long*,
                      const float*, const long long*, const void*, void*, long long, int, int, int, cudaStream_t);
int ln_fwd_impl(const float*, long long, const float*, const float*, void*, long long, long long, int, int, float,
                cudaStream_t);
int ln_bwd_impl(const void*, long long, const float*, long long, const float*, void*, long long, float*, float*,
                long long, int, float, float, cudaStream_t);
int param_perturb_impl(const float*, float*, const void*, int, long long, const float*, const float*,
                       unsigned long long, const unsigned long long*, cudaStream_t);
int dqn_param_noise_adapt_impl(const float*, const float*, long long, int, int, int, float*, const float*, float*,
                               cudaStream_t);
int vecnorm_moments_impl(const void*, int, long long, int, double*, cudaStream_t);
int vecnorm_combine_impl(double*, const double*, int, long long, int, double, cudaStream_t);
int vecnorm_normalize_impl(const void*, int, long long, int, const double*, double, float*, cudaStream_t);
int vecnorm_rewards_impl(const void*, int, const uint8_t*, long long, double*, double*, double, double, double, float*,
                         cudaStream_t);
int vecnorm_add_latency_impl(int, long long, double*, cudaStream_t);

}  // namespace b200rl

using namespace b200rl;
#define S(x) reinterpret_cast<cudaStream_t>(x)

extern "C" {

const char* b200rl_last_error(void) { return g_err; }
int b200rl_version(void) { return 100; }

int b200rl_gae_scan(const float* rewards, const float* values, const uint8_t* dones, const float* last_values,
                    const uint8_t* last_dones, float* advs, float* returns, int T, int N, double gamma, double lam,
                    int variant, void* stream) {
  return gae_scan_impl(rewards, values, dones, last_values, last_dones, advs, returns, T, N, gamma, lam, variant,
                       S(stream));
}

int b200rl_gemm_f16(const void* A, const void* B, void* C, const float* bias, const void* saved, int M, int N, int K,
                    long long lda, long long ldb, long long ldc, long long ld_saved, int mn_major, int mode, int act,
                    float alpha, int split_k, int max_ctas, int rm_C, int rm_OW, int rm_Wg, const void* saved_bits,
                    void* stream) {
  return gemm_f16_impl(A, B, C, bias, saved, M, N, K, lda, ldb, ldc, ld_saved, mn_major, mode, act, alpha, split_k,
                       max_ctas, rm_C, rm_OW, rm_Wg, saved_bits, S(stream));
}

int b200rl_conv_shift_fwd(const void* X, long long B, int Hg, int Wg, int C, const void* W, long long ldw, int N,
                          int taps, const int* shifts, int vy, int vx, void* out, const long long* omap,
                          const long long* smap, const float* bias, int act, int dact, float alpha,
                          const void* u8_x, const long long* u8_idx, int u8_H, int u8_W, int u8_C, int u8_s,
                          void* act_bits_out, const void* saved_bits, void* stream) {
  return conv_shift_fwd_impl(X, B, Hg, Wg, C, W, ldw, N, taps, shifts, vy, vx, out, omap, smap, bias, act, dact, alpha,
                             u8_x, u8_idx, u8_H, u8_W, u8_C, u8_s, act_bits_out, saved_bits, S(stream));
}
int b200rl_conv_shift_wgrad(const void* X, long long rows, int C, const void* dY, int N, int taps, const int* shifts,
                            float* G, long long ldg, float alpha, float* gbias, float alpha_b, int max_ctas,
                            const void* u8_x, const long long* u8_idx, int u8_H, int u8_W, int u8_C, int u8_s,
                            int kx, void* stream) {
  return conv_shift_wgrad_impl(X, rows, C, dY, N, taps, shifts, G, ldg, alpha, gbias, alpha_b, max_ctas, u8_x, u8_idx,
                               u8_H, u8_W, u8_C, u8_s, kx, S(stream));
}

int b200rl_conv_gemm(const void* x, long long B, int H, int W, int C, int R, int S, int stride_h, int stride_w,
                     int pad_h, int pad_w, int OH, int OW, const void* Wt_or_dz, long long ldb, void* out,
                     long long ldc, const float* bias, const void* saved, long long ld_saved, int N, int kind,
                     int mode, int act, float alpha, int split_k, int sh_H, int sh_W, int sh_C, int sh_s,
                     void* stream) {
  return conv_gemm_impl(x, B, H, W, C, R, S, stride_h, stride_w, pad_h, pad_w, OH, OW, Wt_or_dz, ldb, out, ldc, bias,
                        saved, ld_saved, N, kind, mode, act, alpha, split_k, sh_H, sh_W, sh_C, sh_s, S(stream));
}
int b200rl_dgrad_weights(const float* w, void* out, int R, int S_, int Cin, int Cout, int s, long long ld,
                         void* stream) {
  return dgrad_weights_impl(w, out, R, S_, Cin, Cout, s, ld, S(stream));
}

int b200rl_im2col(const void* x, int src_is_u8, const long long* src_idx, void* cols, long long B, int H, int W,
                  int C, int rf, int stride, int same_pad, void* stream) {
  return im2col_impl(x, src_is_u8, src_idx, cols, B, H, W, C, rf, stride, same_pad, S(stream));
}
int b200rl_frame_stack(const void* prev, const void* frame, const void* news, void* out, long long N, long long pixels,
                       int nstack, int c, void* stream) {
  return frame_stack_impl(prev, frame, news, out, N, pixels, nstack, c, S(stream));
}

int b200rl_s2d_gather(const void* x, const long long* src_idx, void* out, long long B, int H, int W, int C, int s,
                      void* stream) {
  return s2d_gather_impl(x, src_idx, out, B, H, W, C, s, S(stream));
}
int b200rl_col2im(const void* dcols, const void* saved, void* dx, long long B, int H, int W, int C, int rf,
                  int stride, int same_pad, int act, void* stream) {
  return col2im_impl(dcols, saved, dx, B, H, W, C, rf, stride, same_pad, act, S(stream));
}
int b200rl_colsum(const void* dz, float* db, long long rows, int C, long long ld, float alpha, void* stream) {
  return colsum_impl(dz, db, rows, C, ld, alpha, S(stream));
}

// CategoricalPd / MultiCategoricalPd .sample + .neglogp (distributions.py:76-94,164-201,206-225)
int b200rl_cat_step(const float* logits, long long ld, int nA, const int* seg_off, int nseg, const float* vpred,
                    long long ldv, const float* uniforms, unsigned long long seed, unsigned long long offset,
                    const unsigned long long* offset_dev, long long* actions, float* values, float* neglogp,
                    long long B, void* stream) {
  return cat_step_impl(logits, ld, nA, seg_off, nseg, vpred, ldv, uniforms, seed, offset, offset_dev, actions, values,
                       neglogp, B, S(stream));
}
// BernoulliPd.sample + .neglogp (distributions.py:115-128,254-276)
int b200rl_bern_step(const float* logits, long long ld, int n, const float* vpred, long long ldv,
                     const float* uniforms, unsigned long long seed, unsigned long long offset,
                     const unsigned long long* offset_dev, float* actions, float* values, float* neglogp, long long B,
                     void* stream) {
  return bern_step_impl(logits, ld, n, vpred, ldv, uniforms, seed, offset, offset_dev, actions, values, neglogp, B,
                        S(stream));
}
int b200rl_shuffle_indices(long long* out, long long n, unsigned long long key, long long T, long long N, void* stream) {
  return shuffle_indices_impl(out, n, key, T, N, S(stream));
}
int b200rl_set_scalars(float* dst, int n, float a, float b, float c, float d, void* stream) {
  return set_scalars_impl(dst, n, a, b, c, d, S(stream));
}
int b200rl_counter_add(unsigned long long* ctr, unsigned long long inc, void* stream) {
  return counter_add_impl(ctr, inc, S(stream));
}
int b200rl_gauss_step(const float* mean, long long ld, const float* logstd, int d, const float* vpred,
                      long long ldv, const float* normals, unsigned long long seed, unsigned long long offset,
                      const unsigned long long* offset_dev, float* actions, float* values, float* neglogp,
                      long long B, void* stream) {
  return gauss_step_impl(mean, ld, logstd, d, vpred, ldv, normals, seed, offset, offset_dev, actions, values, neglogp,
                         B, S(stream));
}
int b200rl_adv_stats(const float* returns, const float* values, const long long* src_idx, long long M, double* out,
                     void* stream) {
  return adv_stats_impl(returns, values, src_idx, M, out, S(stream));
}
// ppo2/model.py:57-91 with CategoricalPd / MultiCategoricalPd (distributions.py:76-94,164-198,206-225)
int b200rl_cat_loss(const float* logits, long long ld, int nA, const int* seg_off, int nseg, const float* vpred,
                    long long ldv, const long long* actions, const long long* src_idx, const float* returns,
                    const float* old_values, const float* old_neglogp, const double* adv_stats, float cliprange,
                    float ent_coef, float vf_coef, void* dlogits, long long ld_dl, void* dv, long long ld_dv,
                    double* stats, long long B, const float* cliprange_dev, void* stream) {
  return cat_loss_impl(logits, ld, nA, seg_off, nseg, vpred, ldv, actions, src_idx, returns, old_values, old_neglogp,
                       adv_stats, cliprange, ent_coef, vf_coef, dlogits, ld_dl, dv, ld_dv, stats, B, cliprange_dev,
                       S(stream));
}
// ppo2/model.py:57-91 with BernoulliPd (distributions.py:115-128,254-276)
int b200rl_bern_loss(const float* logits, long long ld, int n, const float* vpred, long long ldv,
                     const float* actions, const long long* src_idx, const float* returns, const float* old_values,
                     const float* old_neglogp, const double* adv_stats, float cliprange, float ent_coef,
                     float vf_coef, void* dlogits, long long ld_dl, void* dv, long long ld_dv, double* stats,
                     long long B, const float* cliprange_dev, void* stream) {
  return bern_loss_impl(logits, ld, n, vpred, ldv, actions, src_idx, returns, old_values, old_neglogp, adv_stats,
                        cliprange, ent_coef, vf_coef, dlogits, ld_dl, dv, ld_dv, stats, B, cliprange_dev, S(stream));
}
int b200rl_gauss_loss(const float* mean, long long ld, const float* logstd, int d, const float* vpred,
                      long long ldv, const float* actions, const long long* src_idx, const float* returns,
                      const float* old_values, const float* old_neglogp, const double* adv_stats, float cliprange,
                      float ent_coef, float vf_coef, void* dmean, long long ld_dm, void* dv, long long ld_dv,
                      float* dlogstd, float inv_M, double* stats, long long B, const float* cliprange_dev,
                      void* stream) {
  return gauss_loss_impl(mean, ld, logstd, d, vpred, ldv, actions, src_idx, returns, old_values, old_neglogp,
                         adv_stats, cliprange, ent_coef, vf_coef, dmean, ld_dm, dv, ld_dv, dlogstd, inv_M, stats, B,
                         cliprange_dev, S(stream));
}

int b200rl_sumsq(const float* g, long long n, double* out, void* stream) { return sumsq_impl(g, n, out, S(stream)); }
int b200rl_seg_sumsq(const float* g, const long long* seg_off, int nseg, double* out, void* stream) {
  return seg_sumsq_impl(g, seg_off, nseg, out, S(stream));
}
int b200rl_clip_adam(float* p, const float* g, float* m, float* v, long long n, float lr_t, float beta1, float beta2,
                     float eps, float clip, const double* sumsq, const long long* seg_off, int nseg,
                     const float* lr_t_dev, void* stream) {
  return clip_adam_impl(p, g, m, v, n, lr_t, beta1, beta2, eps, clip, sumsq, seg_off, nseg, lr_t_dev, S(stream));
}
int b200rl_clip_accumulate(const float* g, float* acc, long long n, float clip, float weight, const double* sumsq,
                           void* stream) {
  return clip_accumulate_impl(g, acc, n, clip, weight, sumsq, S(stream));
}
int b200rl_cast_transpose(const float* src, int R, int C, void* dst, long long ld_dst, void* dstT, long long ld_t,
                          float scale, void* stream) {
  return cast_transpose_impl(src, R, C, dst, ld_dst, dstT, ld_t, scale, S(stream));
}
int b200rl_cast_transpose_batch(const void* jobs, int njobs, int max_rows, int max_cols, void* stream) {
  return cast_transpose_batch_impl(jobs, njobs, max_rows, max_cols, S(stream));
}
int b200rl_cast_f32_f16(const float* src, void* dst, long long rows, int cols, long long ld_src, long long ld_dst,
                        float scale, void* stream) {
  return cast_f32_f16_impl(src, dst, rows, cols, ld_src, ld_dst, scale, S(stream));
}

// common/input.py:43-63 encode_observation (Discrete :54-55, MultiDiscrete :58-61), policies.py:182-185
int b200rl_obs_encode(const float* x, const long long* src_idx, long long B, int raw_dim, int in_dim, int in_pad,
                      const float* mean, const float* inv_std, float clip_lo, float clip_hi, int onehot_n,
                      const int* seg_off, int nseg, void* out, int* overflow, void* stream) {
  return obs_encode_impl(x, src_idx, B, raw_dim, in_dim, in_pad, mean, inv_std, clip_lo, clip_hi, onehot_n, seg_off,
                         nseg, out, overflow, S(stream));
}

int b200rl_tree_set(double* sum_tree, double* min_tree, long long capacity, const long long* idx, const double* vals,
                    int n, void* stream) {
  return tree_set_impl(sum_tree, min_tree, capacity, idx, vals, n, S(stream));
}
int b200rl_tree_range_sum(const double* tree, long long capacity, long long start, long long end, double* out,
                          void* stream) {
  return tree_range_sum_impl(tree, capacity, start, end, out, S(stream));
}
int b200rl_per_sample(const double* sum_tree, const double* min_tree, long long capacity, long long n_stored,
                      const double* uniforms, int batch, double beta, long long* idx_out, double* w_out,
                      float* w_out_f32, int* bad, void* stream) {
  return per_sample_impl(sum_tree, min_tree, capacity, n_stored, uniforms, batch, beta, idx_out, w_out, w_out_f32,
                         bad, S(stream));
}
int b200rl_per_priorities(const float* td, int n, double eps, double alpha, double* powered, double* max_priority,
                          int* bad, void* stream) {
  return per_priorities_impl(td, n, eps, alpha, powered, max_priority, bad, S(stream));
}
int b200rl_per_pow(const double* x, int n, double y, double* out, void* stream) {
  return per_pow_impl(x, n, y, out, S(stream));
}
int b200rl_dqn_td(const float* a_t, long long lda_t, const float* s_t, long long lds_t, const float* a_on,
                  long long lda_on, const float* s_on, long long lds_on, const float* a_tg, long long lda_tg,
                  const float* s_tg, long long lds_tg, int nA, const long long* idx, const long long* actions,
                  const float* rewards, const float* dones, const float* weights, float gamma, int double_q,
                  float* td_out, void* d_a, long long ld_da, void* d_s, long long ld_ds, double* loss_sum, int B,
                  void* stream) {
  return dqn_td_impl(a_t, lda_t, s_t, lds_t, a_on, lda_on, s_on, lds_on, a_tg, lda_tg, s_tg, lds_tg, nA, idx, actions,
                     rewards, dones, weights, gamma, double_q, td_out, d_a, ld_da, d_s, ld_ds, loss_sum, B, S(stream));
}
int b200rl_dqn_act(const float* a, long long lda, const float* s, long long lds, int nA, float eps,
                   unsigned long long seed, unsigned long long step, const float* eps_dev,
                   const unsigned long long* step_dev, long long* actions, int B, void* stream) {
  return dqn_act_impl(a, lda, s, lds, nA, eps, seed, step, eps_dev, step_dev, actions, B, S(stream));
}

// a2c/utils.py:84-97 lstm() over a sequence; its gradient (ppo2/model.py:102 tf.gradients through the recurrence)
int b200rl_lstm_seq_fwd(const float* xg, long long ldxg, const void* wh, const uint8_t* masks, const long long* mask_idx,
                        const float* state_in, const long long* state_idx, float* state_out, void* h_out,
                        long long ldh, void* hprev_out, float* gates_out, float* c_out, int T, int B, int H,
                        void* stream) {
  return lstm_seq_fwd_impl(xg, ldxg, wh, masks, mask_idx, state_in, state_idx, state_out, h_out, ldh, hprev_out,
                           gates_out, c_out, T, B, H, S(stream));
}
int b200rl_lstm_seq_bwd(const void* dh, long long lddh, const float* gates, const float* c, const uint8_t* masks,
                        const long long* mask_idx, const float* state_in, const long long* state_idx, const void* whT,
                        void* dz, long long lddz, int T, int B, int H, void* stream) {
  return lstm_seq_bwd_impl(dh, lddh, gates, c, masks, mask_idx, state_in, state_idx, whT, dz, lddz, T, B, H,
                           S(stream));
}

// tf.contrib.layers.layer_norm after a fully connected layer (common/models.py:97-98, deepq/models.py:24-25,34-35)
int b200rl_ln_fwd(const float* z, long long ld_z, const float* gamma, const float* beta, void* y, long long ld_y,
                  long long rows, int N, int act, float eps, void* stream) {
  return ln_fwd_impl(z, ld_z, gamma, beta, y, ld_y, rows, N, act, eps, S(stream));
}
int b200rl_ln_bwd(const void* du, long long ld_du, const float* z, long long ld_z, const float* gamma, void* dz,
                  long long ld_dz, float* dgamma, float* dbeta, long long rows, int N, float alpha, float eps,
                  void* stream) {
  return ln_bwd_impl(du, ld_du, z, ld_z, gamma, dz, ld_dz, dgamma, dbeta, rows, N, alpha, eps, S(stream));
}

// deepq/build_graph.py:258-287: perturb_vars, mean_kl and the scale adaptation of parameter-space noise
int b200rl_param_perturb(const float* src, float* dst, const void* jobs, int njobs, long long max_len,
                         const float* scale_dev, const float* normals, unsigned long long seed,
                         const unsigned long long* offset_dev, void* stream) {
  return param_perturb_impl(src, dst, jobs, njobs, max_len, scale_dev, normals, seed, offset_dev, S(stream));
}
int b200rl_dqn_param_noise_adapt(const float* q, const float* q_adapt, long long ld, int nA, int dueling, int B,
                                 float* scale_dev, const float* threshold_dev, float* mean_kl_dev, void* stream) {
  return dqn_param_noise_adapt_impl(q, q_adapt, ld, nA, dueling, B, scale_dev, threshold_dev, mean_kl_dev, S(stream));
}

// common/vec_env/vec_normalize.py:26-47 VecNormalize with running_mean_std.py:22-33 RunningMeanStd
int b200rl_vecnorm_moments(const void* x, int x_f64, long long N, int D, double* ws, void* stream) {
  return vecnorm_moments_impl(x, x_f64, N, D, ws, S(stream));
}
int b200rl_vecnorm_combine(double* rms, const double* ws, int ws_f32, long long N, int D, double eps, void* stream) {
  return vecnorm_combine_impl(rms, ws, ws_f32, N, D, eps, S(stream));
}
int b200rl_vecnorm_normalize(const void* x, int x_f64, long long N, int D, const double* rms, double clip, float* out,
                             void* stream) {
  return vecnorm_normalize_impl(x, x_f64, N, D, rms, clip, out, S(stream));
}
int b200rl_vecnorm_rewards(const void* rew, int rew_f64, const uint8_t* news, long long N, double* ret, double* rms,
                           double gamma, double eps, double cliprew, float* out, void* stream) {
  return vecnorm_rewards_impl(rew, rew_f64, news, N, ret, rms, gamma, eps, cliprew, out, S(stream));
}
int b200rl_vecnorm_add_latency(int f64, long long n, double* out, void* stream) {
  return vecnorm_add_latency_impl(f64, n, out, S(stream));
}

}  // extern "C"
