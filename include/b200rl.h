/* libb200rl -- C-ABI of the H100-native (sm_90a) PPO2 / DQN learner hot path.
 *
 * The reference (openai/baselines) has NO FFI: its hot path is TF1 graph ops + numpy loops called from
 * Python.  Each entry point below therefore names the reference interface (file:line) whose arithmetic it
 * replaces; INTEGRATION.md shows the ctypes binding a baselines maintainer would add.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller (torch tensors in this repo); no hidden
 *    allocation, no host synchronisation inside; `stream` is a cudaStream_t passed as void*.
 *  - return 0 on success, negative on error (see B200RL_ERR_*); b200rl_last_error() gives the text.
 *  - fp16 tensors are IEEE half; "ld*" are row pitches in ELEMENTS.
 *  - rollout arrays are time-major [T, N] (env contiguous); `src_idx` arrays hold buffer offsets t*N+e.
 */
#ifndef B200RL_H
#define B200RL_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200RL_OK 0
#define B200RL_ERR_ARG (-1)
#define B200RL_ERR_CUDA (-2)
#define B200RL_ERR_UNSUPPORTED (-3)
#define B200RL_ERR_DRIVER (-4)

/* GEMM epilogues */
#define B200RL_MODE_F16_ACT 0    /* C16 = act(alpha*acc + bias)                      (forward)            */
#define B200RL_MODE_F32_STORE 1  /* C32 = alpha*acc + bias                           (heads)              */
#define B200RL_MODE_F32_ATOMIC 2 /* C32 += alpha*acc (split-K parts added in order) (weight gradients)   */
#define B200RL_MODE_F16_DACT 3   /* C16 = alpha*acc * act'(saved)                    (data gradients)     */
#define B200RL_MODE_F16_SHUFFLE 4 /* conv data gradient, pixel-shuffle scatter: row (n,i,j), col (py,px,c)
                                     -> dx[n, s*i+py, s*j+px, c] * act'(saved there)  (b200rl_conv_gemm only) */
#define B200RL_ACT_NONE 0
#define B200RL_ACT_RELU 1
#define B200RL_ACT_TANH 2

const char* b200rl_last_error(void);
int b200rl_version(void);

/* GAE(lambda) backward scan: baselines/ppo2/runner.py:53-65 (bit-exact, float64 carry).
 * dones[t] = done BEFORE step t (runner.py:34); last_dones = runner.dones after the last step.
 * variant: -1 auto, 0 register-prefetch kernel, 1 TMA-bulk pipelined kernel (needs N % 32 == 0). */
int b200rl_gae_scan(const float* rewards, const float* values, const uint8_t* dones, const float* last_values,
                    const uint8_t* last_dones, float* advs, float* returns, int T, int N, double gamma, double lam,
                    int variant, void* stream);

/* fp16 x fp16 -> fp32 wgmma GEMM: tf.matmul a2c/utils.py:63; after im2col also tf.nn.conv2d a2c/utils.py:56
 * and their gradients (ppo2/model.py:102).
 *   mn_major = 0 : A[M,K] (lda), B[N,K] (ldb), C = A * B^T
 *   mn_major = 1 : A[K,M] (lda), B[K,N] (ldb), C = A^T * B   (reduction over rows; use split_k > 1)
 * max_ctas <= 0 : one persistent CTA per SM. */
int b200rl_gemm_f16(const void* A, const void* B, void* C, const float* bias, const void* saved, int M, int N, int K,
                    long long lda, long long ldb, long long ldc, long long ld_saved, int mn_major, int mode, int act,
                    float alpha, int split_k, int max_ctas, int rm_C, int rm_OW, int rm_Wg, const void* saved_bits,
                    void* stream);
/* saved_bits (MODE_F16_DACT with ReLU, optional): uint16 words, bit k of word (row*ld_saved + col)/16 set iff the saved
 * activation element (row, col + k) > 0 -- read instead of `saved` (16x less mask traffic; conv_shift_fwd emits it). */
/* rm_C > 0 (fp16 outputs only): output column pix*rm_C + c is stored at ((pix/rm_OW)*rm_Wg + pix%rm_OW)*rm_C + c,
 * i.e. a [.., OH, OW, C] row is scattered into a zero-bordered [.., Hg, Wg, C] grid (fc1 dgrad -> conv3's dY). */

/* Shift-GEMM convolutions (tf.nn.conv2d a2c/utils.py:56 + gradients): stride-1 conv over X[(n,y,x) rows, C]
 * (C = 64 or 128; strided convs arrive space-to-depth transformed).  Each X row is loaded into smem once; filter
 * tap t is the same buffer read through a descriptor shifted by shifts[t] rows.
 *   fwd  : out[map(n,y,x), :N] = act(sum_t X[m+shift_t] * W[:, t*C:(t+1)*C]^T + bias)   for y < vy, x < vx
 *          dact = 1: out = (sum_t ...) * (saved activation at smap(n,y,x) > 0) with the mask read from saved_bits,
 *          or out = sum_t ... without saved_bits  (data gradient: X = zero-bordered dY, shifts <= 0)
 *   omap / smap: {mode, sN, sY, sX, Cq, s}: 0 = n*sN+y*sY+x*sX+col; 1 = depth->space; 2 = space->depth
 *   wgrad: G[t*C + c, n] += alpha * sum_m X[m+shift_t, c] * dY[m, n]  (dY on X's grid, zero at invalid positions) */
int b200rl_conv_shift_fwd(const void* X, long long B, int Hg, int Wg, int C, const void* W, long long ldw, int N,
                          int taps, const int* shifts, int vy, int vx, void* out, const long long* omap,
                          const long long* smap, const float* bias, int act, int dact, float alpha,
                          const void* u8_x, const long long* u8_idx, int u8_H, int u8_W, int u8_C, int u8_s,
                          void* act_bits_out, const void* saved_bits, void* stream);
/* act_bits_out (forward, optional): uint16[numel(out)/16]; bit k of word e/16 is set iff out element e+k > 0 (e = the
 * element offset the output map produces, always a multiple of 16).  saved_bits (dact, optional): the same array for
 * the saved activation, addressed through smap (1 bit instead of 16 per element of backward HBM traffic).
 * u8_x != NULL (first layer): X is ignored; producer warps gather uint8 images u8_x[u8_idx[n], H, W, C], cast them
 * to fp16 and build the space-to-depth (factor u8_s) tile directly in shared memory (models.py:19, ppo2.py:165). */
int b200rl_conv_shift_wgrad(const void* X, long long rows, int C, const void* dY, int N, int taps, const int* shifts,
                            float* G, long long ldg, float alpha, float* gbias, float alpha_b, int max_ctas,
                            const void* u8_x, const long long* u8_idx, int u8_H, int u8_W, int u8_C, int u8_s,
                            int kx, void* stream);
/* kx > 1 ("x-fold"): the filter is ky rows of kx horizontally adjacent taps (row shift of tap (a, b) = a*Wg + b).
 * `shifts` then lists only the ky row shifts a*Wg; tap (a, b) reads X shifted by shifts[a] + b, and G keeps its
 * [(a*kx + b)*C + c, n] row order. */   /* gbias != NULL: gbias[n] += alpha_b * sum_m dY[m, n] (fused) */

/* Implicit-GEMM convolution (tf.nn.conv2d a2c/utils.py:56 and its gradients): the A operand is read
 * straight from the NHWC fp16 activation x[B,H,W,C] by TMA im2col mode (C = 16, 32 or 64 channels per tap).
 *   kind 0: out[B*OH*OW, N] = patches(x) * Wt^T, Wt = [N, R*S*C] fp16 (ldb); modes F16_ACT / F16_DACT /
 *           F16_SHUFFLE (data gradient of a stride-s conv written through the sh_* geometry)
 *   kind 1: out[R*S*C, N] (fp32, ldc) += alpha * patches(x)^T * dz, dz = [B*OH*OW, N] fp16 (ldb); split_k >= 1 */
int b200rl_conv_gemm(const void* x, long long B, int H, int W, int C, int R, int S, int stride_h, int stride_w,
                     int pad_h, int pad_w, int OH, int OW, const void* Wt_or_dz, long long ldb, void* out,
                     long long ldc, const float* bias, const void* saved, long long ld_saved, int N, int kind,
                     int mode, int act, float alpha, int split_k, int sh_H, int sh_W, int sh_C, int sh_s,
                     void* stream);
/* fp16 weight operand for the pixel-shuffle data gradient: out[s*s*Cin, ceil(R/s)^2*Cout] from HWIO fp32 w */
int b200rl_dgrad_weights(const float* w, void* out, int R, int S, int Cin, int Cout, int s, long long ld,
                         void* stream);

/* conv lowering (tf.nn.conv2d NHWC, a2c/utils.py:37-56; SAME padding for tf.contrib convolution2d,
 * common/models.py:241).  src_is_u8 fuses tf.cast(uint8->float) of models.py:19 and, through src_idx,
 * the minibatch gather arr[mbinds] of ppo2/ppo2.py:165. */
int b200rl_im2col(const void* x, int src_is_u8, const long long* src_idx, void* cols, long long B, int H, int W,
                  int C, int rf, int stride, int same_pad, void* stream);
/* gather + uint8->fp16 + space-to-depth: out[b,Y,X,(dy*s+dx)*C+c] = x[src_idx[b], s*Y+dy, s*X+dx, c] */
/* Device half of VecFrameStack.step_wait (common/vec_env/vec_frame_stack.py:17-25): for N envs of `pixels` pixels,
 * out[n, p, :] = roll(prev[n, p, :], -1) (one channel, as the reference does); zeroed where news[n]; the last c
 * bytes = frame[n, p, :].
 * uint8 tensors: prev/out [N, pixels, nstack*c], frame [N, pixels, c], news [N].  out must not alias prev. */
int b200rl_frame_stack(const void* prev, const void* frame, const void* news, void* out, long long N, long long pixels,
                       int nstack, int c, void* stream);

int b200rl_s2d_gather(const void* x, const long long* src_idx, void* out, long long B, int H, int W, int C, int s,
                      void* stream);
int b200rl_col2im(const void* dcols, const void* saved, void* dx, long long B, int H, int W, int C, int rf,
                  int stride, int same_pad, int act, void* stream);
int b200rl_colsum(const void* dz, float* db, long long rows, int C, long long ld, float alpha, void* stream);

/* act path: PolicyWithValue.step common/policies.py:77-96; CategoricalPd.sample/neglogp
 * common/distributions.py:164-201; DiagGaussianPd :238-248.  noise == NULL -> counter-based Philox, uniform j of
 * row b = word j&3 of philox4(seed, b, j>>2, offset).
 * cat_step also replaces MultiCategoricalPd.sample/neglogp (distributions.py:76-94,206-225): seg_off = device int32
 * [nseg + 1] offsets of the components' logit blocks in the row (seg_off[nseg] == nA), actions = [B, nseg] indices
 * inside each block, neglogp = the components' sum.  seg_off == NULL: one block [0, nA) (Discrete), actions [B]. */
int b200rl_cat_step(const float* logits, long long ld, int nA, const int* seg_off, int nseg, const float* vpred,
                    long long ldv, const float* uniforms, unsigned long long seed, unsigned long long offset,
                    const unsigned long long* offset_dev, long long* actions, float* values, float* neglogp,
                    long long B, void* stream);
/* BernoulliPd.sample/neglogp (distributions.py:115-128,254-276): actions float32 [B, n] = (u < sigmoid(l)),
 * neglogp = sum sigmoid_cross_entropy_with_logits(l, x). */
int b200rl_bern_step(const float* logits, long long ld, int n, const float* vpred, long long ldv,
                     const float* uniforms, unsigned long long seed, unsigned long long offset,
                     const unsigned long long* offset_dev, float* actions, float* values, float* neglogp, long long B,
                     void* stream);
int b200rl_gauss_step(const float* mean, long long ld, const float* logstd, int d, const float* vpred,
                      long long ldv, const float* normals, unsigned long long seed, unsigned long long offset,
                      const unsigned long long* offset_dev, float* actions, float* values, float* neglogp,
                      long long B, void* stream);
/* Scalars that change between replays of a CUDA-graph-captured launch sequence live in device memory:
 *   *_dev arguments (offset_dev of the samplers, cliprange_dev of the losses, lr_t_dev of clip_adam), when non-NULL,
 *   override the by-value argument; set_scalars writes up to 4 floats from its own kernel arguments (no host staging
 *   buffer to race with); counter_add advances the sampler's stream position after each acting pass. */
int b200rl_set_scalars(float* dst, int n, float a, float b, float c, float d, void* stream);
/* Device minibatch shuffle: ppo2/ppo2.py:160 (np.random.shuffle(inds)) + the env-major -> buffer index map of sf01
 * (ppo2/runner.py:69-74).  out[i] = offset of sample pi(i), pi = keyed Feistel bijection of [0, n) with cycle walking;
 * T > 0: flat index j = e*T + t -> t*N + e (T*N == n); T == 0: out[i] = pi(i). */
int b200rl_shuffle_indices(long long* out, long long n, unsigned long long key, long long T, long long N, void* stream);
int b200rl_counter_add(unsigned long long* ctr, unsigned long long inc, void* stream);

/* per-minibatch advantage moments: ppo2/model.py:136-139.  out = {mean, std} (float64). */
int b200rl_adv_stats(const float* returns, const float* values, const long long* src_idx, long long M, double* out,
                     void* stream);

/* PPO2 loss + gradient w.r.t. head outputs: ppo2/model.py:57-91.  stats[5] += per-sample sums of
 * {pg_loss, vf_loss, entropy, approxkl, clipfrac} (model.py:115); gradients in "sum" scaling.
 * cat_loss: Categorical (distributions.py:164-198; seg_off == NULL, actions [*]) or MultiCategorical
 * (distributions.py:76-94,206-225; seg_off / nseg as for cat_step, actions [*, nseg]); bern_loss: Bernoulli
 * (distributions.py:115-128,254-276, actions float32 [*, n]). */
int b200rl_cat_loss(const float* logits, long long ld, int nA, const int* seg_off, int nseg, const float* vpred,
                    long long ldv, const long long* actions, const long long* src_idx, const float* returns,
                    const float* old_values, const float* old_neglogp, const double* adv_stats, float cliprange,
                    float ent_coef, float vf_coef, void* dlogits, long long ld_dl, void* dv, long long ld_dv,
                    double* stats, long long B, const float* cliprange_dev, void* stream);
int b200rl_bern_loss(const float* logits, long long ld, int n, const float* vpred, long long ldv,
                     const float* actions, const long long* src_idx, const float* returns, const float* old_values,
                     const float* old_neglogp, const double* adv_stats, float cliprange, float ent_coef,
                     float vf_coef, void* dlogits, long long ld_dl, void* dv, long long ld_dv, double* stats,
                     long long B, const float* cliprange_dev, void* stream);
int b200rl_gauss_loss(const float* mean, long long ld, const float* logstd, int d, const float* vpred,
                      long long ldv, const float* actions, const long long* src_idx, const float* returns,
                      const float* old_values, const float* old_neglogp, const double* adv_stats, float cliprange,
                      float ent_coef, float vf_coef, void* dmean, long long ld_dm, void* dv, long long ld_dv,
                      float* dlogstd, float inv_M, double* stats, long long B, const float* cliprange_dev,
                      void* stream);

/* optimiser: tf.clip_by_global_norm ppo2/model.py:105-107, tf.clip_by_norm deepq/build_graph.py:416-421,
 * tf.train.AdamOptimizer ppo2/model.py:100 == common/mpi_adam.py:37-42. lr_t = lr*sqrt(1-b2^t)/(1-b1^t). */
int b200rl_sumsq(const float* g, long long n, double* out, void* stream);
int b200rl_seg_sumsq(const float* g, const long long* seg_off, int nseg, double* out, void* stream);
int b200rl_clip_adam(float* p, const float* g, float* m, float* v, long long n, float lr_t, float beta1, float beta2,
                     float eps, float clip, const double* sumsq, const long long* seg_off, int nseg,
                     const float* lr_t_dev, void* stream);
/* acc += g * clip/max(||g||, clip) * weight (clip <= 0: no clipping): the clipped per-microbatch gradients that
 * ppo2/microbatched_model.py:60-70 sums and averages before one apply_gradients. */
int b200rl_clip_accumulate(const float* g, float* acc, long long n, float clip, float weight, const double* sumsq,
                           void* stream);
/* Soft (Polyak) target update t <- float32(keep) * t + float32(mix) * s, unfused, over (t0, s0, n0) and (t1, s1, n1)
 * (t1 may be NULL) in one launch: DDPG's (1 - tau, tau) (ddpg/ddpg_learner.py:36-47), HER's (polyak, 1 - polyak)
 * (her/ddpg.py:398-399). */
int b200rl_soft_update(float* t0, const float* s0, long long n0, float* t1, const float* s1, long long n1, double keep,
                       double mix, void* stream);
int b200rl_cast_transpose(const float* src, int R, int C, void* dst, long long ld_dst, void* dstT, long long ld_t,
                          float scale, void* stream);
/* njobs cast_transpose operations in one launch.  jobs: device array of 56-byte records
 *   { const float* src; __half* dst; __half* dstT; long long ld_dst, ld_t; int R, C; float scale; int pad; }
 * (dst / dstT may be NULL); max_rows / max_cols: the largest R / C in the table. */
int b200rl_cast_transpose_batch(const void* jobs, int njobs, int max_rows, int max_cols, void* stream);
int b200rl_cast_f32_f16(const float* src, void* dst, long long rows, int cols, long long ld_src, long long ld_dst,
                        float scale, void* stream);

/* Vector-observation encoding: common/input.py:43-63 encode_observation (Box -> to_float, Discrete -> one_hot
 * :54-55), the optional clip((x - mean) / std, lo, hi) of common/policies.py:182-185, and the minibatch row gather of
 * ppo2/ppo2.py:165.
 * x: float32 [*, raw_dim]; out: fp16 [B, 2*in_pad] = [hi | lo] with hi = fp16(v), lo = fp16(v - hi), so the first
 * GEMM (K = 2*in_pad against [W ; W]) sees the float32 observation to 2^-22 relative (2^-25 absolute once lo is
 * fp16-subnormal, |v| < ~2^-3) instead of an fp16-rounded copy.  overflow (optional device int): set to 1 when an
 * encoded value has |v| >= 65520, which fp16 cannot hold (hi = +-inf); the caller must not use that output.
 * onehot_n > 0: x holds the Discrete value (raw_dim = 1), out row = one_hot(x, n).
 * onehot_n > 0 with seg_off (device int32 [nseg + 1]): x holds a MultiDiscrete value (raw_dim = nseg integers), out
 * row = concat_s one_hot(x[s], seg_off[s+1] - seg_off[s]) of width onehot_n = seg_off[nseg] (input.py:58-61). */
int b200rl_obs_encode(const float* x, const long long* src_idx, long long B, int raw_dim, int in_dim, int in_pad,
                      const float* mean, const float* inv_std, float clip_lo, float clip_hi, int onehot_n,
                      const int* seg_off, int nseg, void* out, int* overflow, void* stream);

/* prioritized replay: common/segment_tree.py:76-86 (__setitem__), :51-74 (reduce), :105-131
 * (find_prefixsum_idx); deepq/replay_buffer.py:107-115 (_sample_proportional), :157-165 (weights),
 * :169-191 (update_priorities).  Every pow is correctly rounded (csrc/pow_cr.cuh).
 * per_priorities: p = float32(|td| + float32(eps)), powered = p^alpha, max_priority = max(max_priority, p); bad
 * (device int, required) is set to 1 when some p is not > 0 (NaN or zero), where the reference asserts.
 * per_sample: bad (optional) is set to 1 when the tree holds a priority that is not > 0 or a descent ends past
 * n_stored; such a slot returns index 0, so an index never leaves the stored range.
 * per_pow: out[i] = x[i]^y, the pow of the leaves (the add path's max_priority ** alpha). */
int b200rl_tree_set(double* sum_tree, double* min_tree, long long capacity, const long long* idx, const double* vals,
                    int n, void* stream);
int b200rl_tree_range_sum(const double* tree, long long capacity, long long start, long long end, double* out,
                          void* stream);
int b200rl_per_sample(const double* sum_tree, const double* min_tree, long long capacity, long long n_stored,
                      const double* uniforms, int batch, double beta, long long* idx_out, double* w_out,
                      float* w_out_f32, int* bad, void* stream);
int b200rl_per_priorities(const float* td, int n, double eps, double alpha, double* powered, double* max_priority,
                          int* bad, void* stream);
int b200rl_per_pow(const double* x, int n, double y, double* out, void* stream);

/* DQN: deepq/build_graph.py:388-413 (double-Q target, Huber tf_util.py:39-45, importance weights),
 * deepq/models.py:38-40 (dueling), build_graph.py:184-191 (epsilon-greedy). s_* == NULL -> no dueling. */
int b200rl_dqn_td(const float* a_t, long long lda_t, const float* s_t, long long lds_t, const float* a_on,
                  long long lda_on, const float* s_on, long long lds_on, const float* a_tg, long long lda_tg,
                  const float* s_tg, long long lds_tg, int nA, const long long* idx, const long long* actions,
                  const float* rewards, const float* dones, const float* weights, float gamma, int double_q,
                  float* td_out, void* d_a, long long ld_da, void* d_s, long long ld_ds, double* loss_sum, int B,
                  void* stream);
int b200rl_dqn_act(const float* a, long long lda, const float* s, long long lds, int nA, float eps,
                   unsigned long long seed, unsigned long long step, const float* eps_dev,
                   const unsigned long long* step_dev, long long* actions, int B, void* stream);

/* LSTM recurrence: a2c/utils.py:84-97 lstm() over T steps (the cell of common/models.py lstm / cnn_lstm) and its
 * gradient (the BPTT TF derives for ppo2/model.py:102).  xg = x.Wx + b comes from b200rl_gemm_f16; rows are time-major
 * (row t*B + b), gate columns the reference's [i | f | o | u] blocks, the state [*, 2H] = [c | h] float32.
 * mask of row r = masks[mask_idx ? mask_idx[r] : r], "done before step t" (c and h are zeroed before the step);
 * environment b starts from state_in row state_idx ? state_idx[b] : b.  H = 64 or 128.
 * fwd: h_out fp16 [T*B, ldh]; optional state_out [B, 2H] (final c, h; may alias state_in when state_idx is NULL),
 * hprev_out fp16 [T*B, H] (masked h_{t-1}), gates_out [T*B, 4H] (sigma(i), sigma(f), sigma(o), tanh(u); may alias xg
 * when ldxg = 4H) and c_out [T*B, H], the last three for the backward.
 * bwd: dz fp16 [T*B, lddz] = d loss / d (pre-activation gates) from dh (d loss / d h_t, fp16) and the forward's saved
 * gates and c; whT = Wh^T fp16 [4H, H].  dWh = hprev^T dz, dWx = x^T dz, db = colsum(dz), dx = dz Wx^T follow on the
 * GEMM. */
int b200rl_lstm_seq_fwd(const float* xg, long long ldxg, const void* wh, const uint8_t* masks, const long long* mask_idx,
                        const float* state_in, const long long* state_idx, float* state_out, void* h_out,
                        long long ldh, void* hprev_out, float* gates_out, float* c_out, int T, int B, int H,
                        void* stream);
int b200rl_lstm_seq_bwd(const void* dh, long long lddh, const float* gates, const float* c, const uint8_t* masks,
                        const long long* mask_idx, const float* state_in, const long long* state_idx, const void* whT,
                        void* dz, long long lddz, int T, int B, int H, void* stream);

/* Row layer normalisation after a fully connected layer (tf.contrib.layers.layer_norm(center=True, scale=True):
 * common/models.py:97-98, deepq/models.py:24-25,34-35), csrc/layer_norm.cu.  N a multiple of 8 in [8, 1024]; row
 * pitches multiples of 8 elements; act 0 none, 1 relu, 2 tanh.
 * fwd: y fp16 [rows, ld_y] = act(gamma * (z - mean) / sqrt(var + eps) + beta) of z fp32 [rows, ld_z] (the
 * pre-activation a MODE_F32_STORE GEMM wrote), mean and biased variance per row.  A row's output depends on the row
 * alone.
 * bwd: du fp16 = d loss / d (gamma * xhat + beta); dz fp16 = d loss / d z (may be du's buffer);
 * dgamma += alpha * sum_r du * xhat, dbeta += alpha * sum_r du, summed over fixed 128-row slices in row order and
 * then over the slices in order.  The statistics are recomputed from z. */
int b200rl_ln_fwd(const float* z, long long ld_z, const float* gamma, const float* beta, void* y, long long ld_y,
                  long long rows, int N, int act, float eps, void* stream);
int b200rl_ln_bwd(const void* du, long long ld_du, const float* z, long long ld_z, const float* gamma, void* dz,
                  long long ld_dz, float* dgamma, float* dbeta, long long rows, int N, float alpha, float eps,
                  void* stream);

/* DQN parameter-space noise (deepq/build_graph.py:202-314; perturb_vars, mean_kl and the scale adaptation :258-287),
 * csrc/param_noise.cu.
 * param_perturb: for each of njobs device records {src_off, dst_off, len, perturb} (4 x int64; max_len = the largest
 * len): dst[dst_off + i] = src[src_off + i] + (perturb ? scale_dev[0] * n : 0), float32, n ~ N(0, 1) by Box-Muller over
 * the Philox4x32-10 stream (seed, position *offset_dev), or normals[dst_off + i] when normals is given.
 * dqn_param_noise_adapt: q, q_adapt = head outputs [B, ld] ([A | S] when dueling) of the plain and the adaptively
 * perturbed network; mean_kl_dev[0] = mean_b KL(softmax(Q_b) || softmax(Q_adapt_b)), summed in a fixed order, then
 * scale_dev[0] <- mean_kl < threshold_dev[0] ? scale * 1.01f : scale / 1.01f (:281-287).  One CTA. */
int b200rl_param_perturb(const float* src, float* dst, const void* jobs, int njobs, long long max_len,
                         const float* scale_dev, const float* normals, unsigned long long seed,
                         const unsigned long long* offset_dev, void* stream);
int b200rl_dqn_param_noise_adapt(const float* q, const float* q_adapt, long long ld, int nA, int dueling, int B,
                                 float* scale_dev, const float* threshold_dev, float* mean_kl_dev, void* stream);

/* VecNormalize (common/vec_env/vec_normalize.py:26-47) with RunningMeanStd (common/running_mean_std.py:22-33) on the
 * device, bit for bit with the numpy wrapper.  Running statistics: float64 [mean(D) | var(D) | std(D) | count],
 * std = sqrt(var + eps) written by every update.  Batch moments: float64 workspace [mean(D) | var(D)].
 * x: [N, D] rows of float32 (x_f64 = 0) or float64 (x_f64 = 1).
 * moments: np.mean / np.var of x along axis 0 in x's dtype -- column-sequential sums for D >= 2, numpy's pairwise sum
 *   for D == 1 (N <= 131072).
 * combine: the Chan update of rms with ws over a batch of N rows (running_mean_std.py:23-31), in float64 except
 *   bvar * N, which is a float32 product when the batch was float32 (ws_f32 = 1), as in numpy.
 * normalize: out f32 [N, D] = float32(clip((x - mean) / std, +-clip)) in float64, NaN kept (vec_normalize.py:43-47);
 *   rms == NULL: out = float32(x).
 * rewards: ret = ret * gamma + rew (float64 [N]); with rms (D = 1): update it with the pairwise moments of ret and
 *   out = float32(clip(rew / std, +-cliprew)), without: out = float32(rew); then ret = 0 where news[e] (news may be
 *   NULL).  rew: float32 (rew_f64 = 0) or float64 [N]; N <= 131072. */
int b200rl_vecnorm_moments(const void* x, int x_f64, long long N, int D, double* ws, void* stream);
int b200rl_vecnorm_combine(double* rms, const double* ws, int ws_f32, long long N, int D, double eps, void* stream);
int b200rl_vecnorm_normalize(const void* x, int x_f64, long long N, int D, const double* rms, double clip, float* out,
                             void* stream);
int b200rl_vecnorm_rewards(const void* rew, int rew_f64, const uint8_t* news, long long N, double* ret, double* rms,
                           double gamma, double eps, double cliprew, float* out, void* stream);
/* Latency probe for the moments' chain bound: one thread runs n dependent float32 (f64 = 0) / float64 adds;
 * out[0] = SM cycles per add.  out[1] seeds the chain (and receives its end). */
int b200rl_vecnorm_add_latency(int f64, long long n, double* out, void* stream);

/* DDPG (ddpg/ddpg_learner.py, ddpg/models.py), csrc/ddpg.cu.  The replay ring (ddpg/memory.py RingBuffer) holds float32
 * rows obs [limit, obs_dim], actions [limit, nA], rewards [limit], terminals [limit]; a ring selection `sel` is the
 * int64 device vector [start, idx_0 .. idx_{B-1}], sample b reads ring row (start + idx_b) % limit.
 * encode: fp16 [hi | lo] operand rows out [B, 2*in_pad] of [clip(normalize(obs), +-clip) | action] (:17-20, :108-111,
 *   models.py:43); normalize is (x - mean) / (std + 1e-8) when mean/std are given; act (may be NULL: obs-only rows)
 *   holds [*, nA] float32 rows read at the ring row (act_sel = 1) or at row b (act_sel = 0).  sel NULL: row b.
 *   overflow as in b200rl_obs_encode.
 * tanh: mu [B, nA] = tanhf(z[b * ldz + j]).  denorm: out[b] = q[b * ldq] * std + mean (mean NULL: q).
 * target: y[b] = r + (1 - d) * gamma * (Q'[b] * std + mean) (:134-135; mean NULL: Q'), r and d read at the ring row.
 * loss: one CTA; rows [0, B) of q are Q(s, a), rows [B, 2B) Q(s, mu(s)).  losses[0] = mean((Q - (y - mean) / (std +
 *   1e-8))^2), losses[1] = -mean(Q_mu * std + mean); dq (fp16, column 0 of row pitch lddq) = 2 (Q - y_n) on the first
 *   B rows and -std (-1 when mean is NULL) on the second: gradients of the sums, the backward scales by 1/B.
 * actor_dz: dz[b, j] = fp16(g[b, j] * (1 - mu[b, j]^2)).
 * l2: one CTA; segs = nseg int64 pairs {offset, len} into w / g; g += reg * w and *loss += sum_s reg * sum(w_s^2) / 2.
 * obs_rms: one CTA; RunningMeanStd state st float64 [sum(D) | sumsq(D) | count] updated by each of the n rows x[(pos0 +
 *   i) % limit] in order, then mean = float32(sum / count), std = sqrtf(max(float32(sumsq / count) - mean^2, 1e-2f))
 *   (common/mpi_running_mean_std.py:29-48).
 * ret_rms: one CTA; the same state with D = 1 updated once by the B values y (numpy's pairwise sums in float64), then
 *   with w0 given Pop-Art (:205-221) on the K-element output kernels w0, w1 and biases b0, b1.
 * pn_adapt: one CTA; *dist = sqrtf(mean((mu - mu_adapt)^2)) over n elements; *stddev (float64) /= 1.01 when dist >
 *   desired, else *= 1.01; *stddev32 = float32(*stddev) (noise.py:12-18). */
int b200rl_ddpg_encode(const float* obs, const long long* sel, long long limit, long long B, int obs_dim,
                       const float* mean, const float* std, float clip, const float* act, int act_sel, int nA,
                       int in_pad, void* out, int* overflow, void* stream);
int b200rl_ddpg_tanh(const float* z, long long ldz, float* mu, long long B, int nA, void* stream);
int b200rl_ddpg_denorm(const float* q, long long ldq, const float* mean, const float* std, float* out, long long B,
                       void* stream);
int b200rl_ddpg_target(const float* q1, long long ldq, const long long* sel, long long limit, const float* rewards,
                       const float* terminals, const float* mean, const float* std, float gamma, float* y, long long B,
                       void* stream);
int b200rl_ddpg_loss(const float* q, long long ldq, const float* y, const float* mean, const float* std, int B,
                     void* dq, long long lddq, float* losses, void* stream);
int b200rl_ddpg_actor_dz(const float* g, long long ldg, const float* mu, long long B, int nA, void* dz,
                         long long lddz, void* stream);
int b200rl_ddpg_l2(const float* w, float* g, const long long* segs, int nseg, float reg, float* loss, void* stream);
int b200rl_ddpg_obs_rms(const float* x, long long pos0, long long limit, long long n, int D, double* st, float* mean,
                        float* std, void* stream);
int b200rl_ddpg_ret_rms(const float* y, long long B, double* st, float* mean, float* std, float* w0, float* b0,
                        float* w1, float* b1, int K, void* stream);
int b200rl_ddpg_pn_adapt(const float* mu, const float* mu_adapt, long long n, double desired, double* stddev,
                         float* stddev32, float* dist, void* stream);

/* HER (her/ddpg.py, her/her_sampler.py, her/normalizer.py, her/actor_critic.py), csrc/her.cu.  The episode ring
 * (her/replay_buffer.py) holds float64 o [S, T+1, dimo], ag [S, T+1, dimg], g [S, T, dimg], u [S, T, dimu] and info
 * [S, T, ninfo]; a sample `sel` is the int64 device array [B, 3] of (episode slot, t, future_t), future_t = -1 keeping
 * the stored goal.
 * sample: g = future_t >= 0 ? ag[ep, future_t] : g[ep, t]; reward_type 1 (sparse) r = -(|ag[ep, t+1] - g| >
 *   threshold), 2 (dense) r = -|ag[ep, t+1] - g|, the norm in float64 with numpy's summation order; 0: r untouched.
 *   Then o, o_2 = o[ep, t], o[ep, t+1] and g, g_2 (minus ag[ep, t], ag[ep, t+1] when relative) are clipped to
 *   +-clip_obs in float64, rounded to float32, normalised as clip((x - mean) / std, +-norm_clip) and written as fp16
 *   [hi | lo] rows: xa [B, 2*pad_a] = [o | g], xta = [o_2 | g_2], xc rows [0, B) = [o | g | u / max_u] and rows [B, 2B)
 *   = [o | g] (action columns untouched), xtc [B, 2*pad_c] = [o_2 | g_2].  ag2_out / g_out (float64 [B, dimg]) and
 *   info_out ([B, ninfo]) receive ag[ep, t+1], the relabelled g and info[ep, t] when given.
 * obs_encode: xa (and xc when given) rows of [normalize(o) | normalize(g)] for n preprocessed float32 rows.
 * pi: pi[b, j] = max_u[j] * tanhf(z[b * ldz + j]); with xc, pi / max_u into columns col0 + j of its rows.
 * target: y = min(max(r + gamma * q, lo), hi).
 * loss: one CTA; *loss = mean((y - Q)^2) over rows [0, B) of q; dq column 0 = -2 (y - Q) there and -1 on rows [B, 2B);
 *   q_pi[b] = q[B + b].  Gradients of sums: the backward scales by 1/B.
 * actor_dz: dz = fp16((g / max_u + 2 action_l2 (pi / max_u) / (max_u dimu)) * max_u * (1 - tanh(z)^2)).
 * norm: two CTAs (o, g statistics, float32 state [sum(D) | sumsq(D) | count]); Normalizer.update over the N samples
 *   of sel (float32 sums when f32_o / f32_g, else float64 sums rounded to float32), then recompute_stats: count += N,
 *   sum += local, sumsq += local_sq, mean = sum / count, std = sqrt(max(eps^2, sumsq / count - mean^2)). */
int b200rl_her_sample(const double* o, const double* ag, const double* g, const double* u, const double* info, int T,
                      int dimo, int dimg, int dimu, int ninfo, const long long* sel, int B, int relative,
                      double clip_obs, const float* o_mean, const float* o_std, const float* g_mean,
                      const float* g_std, float norm_clip, const float* max_u, int reward_type, double threshold,
                      float* r, void* xa, void* xta, int pad_a, void* xc, void* xtc, int pad_c, double* ag2_out,
                      double* g_out, double* info_out, void* stream);
int b200rl_her_obs_encode(const float* o, const float* g, int n, int dimo, int dimg, const float* o_mean,
                          const float* o_std, const float* g_mean, const float* g_std, float norm_clip, void* xa,
                          int pad_a, void* xc, int pad_c, void* stream);
int b200rl_her_pi(const float* z, long long ldz, int B, int dimu, const float* max_u, float* pi, void* xc, int pad_c,
                  int col0, void* stream);
int b200rl_her_target(const float* q, long long ldq, const float* r, int B, float gamma, float lo, float hi, float* y,
                      void* stream);
int b200rl_her_loss(const float* q, long long ldq, const float* y, int B, void* dq, long long lddq, float* loss,
                    float* q_pi, void* stream);
int b200rl_her_actor_dz(const float* g, long long ldg, const float* z, long long ldz, const float* pi, int B, int dimu,
                        const float* max_u, float action_l2, void* dz, long long lddz, void* stream);
int b200rl_her_norm(const double* o, const double* ag, const double* g, int T, int dimo, int dimg,
                    const long long* sel, int N, int relative, double clip_obs, int f32_o, int f32_g, float* o_st,
                    float* o_mean, float* o_std, float* g_st, float* g_mean, float* g_std, float eps, void* stream);

/* ACER (acer/acer.py, acer/buffer.py), csrc/acer.cu.
 * step: actions int64 [B] = the Gumbel-max sample of b200rl_cat_step (same bits for the same seed / offset) and
 *   mu float32 [B, nA] = softmax(logits) (acer.py:105,214).
 * stack_obs: the replay ring holds frames [slots, nenv, nsteps + nstack, F, nc] (uint8, or float32 when f32) and
 *   dones uint8 [slots, nenv, nsteps]; for env e it reads slot idx[e] (idx NULL: slot 0) and writes the stacked
 *   observations of _stack_obs (buffer.py:124-140) to out [nenv * (nsteps + 1), F, nstack * nc], row e*(nsteps+1)+t.
 * take: the slot's actions int64 / rewards float32 / dones uint8 [nenv, nsteps], mus [nenv, nsteps, nA] and masks uint8
 *   [nenv, nsteps + 1], gathered like Buffer.take.
 * loss: acer.py:103-178 over rows e*(nsteps+1)+t of the train head outputs pi / q and the Polyak logits pol; actions,
 *   rewards, dones, mus are step rows e*nsteps+t.  dpi / dq (fp16, nA columns) get N * d loss / d [logits | q],
 *   N = nenv * nsteps, zero on each env's last row.  stats float64 [12]: loss, loss_q, entropy, loss_policy, loss_f,
 *   loss_bc, explained_variance, avg_norm_k, avg_norm_g, avg_norm_k_dot_g, avg_norm_adj, avg_norm_grads_f (the last
 *   five use adj = 0 when trust_region is 0).  f_out [rows, nA], v_out [rows], qret_out [N] may be NULL.
 *   The statistics are reduced through one device-wide scratch and completion counter, like b200rl_sumsq's: at most
 *   one acer_loss launch may be in flight per device (issue them on one stream).
 * clip_rmsprop_ema: g *= clip / max(sqrt(sumsq[0]), clip) (clip <= 0: none); TF RMSProp with momentum 0
 *   ms += (g^2 - ms) (1 - decay), p -= lr g / sqrt(ms + eps), lr read from lr_dev; then the moving average
 *   shadow -= (shadow - p) (1 - alpha) of the updated parameters. */
int b200rl_acer_step(const float* logits, long long ld, int nA, unsigned long long seed, unsigned long long offset,
                     const unsigned long long* offset_dev, long long* actions, float* mu, long long B, void* stream);
int b200rl_acer_stack_obs(const void* ring, int f32, long long slot_stride, const long long* idx, int nenv, int nsteps,
                          int nstack, long long F, int nc, const uint8_t* dones_ring, void* out, void* stream);
int b200rl_acer_take(const long long* idx, int nenv, int nsteps, int nA, const long long* actions_ring,
                     const float* rewards_ring, const float* mus_ring, const uint8_t* dones_ring,
                     const uint8_t* masks_ring, long long* actions, float* rewards, float* mus, uint8_t* dones,
                     uint8_t* masks, void* stream);
int b200rl_acer_loss(const float* pi, long long ldpi, const float* q, long long ldq, const float* pol, long long ldpol,
                     const long long* actions, const float* rewards, const uint8_t* dones, const float* mus, int nenv,
                     int nsteps, int nA, float gamma, float c, float delta, float q_coef, float ent_coef,
                     int trust_region, void* dpi, long long lddpi, void* dq, long long lddq, double* stats,
                     float* f_out, float* v_out, float* qret_out, void* stream);
int b200rl_clip_rmsprop_ema(float* p, const float* g, float* ms, float* shadow, long long n, const float* lr_dev,
                            float clip, const double* sumsq, float decay, float eps, float alpha, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H */
