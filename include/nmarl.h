/* nmarl.h -- C ABI of the H100-native networked-MARL hot path (libnmarl.so).
 *
 * Drop-in boundary (SURVEY.md 8b): the reference has no FFI; the surface it exposes is the
 * Python env/agent API.  This header is what the Python mirror of that API
 * (deeprl_network_b200/) binds with ctypes; each entry point names the reference code it
 * replaces (paths relative to the reference checkout).
 *
 * Conventions: extern "C"; every function returns 0 on success, non-zero on error
 * (message via nmarl_last_error(), thread-local); never throws; never allocates device memory and
 * keeps no global state -- the caller owns every buffer and passes raw device pointers plus an
 * explicit stream (cudaStream_t passed as void*).  The only library-owned resources are the ones
 * inside an opaque `nmarl_ctx`: one helper stream + two events used to fork side work beside the
 * BPTT chain, created by nmarl_create and freed by nmarl_destroy; entry points that fork take
 * the ctx through their argument block.  Re-entrant per ctx, not thread-safe per ctx.  All launches
 * are asynchronous on the given stream and are CUDA-graph capturable.  Device code is sm_90a only.
 *
 * Layout: every per-agent tensor is agent-major, env-minor: X[agent][env][feature]
 * (so an agent's rows are contiguous for its grouped GEMM, and the env kernel is coalesced
 * over envs).  Time-stacked buffers are [t][agent][env][feature].  fp32 unless stated.
 */
#ifndef NMARL_H
#define NMARL_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#pragma GCC visibility push(default)

/* 128: the env kernel's global reward reproduces np.sum bit for bit, whose 8-accumulator block covers at most
 * 128 values (NumPy's PW_BLOCKSIZE), and the model descriptor kernels take by value, 48 + 128 x 192 = 24 624 bytes,
 * stays inside the 32 764-byte kernel-parameter limit of sm_90 with room for each kernel's argument block       */
#define NMARL_MAX_AGENT 128
#define NMARL_MAX_NBR   4
/* LSTM width the tensor-core kernels are built for (num_lstm = 64 in every shipped config).  The FP32-FFMA kernels
 * also run n_h = 16 and 32 (n_h follows from nmarl_model.s_dim); any other model never takes the tensor-core path. */
#define NMARL_NH        64
/* n_a <= NMARL_MAX_NA - 1 = 15: the n_a logits and the value slot of a row fill at most 16 head columns (DESIGN 4.8) */
#define NMARL_MAX_NA    16

enum { NMARL_IA2C = 0, NMARL_NC = 1, NMARL_IC3 = 2, NMARL_DIAL = 3 };
enum { NMARL_SAMPLE_NONE = 0, NMARL_SAMPLE_UNIFORM = 1, NMARL_SAMPLE_PHILOX = 2, NMARL_SAMPLE_GREEDY = 3 };
enum { NMARL_CATCHUP = 0, NMARL_SLOWDOWN = 1 };

/* ---- model description (host builds it; passed by value to kernels) -------------------- */
typedef struct {
  int32_t n_nbr;                         /* |N(i)|                                             */
  int32_t nbr[NMARL_MAX_NBR];            /* neighbours, ascending (tf.boolean_mask order,       */
                                         /*   agents/utils.py:192-194)                          */
  int32_t n_recv;                        /* agents k with i in N(k)  (backward message scatter) */
  int32_t recv_agent[NMARL_MAX_NBR];
  int32_t recv_slot[NMARL_MAX_NBR];      /* position of i inside N(k)                           */
  int32_t x_nsrc;                        /* observation gather: x~ = concat_s obs[x_src[s]][:x_w] */
  int32_t x_src[NMARL_MAX_NBR + 1];
  int32_t x_w;
  /* offsets (floats, multiples of 4) into the flat parameter / gradient / rmsprop buffers; -1 = absent */
  int32_t o_w_ob, o_b_ob;                /* obs encoder  (IA2C: lstm_i/fc)                      */
  int32_t o_w_fp, o_b_fp;                /* fingerprint encoder (NC)                            */
  int32_t o_w_msg, o_b_msg;              /* message encoder (NC, IC3, DIAL).  DIAL, agent without  */
                                         /*   neighbours: o_b_msg = -1 drops the message AND the  */
                                         /*   own-action one-hot from s (lstm_dial_hetero,        */
                                         /*   agents/utils.py:683-685); lstm_dial keeps both      */
  int32_t o_wxh;                         /* [s_dim + 64][256] = wx rows then wh rows            */
  int32_t o_b;                           /* [256]                                               */
  int32_t o_mfc_w, o_mfc_b;              /* DIAL sender-side message fc                         */
  int32_t o_pi_w, o_pi_b, o_v_w, o_v_b;  /* heads                                               */
  /* offsets into the transposed-weight scratch (backward dgrad): */
  int32_t t_wxh;                         /* [256][s_dim + 64]                                   */
  int32_t t_w_msg;                       /* [64][k_m]                                           */
  int32_t t_mfc;                         /* [64][64]                                            */
  int32_t p_begin, p_end;                /* this agent's contiguous parameter range             */
  /* offsets into the packed tensor-core operand buffer (nmarl_pack_weights); -1 = absent:              */
  int32_t tp_x, tp_p, tp_m, tp_g, tp_mfc; /* encoders (N=64 tiles), gate [wx;wh] (N=256 tiles), DIAL mfc  */
  int32_t tp_gT, tp_mT, tp_mfcT;         /* backward: [wx;wh]^T (N=s_dim+64), w_msg^T (N=k_m), w_mfc^T     */
} nmarl_agent;

typedef struct {
  int32_t variant;                       /* NMARL_IA2C / NC / IC3 / DIAL                        */
  int32_t n_agent, n_a, s_dim;           /* s_dim = 3 * n_h (NC) or n_h, which gives the LSTM     */
                                         /*   width n_h = num_lstm: 16, 32 or 64 (NMARL_NH, the   */
                                         /*   only width with tensor-core kernels).  Every "64"   */
                                         /*   below is n_h, every "256" is 4 * n_h                */
  int32_t obs_stride;                    /* floats per obs row (>= x_w of every agent).  Only the  */
                                         /*   first x_w columns of a row are ever read: what lies  */
                                         /*   behind them is the caller's, and need not be zero    */
  int32_t kx_pad, kp_pad, km_pad;        /* padded (x4) widths of the x~ / p~ / m~ input segments */
  int32_t n_param, n_wt;                 /* flat buffer sizes (floats)                          */
  int32_t per_agent_norm;                /* 1: clip each agent's range separately (IA2C)        */
  int32_t n_wp;                          /* floats in the packed tensor-core operand buffer     */
  nmarl_agent agent[NMARL_MAX_AGENT];
} nmarl_model;

/* ---- CACC environment constants (envs/cacc_env.py:320-343) ----------------------------- */
typedef struct {
  int32_t n_agent, platoon_len;          /* platoon_len == n_agent for CACC; <n_agent: several  */
                                         /*   independent platoons (5x5-grid dynamics stub)     */
  int32_t scenario;                      /* NMARL_CATCHUP / NMARL_SLOWDOWN                      */
  int32_t T, batch_size;                 /* episode length in steps; collision-done period      */
  int32_t global_reward;                 /* coop_gamma < 0: reward := sum over agents           */
  double dt, h_min, h_star, h_s, h_g, v_max, v_star, u_min, u_max, rew_a, rew_b, G;
} nmarl_cacc_cfg;

/* ---- per-env CACC scenario parameters (table [B], one row per env) ----------------------------
 * Read by nmarl_cacc_reset_pe / nmarl_cacc_step_pe in place of the same-named fields of nmarl_cacc_cfg; every
 * other field (dt, h_min, T, batch_size, reward weights, ...) stays the config's.                     */
typedef struct {
  double h_star, v_star, h_s, h_g, v_max, u_min, u_max;
  int32_t scenario;                      /* NMARL_CATCHUP / NMARL_SLOWDOWN                      */
  int32_t pad_;
} nmarl_cacc_env_par;

/* Ranges nmarl_cacc_draw_par draws the table from: field k of a row (nmarl_cacc_env_par order, k < 7) is
 * lo[k] + u * (hi[k] - lo[k]); lo[k] == hi[k] gives exactly lo[k].  slowdown_prob < 0: every env runs
 * cfg->scenario; in [0, 1]: an env runs slow-down with this probability, else catch-up.             */
#define NMARL_ENV_PAR_FIELDS 7
typedef struct {
  double lo[NMARL_ENV_PAR_FIELDS], hi[NMARL_ENV_PAR_FIELDS];
  double slowdown_prob;
} nmarl_cacc_par_ranges;

const char* nmarl_last_error(void);
int nmarl_version(void);
/* ---- context (SURVEY 8b): owns the helper stream/events of the CURRENT device; no other state ---------- */
typedef struct nmarl_ctx nmarl_ctx;
int nmarl_create(nmarl_ctx** out);
int nmarl_destroy(nmarl_ctx* ctx);
/* size-of checks so the ctypes mirror can assert its struct layout */
int nmarl_sizeof_model(void);
int nmarl_sizeof_agent(void);
int nmarl_sizeof_cacc_cfg(void);
int nmarl_sizeof_cacc_env_par(void);
int nmarl_sizeof_cacc_par_ranges(void);
int nmarl_sizeof_fwd_args(void);
int nmarl_sizeof_bwd_args(void);

/* ---- K1: environment ---------------------------------------------------------------------
 * Replaces CACCEnv.reset/_init_catchup/_init_slowdown (envs/cacc_env.py:166-189,285-318) and
 * CACCEnv.step/_get_reward/_get_state (envs/cacc_env.py:191-242,40-79).  State is float64
 * (the reference is), observations are emitted as float32.
 *   hs,vs,us  double [N][B]     t int32 [B]     collision int32 [B]     v_init double [B]
 *   u01       double [B]  one uniform per env (the reference's single np.random.rand()); may be
 *             NULL -> Philox(seed, env, episode[b])
 *   mask      float [B] or NULL: reset only envs with mask != 0
 *   obs       float [N][B][obs_stride] (first 5 columns written); fp float [N][B][n_a] := 1/n_a
 */
int nmarl_cacc_reset(const nmarl_cacc_cfg* cfg, int B, const double* u01, const float* mask,
                     uint64_t seed, int32_t* episode,
                     double* hs, double* vs, double* us, int32_t* t, int32_t* collision, double* v_init,
                     float* obs, int obs_stride, float* fp, int n_a, void* stream);
/*   action int32 [N][B];  reward double [NR][B] (NR = 1 if global_reward else N);
 *   greward double [B];  done float [B] (1.0 / 0.0)                                           */
int nmarl_cacc_step(const nmarl_cacc_cfg* cfg, int B, int train_mode, const int32_t* action,
                    double* hs, double* vs, double* us, int32_t* t, int32_t* collision, const double* v_init,
                    float* obs, int obs_stride, double* reward, double* greward, float* done, void* stream);
/* The same two calls with per-env scenario parameters: env b reads h_star, v_star, h_s, h_g, v_max, u_min, u_max and
 * scenario from par[b] (device nmarl_cacc_env_par [B]) and behaves exactly like the one-env CACCEnv constructed
 * with those values.  Every other argument is that of nmarl_cacc_reset / nmarl_cacc_step.                      */
int nmarl_cacc_reset_pe(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, const double* u01,
                        const float* mask, uint64_t seed, int32_t* episode,
                        double* hs, double* vs, double* us, int32_t* t, int32_t* collision, double* v_init,
                        float* obs, int obs_stride, float* fp, int n_a, void* stream);
int nmarl_cacc_step_pe(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, int train_mode,
                       const int32_t* action, double* hs, double* vs, double* us, int32_t* t, int32_t* collision,
                       const double* v_init, float* obs, int obs_stride, double* reward, double* greward,
                       float* done, void* stream);
/* Draw the table rows of the envs with mask[b] != 0 (mask NULL: all) for the episode they are about to start:
 * call it before nmarl_cacc_reset_pe with the same seed, episode and mask (episode NULL: counter 0).
 * Keying: Philox4x32-10, key = (seed low, seed high), counter words = (c low, c high, env, 0x454e5650) with
 * c = episode[b] << 8 | k; u = ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53 from output words 0, 1.  k = 0..6 draw the
 * fields in nmarl_cacc_env_par order, k = 7 the scenario (slow-down iff u < slowdown_prob).
 * Checked before the launch, with a message each: lo <= hi for every field; cfg->h_min < h_s and h_s < h_g for
 * every draw (h_min < lo[h_s], hi[h_s] < lo[h_g]); u_min < 0 < u_max; v_star > 0; h_star > 0; slowdown_prob <= 1. */
int nmarl_cacc_draw_par(const nmarl_cacc_cfg* cfg, const nmarl_cacc_par_ranges* ranges, int B, uint64_t seed,
                        const int32_t* episode, const float* mask, nmarl_cacc_env_par* par, void* stream);
/* Envs sharded over processes: the same three calls for the global envs env0 .. env0 + B - 1 (the Philox lane of env
 * b is env0 + b, so a shard draws exactly what those envs of one process holding all of them draw).  The unsuffixed
 * calls are these with env0 = 0.  Refused unless env0 >= 0 (env0 + B - 1 then always fits the 32-bit lane word).   */
int nmarl_cacc_reset_shard(const nmarl_cacc_cfg* cfg, int B, const double* u01, const float* mask, uint64_t seed,
                           int32_t* episode, double* hs, double* vs, double* us, int32_t* t, int32_t* collision,
                           double* v_init, float* obs, int obs_stride, float* fp, int n_a, void* stream, int env0);
int nmarl_cacc_reset_pe_shard(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, const double* u01,
                              const float* mask, uint64_t seed, int32_t* episode, double* hs, double* vs, double* us,
                              int32_t* t, int32_t* collision, double* v_init, float* obs, int obs_stride, float* fp,
                              int n_a, void* stream, int env0);
int nmarl_cacc_draw_par_shard(const nmarl_cacc_cfg* cfg, const nmarl_cacc_par_ranges* ranges, int B, uint64_t seed,
                              const int32_t* episode, const float* mask, nmarl_cacc_env_par* par, void* stream,
                              int env0);

/* ---- K2-K6: fused message-gather + encoders + LSTM cell + heads ----------------------------
 * Replaces lstm / lstm_comm / lstm_ic3 / lstm_dial (agents/utils.py:87-115,118-217,344-417,
 * 515-599), the actor/critic heads (agents/policies.py:50-77,291-312), the 'p' / 'v' forward
 * protocol (agents/policies.py:119-134,215-230) and action sampling (utils.py:135-141).      */
typedef struct {
  int32_t B;
  const float* params;
  const float* obs;        /* [N][B][obs_stride]                                              */
  const float* fp;         /* [N][B][n_a]  previous-step policies (NC, DIAL) or NULL           */
  const float* done;       /* [B] pre-step done (1 -> own c,h zeroed; messages NOT masked)     */
  const float* c_in;       /* [N][B][64]                                                       */
  const float* h_in;       /* [N][B][64]                                                       */
  const float* msg_in;     /* DIAL: [N][B][64] relu(h_in W_mfc + b)                            */
  float* c_out;            /* p-call: new state (must not alias *_in)                          */
  float* h_out;
  float* msg_out;          /* DIAL p-call                                                      */
  float* pi;               /* p-call: [N][B][n_a]                                              */
  int32_t* action;         /* p-call: [N][B] or NULL                                           */
  int32_t sample_mode;     /* NMARL_SAMPLE_*                                                   */
  const double* uniforms;  /* [N][B] for NMARL_SAMPLE_UNIFORM                                  */
  const uint64_t* rng;     /* device [2] = {seed, counter} for NMARL_SAMPLE_PHILOX             */
  uint64_t rng_offset;     /* added to the device counter (distinct per call inside a graph)   */
                           /* Keying, which any other binding has to match: Philox4x32-10 with  */
                           /* key = (seed low, seed high) and counter words = (c low, c high,   */
                           /* lane, 0x41435431), c = rng[1] + rng_offset (mod 2^64), lane =     */
                           /* agent * B_total + env0 + env (the GLOBAL env index; env0 = 0 and  */
                           /* B_total = B unless the envs are sharded over processes);          */
                           /* u = ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53 from output words 0, 1. */
                           /* The call does not move rng[1]: a rollout passes offsets 0..T and  */
                           /* then calls nmarl_rng_advance(rng, T + 1).                          */
                           /* nmarl_cacc_reset draws from the same generator with counter =     */
                           /* episode << 8 | platoon, lane = env0 + env and the tag 0x454e5601, */
                           /* and nmarl_cacc_draw_par with counter = episode << 8 | parameter k, */
                           /* lane = env0 + env and the tag 0x454e5650 (env0: the *_shard calls) */
  const int32_t* act_in;   /* v-call: [N][B] same-step actions                                 */
  float* v;                /* v-call: [N][B]                                                   */
  const float* wpack;      /* packed 3xTF32 operands (nmarl_pack_weights) or NULL.  When set and  */
                           /* B % 128 == 0 and n_h == 64 the wgmma tensor-core kernel is used,  */
                           /* else FP32 FFMA (which ignores wpack)                              */
  int32_t* tc_err;         /* device int: tensor-core pipeline watchdog (0 = ok); may be NULL      */
  /* optional (p-call, tensor-core path only): save the activations BPTT needs while rolling out, so the
   * update can skip the separate training forward (same inputs, same weights => same numbers):         */
  float* sv_xin; float* sv_sh; float* sv_gates; float* sv_enc;   /* step-t slices, see nmarl_bwd_args      */
  int32_t state_fm;        /* layout of c/h: 1 = feature-major [N][64][B], required on the tensor-  */
                           /* core path except for DIAL; 0 = env-major, required everywhere else */
  /* envs sharded over processes: this call's B envs are the global envs env0 .. env0 + B - 1 of B_total, and the
   * sampling lane is keyed by the global index (see rng above), so that a sharded run samples what one process
   * holding all B_total envs samples.  B_total = 0 means B.  Refused unless env0 >= 0, env0 + B <= B_total and
   * every lane fits the 32-bit counter word (n_agent * B_total <= 2^32).                                        */
  int32_t env0;
  int32_t B_total;
} nmarl_fwd_args;

int nmarl_policy_step_p(const nmarl_model* m, const nmarl_fwd_args* a, void* stream);
int nmarl_policy_step_v(const nmarl_model* m, const nmarl_fwd_args* a, void* stream);
/* Pack the GEMM weights for the tensor-core path: per 32-wide k-block a [hi | lo] pair of 128B-swizzled
 * K-major tiles of W^T (hi = value rounded to TF32, lo = rounded remainder).  Call after every parameter
 * change.  wt (transposed weights scratch, n_wt floats) is also refreshed.                           */
int nmarl_pack_weights(const nmarl_model* m, const float* params, float* wt, float* wpack, void* stream);
/* DIAL only: msg[N][B][64] = relu(h W_mfc + b) (agents/utils.py:563-566); needed after a reset */
int nmarl_dial_msg(const nmarl_model* m, int B, const float* params, const float* h, float* msg, void* stream);
/* advance the device Philox counter by n (one tiny kernel; keeps graph replays fresh) */
int nmarl_rng_advance(uint64_t* rng, uint64_t n, void* stream);

/* ---- K7: n-step returns / advantages -------------------------------------------------------
 * Replaces add_transition's reward norm/clip (agents/models.py:26-32,198-209) and
 * _add_R_Adv / _add_s_R_Adv (agents/utils.py:763-775,800-816,837-855,888-912); float64 math,
 * float32 outputs like the reference.
 *   reward double [T][NR][B] raw;  value float [T][N][B];  done_post float [T][B];
 *   R_end float [N][B] (ignored where done_post[T-1] != 0 when zero_end_if_done);
 *   alpha < 0: global reward (NR == 1);  alpha > 0: spatial, dist int32 [N][N],
 *   alpha_pow double [maxdist+1] = alpha**d
 *   Rs, Advs float [T][N][B]                                                                 */
int nmarl_nstep_return_adv(int n_agent, int B, int T, int NR, const double* reward, const float* value,
                           const float* done_post, const float* R_end, int zero_end_if_done,
                           double gamma, double reward_norm, double reward_clip,
                           double alpha, const int32_t* dist, const double* alpha_pow, int n_pow,
                           float* Rs, float* Advs, void* stream);

/* ---- K8-K9: A2C loss, BPTT with message-gradient scatter, weight gradients ------------------
 * Replaces the 'backward' graph + prepare_loss + tf.gradients (agents/policies.py:20-39,
 * 232-264) for a batch of T steps starting from states_bw.  Buffers (all caller-owned):
 *   obs [T][N][B][obs_stride]  fp [T][N][B][n_a]  act int32 [T][N][B]  done_pre float [T][B]
 *   Rs, Advs float [T][N][B]
 *   h_seq, c_seq [T+1][N][B][64]  (index 0 = states_bw, filled by the caller)
 *   msg_seq      [T+1][N][B][64]  (DIAL; index 0 filled by nmarl_dial_msg)
 *   sv_xin [T][N][B][kx_pad+kp_pad+km_pad]  sv_sh [T][N][B][s_dim+64]  sv_gates [T][N][B][256]
 *   sv_enc [T][N][B][2*n_h] (IC3: n_h used; DIAL: 2*n_h)   sv_dlv [T][N][B][HW]
 *   (head width HW = 8 for n_a <= 7, 16 for n_a 8..15: a row holds d(loss)/d(logits) in columns [0, n_a),
 *    d(loss)/d(v) in column n_a and zeros behind it)
 *   sv_dz [T][N][B][4*n_h]   sv_dpre [T][N][B][3*n_h]   sv_dmp [T][N][B][n_h] (DIAL)
 *   (the widths written 64 / 256 / 192 in this block are n_h / 4*n_h / 3*n_h; the tensor-core path has n_h = 64)
 *   (tensor-core path: sv_dz = [T][N][B/32][256] gate-bias partial sums per 32 rows, sv_dpre unused)
 *   dh_rec, dc_rec [2][N][B][64]   dmsg [2][N][MAX_NBR][B][64]
 *   wt [n_wt] transposed weights   ws: split-K workspace of ws_floats floats
 *   loss_part float [T][N][tiles][4] partial sums (policy, value, entropy, pad) in 64-row tiles; each
 *             even tile holds the sum of 128 rows and the odd tile after it holds zeros
 *   grads [n_param] (fully overwritten)
 */
typedef struct {
  int32_t B, T;
  int32_t B_total;           /* global env count (all ranks) for the 1/(T*B_total) loss scale  */
  float v_coef, e_coef;
  const float* params;
  const float* obs; const float* fp; const int32_t* act; const float* done_pre;
  const float* Rs; const float* Advs;
  float* h_seq; float* c_seq; float* msg_seq;
  float* sv_xin; float* sv_sh; float* sv_gates; float* sv_enc; float* sv_dlv;
  float* sv_dz; float* sv_dpre; float* sv_dmp;
  float* dh_rec; float* dc_rec; float* dmsg;
  float* wt; float* ws; int64_t ws_floats;
  float* loss_part;
  float* grads;
  const float* wpack;        /* packed tensor-core operands or NULL (see nmarl_fwd_args)            */
  int32_t* tc_err;
  float* sv_dzT;             /* tensor-core path: dz^T as [T][N][B/32][256][32], one raw fp32 128B-swizzled tile per
                                32 env rows (the weight-gradient kernel splits it into 3xTF32 hi / lo itself)        */
  float* sv_dpT;             /* tensor-core path: encoder pre-activation grads^T, [T][N][B/32][ndp][32] raw tiles
                                like sv_dzT, ndp = 192 (NC) / 128 (IC3, DIAL) / 64 (IA2C).  On the tensor-core path
                                (wpack set, B % 128 == 0) sv_xin / sv_sh / sv_gates / sv_enc are FEATURE-MAJOR
                                [T][N][feature][B] and sv_dpre is unused.  With state_fm the done-masked own state
                                (rows s_dim.. of sv_sh) and, for NeurComm, the neighbour messages (the m~ block of
                                sv_xin) are NOT stored a second time: the weight-gradient kernel reads h_seq.        */
  int32_t state_fm;          /* h_seq / c_seq / msg_seq / dh_rec / dc_rec / dmsg are feature-major ([..][64][B]
                                instead of [..][B][64]): 1 on the tensor-core path except for DIAL, else 0           */
  nmarl_ctx* ctx;            /* required by nmarl_a2c_bptt / nmarl_a2c_backward (forked side work)                  */
  void** ev_step;            /* optional timing hooks (bench.py): 2*T cudaEvent_t, recorded on `stream` before /
                                after the cell kernel of reverse step t at [2t], [2t+1]; NULL = none               */
  void** ev_wgrad;           /* optional: 2 cudaEvent_t around the weight-gradient GEMM kernel; NULL = none         */
} nmarl_bwd_args;

int nmarl_loss_tiles(const nmarl_model* m, int B);       /* tiles per agent in loss_part      */
int64_t nmarl_ws_floats(const nmarl_model* m, int B, int T);   /* required workspace          */
/* float offset in sv_dzT (rows = 256) or sv_dpT (rows = ndp) of the tile of time step t, agent, 32-env block */
int64_t nmarl_operand_tile_offset(int rows, int t, int n_agent, int B, int agent, int block);
int nmarl_a2c_backward(const nmarl_model* m, const nmarl_bwd_args* a, void* stream);
/* the two halves: the training forward re-runs the T cell steps from states_bw and saves the activations
 * (sv_xin, sv_sh, sv_gates, sv_enc) and h_seq / c_seq / msg_seq.  nmarl_a2c_bptt computes the heads, the loss
 * partials and sv_dlv = d(loss)/d(logits, v) from h_seq, then the reverse pass and the weight gradients.
 * When the rollout p-calls already saved the activations (nmarl_fwd_args.sv_*), call nmarl_a2c_bptt alone. */
int nmarl_a2c_train_forward(const nmarl_model* m, const nmarl_bwd_args* a, void* stream);
int nmarl_a2c_bptt(const nmarl_model* m, const nmarl_bwd_args* a, void* stream);

/* ---- K10: global-norm clip + TF-semantics RMSProp -------------------------------------------
 * Replaces tf.clip_by_global_norm + tf.train.RMSPropOptimizer (agents/policies.py:34-39,
 * 259-264): g *= clip/max(|g|,clip); ms = rho*ms + (1-rho) g^2 (ms0 = 1); w -= lr*g/sqrt(ms+eps).
 *   lr: device float[1];  norm_out: device float [n_groups] (n_groups = n_agent if
 *   per_agent_norm else 1);  scratch: device float [>= 1024]                                  */
int nmarl_clip_rmsprop_step(const nmarl_model* m, float* params, float* grads, float* ms,
                            const float* lr, float max_grad_norm, float rho, float eps,
                            float* norm_out, float* scratch, void* stream);

/* ---- consensus update (IA2C_CU / `ma2c_cu`) ----------------------------------------------------
 * Replaces ConsensusPolicy._consensus_update (agents/policies.py:351-359, 401-426), run after every
 * optimizer step: agent i's LSTM variables (wx, wh, b -- one contiguous block of the flat buffer) become
 * the mean of the blocks of {i} + its neighbours (ascending index), all read BEFORE any is written.
 *   scratch: device float [n_agent * ((s_dim + n_h) * 4*n_h + 4*n_h)]                                         */
int nmarl_consensus_update(const nmarl_model* m, float* params, float* scratch, void* stream);

/* ---- greedy evaluation episodes: episode recorder ----------------------------------------------
 * Replaces the per-step recording of CACCEnv (_log_control_data / _log_traffic_data, envs/cacc_env.py:81-112,
 * 225-241) for B envs that run one greedy episode each.  Call once with start = 1 right after the reset (records
 * slot 0: the reset state, us = 0, reward 0; sets alive = 1, steps = 0), then with start = 0 after every env step.
 * An env whose alive flag is set records the step at slot steps + 1, then clears alive if that step returned done
 * (or reached slot T); envs that ended are not recorded again.  Reads the env's state in place; no host sync.
 *   action int32 [N][B], greward double [B], done float [B] (the step's outputs; unused when start = 1)
 *   hs, vs, us double [N][B] (env state after the step)     alive, steps int32 [B]
 *   rec_action int32 [T+1][B][N] (slot 0 = 0)   rec_reward double [T+1][B]
 *   rec_hs, rec_vs, rec_us double [T+1][B][N]                                                        */
int nmarl_eval_record(int n_agent, int B, int T, int start, const int32_t* action, const double* greward,
                      const float* done, const double* hs, const double* vs, const double* us,
                      int32_t* alive, int32_t* steps, int32_t* rec_action, double* rec_reward,
                      double* rec_hs, double* rec_vs, double* rec_us, void* stream);

#pragma GCC visibility pop
#ifdef __cplusplus
}
#endif
#endif /* NMARL_H */
