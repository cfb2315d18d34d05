// env.cu -- K1: vectorised CACC platoon environment (float64 state, float32 observations).
// Compiled with --fmad=false: the reference is NumPy float64 without FMA contraction, and the
// kernels below keep its operation order so h, v, u and the rewards are bit-identical.
//
// Step kernel: one thread per env and agent row -- see cacc_step_kernel.  Reset kernel: one thread per env (off the
// critical path).  All arrays are [agent][env], so a warp's loads/stores are coalesced over envs.
//
// Restates envs/cacc_env.py: step :191-242, reward :40-52, observation :54-65,
// OVM :360-385, reset :166-189 / :285-318.
#include "common.cuh"

namespace {

struct EnvK {
  nmarl_cacc_cfg c;
  int B;
};

// The scenario parameters (h_star, v_star, h_s, h_g, v_max, u_min, u_max, scenario) come from `p`: the config itself
// (P = nmarl_cacc_cfg, the nmarl_cacc_reset / _step kernels) or env b's row of the per-env table (P = nmarl_cacc_env_par,
// the *_pe kernels); both structs name these fields alike.  Everything else is read from the config `c`.
template <bool PE>
__device__ __forceinline__ const auto& env_par(const nmarl_cacc_cfg& c, const nmarl_cacc_env_par& e) {
  if constexpr (PE) return e; else return c;
}

template <class P>
__device__ __forceinline__ double leader_speed(const P& p, double v_init, int t) {
  // v0s[t]: catch-up == v*; slow-down == np.linspace(v_init, v*, 300)[t] for t < 300 then v*
  if (p.scenario == NMARL_CATCHUP || t >= 299) return p.v_star;
  const double step = (p.v_star - v_init) / 299.0;
  return (double)t * step + v_init;
}

template <class P>
__device__ __forceinline__ double ovm_vh(const P& p, double h) {
  if (h <= p.h_s) return 0.0;
  if (h < p.h_g) return p.v_max / 2 * (1 - cos(3.141592653589793 * (h - p.h_s) / (p.h_g - p.h_s)));
  return p.v_max;
}

__device__ __forceinline__ double clipd(double x, double lo, double hi) { return fmin(fmax(x, lo), hi); }

template <class P>
__device__ __forceinline__ void write_obs(const nmarl_cacc_cfg& c, const P& p, int B, int b, int tcur, const double* hs,
                                          const double* vs, const double* us, const double* v_init, float* obs,
                                          int obs_stride) {
  const int L = c.platoon_len;
  double v_prev = 0.0;
  for (int i = 0; i < c.n_agent; ++i) {
    const int pos = i % L;
    const double v = vs[(size_t)i * B + b], h = hs[(size_t)i * B + b], u = us[(size_t)i * B + b];
    const double lead = pos ? v_prev : leader_speed(p, v_init[(size_t)(i / L) * B + b], tcur);
    float* o = obs + ((size_t)i * B + b) * obs_stride;
    o[0] = (float)((v - p.v_star) / p.v_star);
    o[1] = (float)clipd((lead - v) / 5.0, -2.0, 2.0);
    o[2] = (float)clipd((ovm_vh(p, h) - v) / 5.0, -2.0, 2.0);
    o[3] = (float)((h + (lead - v) * c.dt - p.h_star) / p.h_star);
    o[4] = (float)(u / p.u_max);
    v_prev = v;
  }
}

// PE: env b's scenario parameters come from par[b] (nmarl_cacc_reset_pe); without it, from the config.  par is the
// last parameter but one so that the other parameters keep their offsets and the PE = false code is that of the
// config-only kernel.  env0: global index of env 0 (the Philox lane of env b is env0 + b).
template <bool PE>
__global__ void cacc_reset_kernel(const EnvK k, const double* __restrict__ u01, const float* __restrict__ mask,
                                  uint64_t seed, int32_t* episode, double* hs, double* vs, double* us, int32_t* t,
                                  int32_t* collision, double* v_init, float* obs, int obs_stride, float* fp, int n_a,
                                  const nmarl_cacc_env_par* __restrict__ par, int env0) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int B = k.B;
  if (b >= B) return;
  if (mask != nullptr && mask[b] == 0.0f) return;
  const nmarl_cacc_cfg& c = k.c;
  nmarl_cacc_env_par pv = {};
  if constexpr (PE) pv = par[b];
  const auto& pr = env_par<PE>(c, pv);
  const int L = c.platoon_len, P = c.n_agent / L;
  uint32_t ep = 0;
  if (episode != nullptr) { ep = (uint32_t)episode[b]; episode[b] = (int32_t)(ep + 1); }
  for (int p = 0; p < P; ++p) {
    const double u = (u01 != nullptr) ? u01[(size_t)p * B + b] : philox_u01(seed, ((uint64_t)ep << 8) | (uint64_t)p, (uint32_t)env0 + (uint32_t)b, 0x454e5601u);
    const double scale = 1.5 + u;
    v_init[(size_t)p * B + b] = (pr.scenario == NMARL_SLOWDOWN) ? pr.v_star * scale : pr.v_star;
    for (int pos = 0; pos < L; ++pos) {
      const size_t o = (size_t)(p * L + pos) * B + b;
      hs[o] = (pr.scenario == NMARL_CATCHUP && pos == 0) ? pr.h_star * scale : pr.h_star;
      vs[o] = (pr.scenario == NMARL_SLOWDOWN) ? pr.v_star * scale : pr.v_star;
      us[o] = 0.0;
    }
  }
  t[b] = 0;
  collision[b] = 0;
  write_obs(c, pr, B, b, 0, hs, vs, us, v_init, obs, obs_stride);
  if (fp != nullptr) {
    const float p0 = (float)(1.0 / (double)n_a);
    for (int i = 0; i < c.n_agent; ++i)
      for (int a = 0; a < n_a; ++a) fp[((size_t)i * B + b) * n_a + a] = p0;
  }
}

// Block = 32 envs x NY = min(N, 32) agent rows; a warp is one agent over 32 consecutive envs (coalesced [agent][env]
// accesses) and thread row y handles agents y, y + NY, y + 2 NY, ... (at most ENV_J of them).  The serial vehicle chain
// of the reference disappears: vehicle i's update needs its predecessor's OLD and NEW speed, and the predecessor's new
// speed depends only on the predecessor's own old state (and on ITS predecessor's old speed) -- each thread recomputes
// it with the very same operations, so every number is bit-identical to the sequential sweep.  Every old value of the
// block's envs is read, __syncthreads, then the new state is written.
// The per-env reductions run in shared memory: collision = min headway (per-thread minima, then a min over the rows:
// min is exact in any order), global reward = np.sum over agents in the reference's order (sequential below 8 values,
// otherwise 8 strided accumulators + pairwise tree + sequential tail: NumPy's pairwise-sum block, which is the whole
// sum for N <= 128 = PW_BLOCKSIZE = NMARL_MAX_AGENT).
struct VehStep { double vn, uc; };
template <class P>
__device__ __forceinline__ VehStep veh_update(const nmarl_cacc_cfg& c, const P& p, int a, double h, double v,
                                              double lead) {
  const double al = (a & 1) ? 0.5 : 0.0;          // a_map = [(0,0),(.5,0),(0,.5),(.5,.5)]  (:275)
  const double be = (a & 2) ? 0.5 : 0.0;
  const double u = al * (ovm_vh(p, h) - v) + be * (lead - v);
  double vn = v + clipd(u, p.u_min, p.u_max) * c.dt;
  vn = clipd(vn, 0.0, p.v_max);
  VehStep r;
  r.vn = vn;
  r.uc = (vn - v) / c.dt;
  return r;
}

constexpr int ENV_ROWS = 32;                           // agent rows per block
constexpr int ENV_J = NMARL_MAX_AGENT / ENV_ROWS;      // agents per thread, at most
static_assert(NMARL_MAX_AGENT <= 128, "the global reward restates np.sum's pairwise block, exact up to 128 values");
static_assert(NMARL_MAX_AGENT % ENV_ROWS == 0, "agent rows");

// PE: as in cacc_reset_kernel.  Every thread of env b's column reads par[b] (the 32 rows share it through L1).
template <bool PE>
__global__ void __launch_bounds__(32 * ENV_ROWS) cacc_step_kernel(const EnvK k, int train_mode,
                                                                 const int32_t* __restrict__ action, double* hs,
                                                                 double* vs, double* us, int32_t* t, int32_t* collision,
                                                                 const double* __restrict__ v_init, float* obs,
                                                                 int obs_stride, double* reward, double* greward,
                                                                 float* done,
                                                                 const nmarl_cacc_env_par* __restrict__ par) {
  extern __shared__ double sm_env[];                 // [N][32] per-agent reward, then [NY][32] per-thread min headway
  // programmatic dependent launch: the CTAs may already be resident while the policy call that produces `action`
  // finishes; let the next policy call's CTAs start their prologue as well
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const nmarl_cacc_cfg& c = k.c;
  const int N = c.n_agent, L = c.platoon_len, B = k.B, NY = blockDim.y;
  const int e = threadIdx.x, y = threadIdx.y;
  const int b = blockIdx.x * 32 + e;
  const bool live = b < B;
  double* s_r = sm_env;
  double* s_h = sm_env + N * 32;
  __shared__ int s_col[32];
  int tcur = 0, col = 0;
  if (live) { tcur = t[b]; col = collision[b]; }
  nmarl_cacc_env_par pv = {};
  if constexpr (PE) { if (live) pv = par[b]; }
  const auto& p = env_par<PE>(c, pv);
  double hn[ENV_J], vn[ENV_J], un[ENV_J];            // new state (the old one after a collision)
  double hmin = 1e300;
#pragma unroll
  for (int j = 0; j < ENV_J; ++j) {
    hn[j] = vn[j] = un[j] = 0.0;
    const int i = y + NY * j;
    if (!live || i >= N) continue;
    const int pos = i % L;
    const size_t o = (size_t)i * B + b;
    const double h = hs[o], v = vs[o], uo = us[o];
    const double vi0 = v_init[(size_t)(i / L) * B + b];
    hn[j] = h; vn[j] = v; un[j] = uo;
    if (!col) {
      double lead, lead_next;
      if (pos) {
        // predecessor's old state and ITS leader's old speed -> predecessor's new speed, recomputed locally
        const double vp = vs[o - B], hp = hs[o - B];
        const double lead_p = (pos > 1) ? vs[o - 2 * (size_t)B] : leader_speed(p, vi0, tcur);
        lead = vp;
        lead_next = veh_update(c, p, action[o - B], hp, vp, lead_p).vn;
      } else {
        lead = leader_speed(p, vi0, tcur);
        lead_next = leader_speed(p, vi0, tcur + 1);
      }
      const VehStep s = veh_update(c, p, action[o], h, v, lead);
      vn[j] = s.vn; un[j] = s.uc;
      hn[j] = h + 0.5 * c.dt * (lead + lead_next - v - vn[j]);
      double r = -((hn[j] - p.h_star) * (hn[j] - p.h_star));
      r = r + (-c.rew_a * ((vn[j] - p.v_star) * (vn[j] - p.v_star)));
      r = r + (-c.rew_b * (un[j] * un[j]));
      if (train_mode) {
        const double m = fmin(hn[j] - 10.0, 0.0);
        r = r + (-5.0 * (m * m));
      } else {
        r = r + 0.0;
      }
      s_r[i * 32 + e] = r;
      hmin = fmin(hmin, hn[j]);
    }
  }
  s_h[y * 32 + e] = hmin;
  __syncthreads();                                   // every old value has been read
  if (live && !col) {
#pragma unroll
    for (int j = 0; j < ENV_J; ++j) {
      const int i = y + NY * j;
      if (i >= N) continue;
      const size_t o = (size_t)i * B + b;
      hs[o] = hn[j]; vs[o] = vn[j]; us[o] = un[j];
    }
  }
  if (live && y == 0) {
    double gsum;
    int cnew = col;
    if (!col) {
      double hm = 1e300;
      for (int yy = 0; yy < NY; ++yy) hm = fmin(hm, s_h[yy * 32 + e]);
      if (hm < c.h_min) { cnew = 1; collision[b] = 1; }         // collision latch (:42-44)
    }
    if (cnew) {
      gsum = -c.G * (double)N;                       // sum of N equal values is exact in any order
    } else {
      // np.sum order: sequential for N < 8, otherwise 8 strided accumulators + pairwise tree + tail
      double r8[8];
      double tail = 0.0;
      const int nblk = N - (N % 8);
      for (int j = 0; j < N; ++j) {
        const double r = s_r[j * 32 + e];
        if (N < 8) tail += r;
        else if (j < 8) r8[j] = r;
        else if (j < nblk) r8[j & 7] += r;
        else { if (j == nblk) tail = ((r8[0] + r8[1]) + (r8[2] + r8[3])) + ((r8[4] + r8[5]) + (r8[6] + r8[7])); tail += r; }
      }
      if (N >= 8 && N == nblk) tail = ((r8[0] + r8[1]) + (r8[2] + r8[3])) + ((r8[4] + r8[5]) + (r8[6] + r8[7]));
      gsum = tail;
    }
    s_col[e] = cnew;
    const int tn = tcur + 1;
    t[b] = tn;
    greward[b] = gsum;
    if (c.global_reward) reward[b] = gsum;
    const bool d = (cnew && (tn % c.batch_size == 0)) || (tn == c.T);
    done[b] = d ? 1.0f : 0.0f;
  }
  __syncthreads();                                   // the new state of the block's envs is in hs / vs / us
  if (!live) return;
#pragma unroll
  for (int j = 0; j < ENV_J; ++j) {
    const int i = y + NY * j;
    if (i >= N) continue;
    const int pos = i % L;
    const size_t o = (size_t)i * B + b;
    if (!c.global_reward) reward[o] = s_col[e] ? -c.G : s_r[i * 32 + e];   // frozen / new collision: -G (:193-194)
    // observation from the NEW state and the NEW time (:54-65); the predecessor's new speed is the value its thread
    // stored (frozen after a collision: the old one), bit-identical to the lead_next this thread computed
    const double lead = pos ? vs[o - B] : leader_speed(p, v_init[(size_t)(i / L) * B + b], tcur + 1);
    float* ob = obs + o * obs_stride;
    ob[0] = (float)((vn[j] - p.v_star) / p.v_star);
    ob[1] = (float)clipd((lead - vn[j]) / 5.0, -2.0, 2.0);
    ob[2] = (float)clipd((ovm_vh(p, hn[j]) - vn[j]) / 5.0, -2.0, 2.0);
    ob[3] = (float)((hn[j] + (lead - vn[j]) * c.dt - p.h_star) / p.h_star);
    ob[4] = (float)(un[j] / p.u_max);
  }
}

// One thread per env: the rows of the masked envs for the episode each is about to start (see nmarl_cacc_draw_par).
// env0: global index of env 0 (the Philox lane of env b is env0 + b).
__global__ void cacc_draw_par_kernel(const nmarl_cacc_par_ranges r, int scenario, int B, uint64_t seed,
                                     const int32_t* __restrict__ episode, const float* __restrict__ mask,
                                     nmarl_cacc_env_par* __restrict__ par, int env0) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (mask != nullptr && mask[b] == 0.0f) return;
  const uint64_t ep = (episode != nullptr) ? (uint64_t)(uint32_t)episode[b] : 0;
  double v[NMARL_ENV_PAR_FIELDS];
#pragma unroll
  for (int k = 0; k < NMARL_ENV_PAR_FIELDS; ++k) {
    const double u = philox_u01(seed, (ep << 8) | (uint64_t)k, (uint32_t)env0 + (uint32_t)b, 0x454e5650u);
    v[k] = r.lo[k] + u * (r.hi[k] - r.lo[k]);
  }
  if (r.slowdown_prob >= 0.0) {
    const double u = philox_u01(seed, (ep << 8) | (uint64_t)NMARL_ENV_PAR_FIELDS, (uint32_t)env0 + (uint32_t)b, 0x454e5650u);
    scenario = (u < r.slowdown_prob) ? NMARL_SLOWDOWN : NMARL_CATCHUP;
  }
  nmarl_cacc_env_par e;
  e.h_star = v[0]; e.v_star = v[1]; e.h_s = v[2]; e.h_g = v[3]; e.v_max = v[4]; e.u_min = v[5]; e.u_max = v[6];
  e.scenario = scenario;
  e.pad_ = 0;
  par[b] = e;
}

}  // namespace

static int cacc_reset(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, const double* u01,
                      const float* mask, uint64_t seed, int32_t* episode, double* hs, double* vs, double* us,
                      int32_t* t, int32_t* collision, double* v_init, float* obs, int obs_stride, float* fp, int n_a,
                      void* stream, int env0) {
  NMARL_CHECK(cfg && B > 0, "cacc_reset: bad arguments");
  NMARL_CHECK(env0 >= 0, "cacc_reset: env0 %d < 0", env0);
  NMARL_CHECK(cfg->platoon_len > 0 && cfg->n_agent % cfg->platoon_len == 0, "cacc_reset: n_agent %% platoon_len != 0");
  NMARL_CHECK(obs_stride >= 5, "cacc_reset: obs_stride < 5");
  EnvK k{*cfg, B};
  const int nt = 64;
  if (par != nullptr)
    cacc_reset_kernel<true><<<(B + nt - 1) / nt, nt, 0, (cudaStream_t)stream>>>(
        k, u01, mask, seed, episode, hs, vs, us, t, collision, v_init, obs, obs_stride, fp, n_a, par, env0);
  else
    cacc_reset_kernel<false><<<(B + nt - 1) / nt, nt, 0, (cudaStream_t)stream>>>(
        k, u01, mask, seed, episode, hs, vs, us, t, collision, v_init, obs, obs_stride, fp, n_a, nullptr, env0);
  NMARL_LAUNCH_CHECK();
  return 0;
}

static int cacc_step(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, int train_mode,
                     const int32_t* action, double* hs, double* vs, double* us, int32_t* t, int32_t* collision,
                     const double* v_init, float* obs, int obs_stride, double* reward, double* greward, float* done,
                     void* stream) {
  NMARL_CHECK(cfg && B > 0 && action, "cacc_step: bad arguments");
  NMARL_CHECK(cfg->platoon_len > 0 && cfg->n_agent % cfg->platoon_len == 0, "cacc_step: n_agent %% platoon_len != 0");
  NMARL_CHECK(cfg->n_agent > 0 && cfg->n_agent <= NMARL_MAX_AGENT, "cacc_step: n_agent %d out of range (1..%d)",
              cfg->n_agent, NMARL_MAX_AGENT);
  EnvK k{*cfg, B};
  const int rows = cfg->n_agent < ENV_ROWS ? cfg->n_agent : ENV_ROWS;
  const dim3 blk(32, rows);
  const size_t smem = (size_t)(cfg->n_agent + rows) * 32 * sizeof(double);     // <= 40 KB: no opt-in needed
  NMARL_CUDA(nmarl_launch(par != nullptr ? cacc_step_kernel<true> : cacc_step_kernel<false>, dim3((B + 31) / 32), blk,
                          smem, (cudaStream_t)stream, true, k, train_mode, action, hs, vs, us, t, collision, v_init,
                          obs, obs_stride, reward, greward, done, par));
  NMARL_LAUNCH_CHECK();
  return 0;
}

extern "C" int nmarl_cacc_reset_shard(const nmarl_cacc_cfg* cfg, int B, const double* u01, const float* mask,
                                      uint64_t seed, int32_t* episode, double* hs, double* vs, double* us, int32_t* t,
                                      int32_t* collision, double* v_init, float* obs, int obs_stride, float* fp, int n_a,
                                      void* stream, int env0) {
  return cacc_reset(cfg, nullptr, B, u01, mask, seed, episode, hs, vs, us, t, collision, v_init, obs, obs_stride, fp,
                    n_a, stream, env0);
}

extern "C" int nmarl_cacc_reset(const nmarl_cacc_cfg* cfg, int B, const double* u01, const float* mask, uint64_t seed,
                                int32_t* episode, double* hs, double* vs, double* us, int32_t* t, int32_t* collision,
                                double* v_init, float* obs, int obs_stride, float* fp, int n_a, void* stream) {
  return nmarl_cacc_reset_shard(cfg, B, u01, mask, seed, episode, hs, vs, us, t, collision, v_init, obs, obs_stride,
                                fp, n_a, stream, 0);
}

extern "C" int nmarl_cacc_step(const nmarl_cacc_cfg* cfg, int B, int train_mode, const int32_t* action, double* hs,
                               double* vs, double* us, int32_t* t, int32_t* collision, const double* v_init, float* obs,
                               int obs_stride, double* reward, double* greward, float* done, void* stream) {
  return cacc_step(cfg, nullptr, B, train_mode, action, hs, vs, us, t, collision, v_init, obs, obs_stride, reward,
                   greward, done, stream);
}

extern "C" int nmarl_cacc_reset_pe_shard(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B,
                                         const double* u01, const float* mask, uint64_t seed, int32_t* episode,
                                         double* hs, double* vs, double* us, int32_t* t, int32_t* collision,
                                         double* v_init, float* obs, int obs_stride, float* fp, int n_a, void* stream,
                                         int env0) {
  NMARL_CHECK(par != nullptr, "cacc_reset_pe: par is NULL");
  return cacc_reset(cfg, par, B, u01, mask, seed, episode, hs, vs, us, t, collision, v_init, obs, obs_stride, fp,
                    n_a, stream, env0);
}

extern "C" int nmarl_cacc_reset_pe(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, const double* u01,
                                   const float* mask, uint64_t seed, int32_t* episode, double* hs, double* vs,
                                   double* us, int32_t* t, int32_t* collision, double* v_init, float* obs,
                                   int obs_stride, float* fp, int n_a, void* stream) {
  return nmarl_cacc_reset_pe_shard(cfg, par, B, u01, mask, seed, episode, hs, vs, us, t, collision, v_init, obs,
                                   obs_stride, fp, n_a, stream, 0);
}

extern "C" int nmarl_cacc_step_pe(const nmarl_cacc_cfg* cfg, const nmarl_cacc_env_par* par, int B, int train_mode,
                                  const int32_t* action, double* hs, double* vs, double* us, int32_t* t,
                                  int32_t* collision, const double* v_init, float* obs, int obs_stride,
                                  double* reward, double* greward, float* done, void* stream) {
  NMARL_CHECK(par != nullptr, "cacc_step_pe: par is NULL");
  return cacc_step(cfg, par, B, train_mode, action, hs, vs, us, t, collision, v_init, obs, obs_stride, reward,
                   greward, done, stream);
}

extern "C" int nmarl_cacc_draw_par_shard(const nmarl_cacc_cfg* cfg, const nmarl_cacc_par_ranges* ranges, int B,
                                         uint64_t seed, const int32_t* episode, const float* mask,
                                         nmarl_cacc_env_par* par, void* stream, int env0) {
  static const char* const name[NMARL_ENV_PAR_FIELDS] = {"h_star", "v_star", "h_s", "h_g", "v_max", "u_min", "u_max"};
  NMARL_CHECK(cfg && ranges && par && B > 0, "cacc_draw_par: bad arguments");
  NMARL_CHECK(env0 >= 0, "cacc_draw_par: env0 %d < 0", env0);
  const nmarl_cacc_par_ranges& r = *ranges;
  for (int k = 0; k < NMARL_ENV_PAR_FIELDS; ++k)
    NMARL_CHECK(r.lo[k] <= r.hi[k], "cacc_draw_par: %s range [%g, %g] needs lo <= hi", name[k], r.lo[k], r.hi[k]);
  NMARL_CHECK(cfg->h_min < r.lo[2], "cacc_draw_par: needs h_min < h_s (h_min %g, h_s from %g)", cfg->h_min, r.lo[2]);
  NMARL_CHECK(r.hi[2] < r.lo[3], "cacc_draw_par: needs h_s < h_g for every draw (h_s up to %g, h_g from %g)",
              r.hi[2], r.lo[3]);
  NMARL_CHECK(r.hi[5] < 0.0, "cacc_draw_par: needs u_min < 0 (u_min up to %g)", r.hi[5]);
  NMARL_CHECK(r.lo[6] > 0.0, "cacc_draw_par: needs u_max > 0 (u_max from %g)", r.lo[6]);
  NMARL_CHECK(r.lo[1] > 0.0, "cacc_draw_par: needs v_star > 0 (v_star from %g)", r.lo[1]);
  NMARL_CHECK(r.lo[0] > 0.0, "cacc_draw_par: needs h_star > 0 (h_star from %g)", r.lo[0]);
  NMARL_CHECK(r.slowdown_prob <= 1.0, "cacc_draw_par: slowdown_prob %g > 1", r.slowdown_prob);
  const int nt = 128;
  cacc_draw_par_kernel<<<(B + nt - 1) / nt, nt, 0, (cudaStream_t)stream>>>(r, cfg->scenario, B, seed, episode, mask,
                                                                          par, env0);
  NMARL_LAUNCH_CHECK();
  return 0;
}

extern "C" int nmarl_cacc_draw_par(const nmarl_cacc_cfg* cfg, const nmarl_cacc_par_ranges* ranges, int B,
                                   uint64_t seed, const int32_t* episode, const float* mask, nmarl_cacc_env_par* par,
                                   void* stream) {
  return nmarl_cacc_draw_par_shard(cfg, ranges, B, seed, episode, mask, par, stream, 0);
}
