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

__device__ __forceinline__ double leader_speed(const nmarl_cacc_cfg& c, double v_init, int t) {
  // v0s[t]: catch-up == v*; slow-down == np.linspace(v_init, v*, 300)[t] for t < 300 then v*
  if (c.scenario == NMARL_CATCHUP || t >= 299) return c.v_star;
  const double step = (c.v_star - v_init) / 299.0;
  return (double)t * step + v_init;
}

__device__ __forceinline__ double ovm_vh(const nmarl_cacc_cfg& c, double h) {
  if (h <= c.h_s) return 0.0;
  if (h < c.h_g) return c.v_max / 2 * (1 - cos(3.141592653589793 * (h - c.h_s) / (c.h_g - c.h_s)));
  return c.v_max;
}

__device__ __forceinline__ double clipd(double x, double lo, double hi) { return fmin(fmax(x, lo), hi); }

__device__ __forceinline__ void write_obs(const nmarl_cacc_cfg& c, int B, int b, int tcur, const double* hs,
                                          const double* vs, const double* us, const double* v_init, float* obs,
                                          int obs_stride) {
  const int L = c.platoon_len;
  double v_prev = 0.0;
  for (int i = 0; i < c.n_agent; ++i) {
    const int pos = i % L;
    const double v = vs[(size_t)i * B + b], h = hs[(size_t)i * B + b], u = us[(size_t)i * B + b];
    const double lead = pos ? v_prev : leader_speed(c, v_init[(size_t)(i / L) * B + b], tcur);
    float* o = obs + ((size_t)i * B + b) * obs_stride;
    o[0] = (float)((v - c.v_star) / c.v_star);
    o[1] = (float)clipd((lead - v) / 5.0, -2.0, 2.0);
    o[2] = (float)clipd((ovm_vh(c, h) - v) / 5.0, -2.0, 2.0);
    o[3] = (float)((h + (lead - v) * c.dt - c.h_star) / c.h_star);
    o[4] = (float)(u / c.u_max);
    v_prev = v;
  }
}

__global__ void cacc_reset_kernel(const EnvK k, const double* __restrict__ u01, const float* __restrict__ mask,
                                  uint64_t seed, int32_t* episode, double* hs, double* vs, double* us, int32_t* t,
                                  int32_t* collision, double* v_init, float* obs, int obs_stride, float* fp, int n_a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int B = k.B;
  if (b >= B) return;
  if (mask != nullptr && mask[b] == 0.0f) return;
  const nmarl_cacc_cfg& c = k.c;
  const int L = c.platoon_len, P = c.n_agent / L;
  uint32_t ep = 0;
  if (episode != nullptr) { ep = (uint32_t)episode[b]; episode[b] = (int32_t)(ep + 1); }
  for (int p = 0; p < P; ++p) {
    const double u = (u01 != nullptr) ? u01[(size_t)p * B + b] : philox_u01(seed, ((uint64_t)ep << 8) | (uint64_t)p, (uint32_t)b, 0x454e5601u);
    const double scale = 1.5 + u;
    v_init[(size_t)p * B + b] = (c.scenario == NMARL_SLOWDOWN) ? c.v_star * scale : c.v_star;
    for (int pos = 0; pos < L; ++pos) {
      const size_t o = (size_t)(p * L + pos) * B + b;
      hs[o] = (c.scenario == NMARL_CATCHUP && pos == 0) ? c.h_star * scale : c.h_star;
      vs[o] = (c.scenario == NMARL_SLOWDOWN) ? c.v_star * scale : c.v_star;
      us[o] = 0.0;
    }
  }
  t[b] = 0;
  collision[b] = 0;
  write_obs(c, B, b, 0, hs, vs, us, v_init, obs, obs_stride);
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
__device__ __forceinline__ VehStep veh_update(const nmarl_cacc_cfg& c, int a, double h, double v, double lead) {
  const double al = (a & 1) ? 0.5 : 0.0;          // a_map = [(0,0),(.5,0),(0,.5),(.5,.5)]  (:275)
  const double be = (a & 2) ? 0.5 : 0.0;
  const double u = al * (ovm_vh(c, h) - v) + be * (lead - v);
  double vn = v + clipd(u, c.u_min, c.u_max) * c.dt;
  vn = clipd(vn, 0.0, c.v_max);
  VehStep r;
  r.vn = vn;
  r.uc = (vn - v) / c.dt;
  return r;
}

constexpr int ENV_ROWS = 32;                           // agent rows per block
constexpr int ENV_J = NMARL_MAX_AGENT / ENV_ROWS;      // agents per thread, at most
static_assert(NMARL_MAX_AGENT <= 128, "the global reward restates np.sum's pairwise block, exact up to 128 values");
static_assert(NMARL_MAX_AGENT % ENV_ROWS == 0, "agent rows");

__global__ void __launch_bounds__(32 * ENV_ROWS) cacc_step_kernel(const EnvK k, int train_mode,
                                                                 const int32_t* __restrict__ action, double* hs,
                                                                 double* vs, double* us, int32_t* t, int32_t* collision,
                                                                 const double* __restrict__ v_init, float* obs,
                                                                 int obs_stride, double* reward, double* greward,
                                                                 float* done) {
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
        const double lead_p = (pos > 1) ? vs[o - 2 * (size_t)B] : leader_speed(c, vi0, tcur);
        lead = vp;
        lead_next = veh_update(c, action[o - B], hp, vp, lead_p).vn;
      } else {
        lead = leader_speed(c, vi0, tcur);
        lead_next = leader_speed(c, vi0, tcur + 1);
      }
      const VehStep s = veh_update(c, action[o], h, v, lead);
      vn[j] = s.vn; un[j] = s.uc;
      hn[j] = h + 0.5 * c.dt * (lead + lead_next - v - vn[j]);
      double r = -((hn[j] - c.h_star) * (hn[j] - c.h_star));
      r = r + (-c.rew_a * ((vn[j] - c.v_star) * (vn[j] - c.v_star)));
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
    const double lead = pos ? vs[o - B] : leader_speed(c, v_init[(size_t)(i / L) * B + b], tcur + 1);
    float* ob = obs + o * obs_stride;
    ob[0] = (float)((vn[j] - c.v_star) / c.v_star);
    ob[1] = (float)clipd((lead - vn[j]) / 5.0, -2.0, 2.0);
    ob[2] = (float)clipd((ovm_vh(c, hn[j]) - vn[j]) / 5.0, -2.0, 2.0);
    ob[3] = (float)((hn[j] + (lead - vn[j]) * c.dt - c.h_star) / c.h_star);
    ob[4] = (float)(un[j] / c.u_max);
  }
}

}  // namespace

extern "C" int nmarl_cacc_reset(const nmarl_cacc_cfg* cfg, int B, const double* u01, const float* mask, uint64_t seed,
                                int32_t* episode, double* hs, double* vs, double* us, int32_t* t, int32_t* collision,
                                double* v_init, float* obs, int obs_stride, float* fp, int n_a, void* stream) {
  NMARL_CHECK(cfg && B > 0, "cacc_reset: bad arguments");
  NMARL_CHECK(cfg->platoon_len > 0 && cfg->n_agent % cfg->platoon_len == 0, "cacc_reset: n_agent %% platoon_len != 0");
  NMARL_CHECK(obs_stride >= 5, "cacc_reset: obs_stride < 5");
  EnvK k{*cfg, B};
  const int nt = 64;
  cacc_reset_kernel<<<(B + nt - 1) / nt, nt, 0, (cudaStream_t)stream>>>(k, u01, mask, seed, episode, hs, vs, us, t,
                                                                         collision, v_init, obs, obs_stride, fp, n_a);
  NMARL_LAUNCH_CHECK();
  return 0;
}

extern "C" int nmarl_cacc_step(const nmarl_cacc_cfg* cfg, int B, int train_mode, const int32_t* action, double* hs,
                               double* vs, double* us, int32_t* t, int32_t* collision, const double* v_init, float* obs,
                               int obs_stride, double* reward, double* greward, float* done, void* stream) {
  NMARL_CHECK(cfg && B > 0 && action, "cacc_step: bad arguments");
  NMARL_CHECK(cfg->platoon_len > 0 && cfg->n_agent % cfg->platoon_len == 0, "cacc_step: n_agent %% platoon_len != 0");
  NMARL_CHECK(cfg->n_agent > 0 && cfg->n_agent <= NMARL_MAX_AGENT, "cacc_step: n_agent %d out of range (1..%d)",
              cfg->n_agent, NMARL_MAX_AGENT);
  EnvK k{*cfg, B};
  const int rows = cfg->n_agent < ENV_ROWS ? cfg->n_agent : ENV_ROWS;
  const dim3 blk(32, rows);
  const size_t smem = (size_t)(cfg->n_agent + rows) * 32 * sizeof(double);     // <= 40 KB: no opt-in needed
  NMARL_CUDA(nmarl_launch(cacc_step_kernel, dim3((B + 31) / 32), blk, smem, (cudaStream_t)stream, true, k, train_mode,
                          action, hs, vs, us, t, collision, v_init, obs, obs_stride, reward, greward, done));
  NMARL_LAUNCH_CHECK();
  return 0;
}
