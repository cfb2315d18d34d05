// eval.cu -- episode recorder for greedy evaluation episodes run over B envs on the device.
//
// Runs once after the reset and once after every env step of a greedy episode.  It copies what the reference's
// _log_control_data / _log_traffic_data keep per step (envs/cacc_env.py:81-112) out of the env's device state:
// the joint action and global reward of the step and the float64 headway / speed / acceleration of every vehicle.
// An env records until the step that returned done (Trainer.perform returns there, utils.py:199-214); later steps
// of an env that already ended are not recorded, so the host sees each episode exactly as long as the reference's.
//
// Records are [T+1][B][N] (env-major, so one env's step is N contiguous values); slot 0 is the reset state with
// us = 0 and reward 0, as CACCEnv.reset logs it.  One block handles 32 envs: each field is read [agent][env]
// (coalesced over envs) into a shared tile, then written [env][agent] at the env's own slot.
#include "common.cuh"

namespace {

constexpr int REC_ENVS = 32;
constexpr int REC_THREADS = 256;

__global__ void __launch_bounds__(REC_THREADS) eval_record_kernel(
    int N, int B, int T, int start, const int32_t* __restrict__ action, const double* __restrict__ greward,
    const float* __restrict__ done, const double* __restrict__ hs, const double* __restrict__ vs,
    const double* __restrict__ us, int32_t* __restrict__ alive, int32_t* __restrict__ steps,
    int32_t* __restrict__ rec_action, double* __restrict__ rec_reward, double* __restrict__ rec_hs,
    double* __restrict__ rec_vs, double* __restrict__ rec_us) {
  __shared__ double tile[NMARL_MAX_AGENT * (REC_ENVS + 1)];     // [agent][env], padded against bank conflicts
  __shared__ int s_slot[REC_ENVS];                               // slot this call writes per env, -1 = none
  const int tid = threadIdx.x, b0 = blockIdx.x * REC_ENVS;
  const int nb = min(REC_ENVS, B - b0);
  if (tid < REC_ENVS) {
    int slot = -1;
    if (tid < nb) {
      const int b = b0 + tid;
      if (start) {
        slot = 0;
        alive[b] = 1;
        steps[b] = 0;
        rec_reward[b] = 0.0;
      } else if (alive[b]) {
        const int s = steps[b] + 1;
        if (s <= T) {
          slot = s;
          steps[b] = s;
          rec_reward[(size_t)s * B + b] = greward[b];
        }
        if (s >= T || done[b] != 0.0f) alive[b] = 0;
      }
    }
    s_slot[tid] = slot;
  }
  // one field at a time through the tile: 0 = action, 1 = hs, 2 = vs, 3 = us
  for (int f = 0; f < 4; ++f) {
    __syncthreads();
    const double* src = f == 1 ? hs : f == 2 ? vs : us;
    for (int idx = tid; idx < N * REC_ENVS; idx += REC_THREADS) {
      const int i = idx / REC_ENVS, e = idx - i * REC_ENVS;
      if (e >= nb) continue;
      const size_t o = (size_t)i * B + b0 + e;
      double v;
      if (f == 0) v = start ? 0.0 : (double)action[o];
      else if (f == 3 && start) v = 0.0;
      else v = src[o];
      tile[i * (REC_ENVS + 1) + e] = v;
    }
    __syncthreads();
    for (int idx = tid; idx < N * REC_ENVS; idx += REC_THREADS) {
      const int e = idx / N, i = idx - e * N;
      const int s = e < nb ? s_slot[e] : -1;
      if (s < 0) continue;
      const double v = tile[i * (REC_ENVS + 1) + e];
      const size_t o = ((size_t)s * B + b0 + e) * N + i;
      if (f == 0) rec_action[o] = (int32_t)v;
      else if (f == 1) rec_hs[o] = v;
      else if (f == 2) rec_vs[o] = v;
      else rec_us[o] = v;
    }
  }
}

}  // namespace

extern "C" int nmarl_eval_record(int n_agent, int B, int T, int start, const int32_t* action, const double* greward,
                                 const float* done, const double* hs, const double* vs, const double* us,
                                 int32_t* alive, int32_t* steps, int32_t* rec_action, double* rec_reward,
                                 double* rec_hs, double* rec_vs, double* rec_us, void* stream) {
  NMARL_CHECK(n_agent > 0 && n_agent <= NMARL_MAX_AGENT, "eval_record: n_agent %d out of range (1..%d)", n_agent,
              NMARL_MAX_AGENT);
  NMARL_CHECK(B > 0 && T > 0, "eval_record: bad B %d / T %d", B, T);
  NMARL_CHECK(hs && vs && us && alive && steps && rec_action && rec_reward && rec_hs && rec_vs && rec_us,
              "eval_record: missing buffers");
  NMARL_CHECK(start || (action && greward && done), "eval_record: a step record needs action, greward and done");
  eval_record_kernel<<<(B + REC_ENVS - 1) / REC_ENVS, REC_THREADS, 0, (cudaStream_t)stream>>>(
      n_agent, B, T, start, action, greward, done, hs, vs, us, alive, steps, rec_action, rec_reward, rec_hs, rec_vs,
      rec_us);
  NMARL_LAUNCH_CHECK();
  return 0;
}
