// bwd_common.cuh -- argument block of one reverse step, shared by cell_bwd_kernel (FFMA, train.cu) and
// tc_cell_bwd_kernel (tensor cores, tc_bwd.cu)
#pragma once
#include "common.cuh"

// the opaque context of the C ABI: helper stream + events for forked side work (created on the current device)
struct nmarl_ctx {
  cudaStream_t side;
  cudaEvent_t fork, join, heads;
  int device;
};

struct BwdK {
  int B, t, has_next;
  const float* params; const float* wt;
  const float* done_pre;        // [B] for step t
  const float* sv_gates; const float* sv_sh; const float* sv_enc; const float* sv_dlv;   // step t
  const float* c_prev; const float* c_cur;      // c_seq[t], c_seq[t+1]
  const float* dh_in; const float* dc_in; const float* dmsg_in;       // produced by step t+1
  float* dh_out; float* dc_out; float* dmsg_out;                       // consumed by step t-1
  float* sv_dz; float* sv_dpre;                                        // step t (tensor-core path: sv_dz = [N][B/32][256] gate-bias partials)
  const float* wpack; int* tc_err;                                     // tensor-core path (NULL -> FFMA)
  float* dzT;                                                          // step t: [N][B/32][256][32] tiles or NULL
  float* dpT;                                                          // step t: [N][B/32][ndp][32] tiles (encoder pre-act grads)
  int state_fm;                                                        // c/dh/dc/dmsg tensors are feature-major
  int ndp;                                                             // rows of a dpT tile: 192 (NC) / 128 (IC3, DIAL) / 64 (IA2C)
};

// Operand tiles of the tensor-core weight-gradient GEMMs (sv_dzT, sv_dpT): one raw fp32 tile of `rows` x 32 env rows
// (128B-swizzled, K-major over the envs) per (time step t, agent i, 32-env block rb), packed as [T][N][B/32][rows][32].
// Float offset of tile (t, i, rb); tc_cell_bwd_kernel writes and tc_wgrad_kernel reads every tile through it.
__host__ __device__ __forceinline__ size_t nmarl_tc_tile_offset(int rows, int t, int n_agent, int blocks, int i, int rb) {
  return (((size_t)t * n_agent + i) * blocks + rb) * (size_t)(rows * 32);
}

int nmarl_tc_launch_bwd(const nmarl_model* m, const BwdK& k, cudaStream_t st);
int nmarl_tc_wgrad_splits(int n_agent);
int64_t nmarl_tc_wgrad_ws_floats(const nmarl_model* m);
int nmarl_tc_ndp(const nmarl_model* m);
// all GEMM weight gradients (gate + encoders) of the tensor-core path; activations are feature-major
int nmarl_tc_launch_wgrads(const nmarl_model* m, int B, int T, const float* sv_sh, const float* sv_xin, const float* dzT,
                           const float* dpT, const float* sv_dz, float* ws, float* grads, int* err, cudaStream_t st, cudaStream_t st_bias,
                           void** ev_wgrad = nullptr,
                           const float* h_seq = nullptr, const float* done_pre = nullptr);
