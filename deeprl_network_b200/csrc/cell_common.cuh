// cell_common.cuh -- argument block shared by the FFMA (cell_fwd.cu) and tensor-core (tc_cell.cu) forward kernels
#pragma once
#include "common.cuh"

enum { MODE_P = 0, MODE_V = 1, MODE_TRAIN = 2, MODE_PS = 3 };   // PS: p-call that also saves activations for BPTT

struct FwdK {
  nmarl_fwd_args a;
  // TRAIN-mode extras (all for one time step; pointers already offset to step t)
  const float* Rs; const float* Advs;   // [N][B]
  float* sv_xin; float* sv_sh; float* sv_gates; float* sv_enc; float* sv_dlv;
  float* loss_part;                      // [N][loss_tiles][4]
  int loss_tiles;                        // entries per agent in loss_part (64-row tiles)
  float loss_scale, v_coef, e_coef;
  long long* prof;                       // debug: per-phase clock64 stamps of CTA (0,0) or NULL
};
extern long long* g_nmarl_prof;          // set by nmarl_debug_set_prof

// tensor-core path (tc_cell.cu): returns 0 on success
int nmarl_tc_launch_fwd(const nmarl_model* m, const FwdK& k, int mode, cudaStream_t st);
bool nmarl_tc_fwd_supported(const nmarl_model* m, const nmarl_fwd_args* a);
