// cell_common.cuh -- argument block shared by the FFMA (cell_fwd.cu) and tensor-core (tc_cell.cu) forward kernels
#pragma once
#include "common.cuh"

enum { MODE_P = 0, MODE_V = 1, MODE_PS = 3 };   // PS: p-call that also saves activations (a.sv_*) for BPTT

struct FwdK {
  nmarl_fwd_args a;
  long long* prof;                       // debug: per-phase clock64 stamps of CTA (0,0) or NULL
};
extern long long* g_nmarl_prof;          // set by nmarl_debug_set_prof

// tensor-core path (tc_cell.cu): returns 0 on success
int nmarl_tc_launch_fwd(const nmarl_model* m, const FwdK& k, int mode, cudaStream_t st);
bool nmarl_tc_fwd_supported(const nmarl_model* m, const nmarl_fwd_args* a);
