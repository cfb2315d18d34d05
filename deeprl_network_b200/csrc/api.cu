// api.cu -- error reporting and ABI self-description for libnmarl.
#include <stdarg.h>
#include <new>
#include "bwd_common.cuh"

static thread_local char g_err[512] = "";

void nmarl_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* nmarl_last_error(void) { return g_err; }
// 101: NMARL_MAX_AGENT 32 -> 128; 102: n_h = 16 / 32 (s_dim); 103: nmarl_eval_record; 104: n_a up to 15 (sv_dlv rows
// are nmarl_head_width(n_a) floats wide); 105: nmarl_a2c_bptt always computes the heads; the bwd_args field and the
// entry point that chose whether it did are gone; 106: nmarl_bwd_args.raw_tiles is gone (sv_dzT / sv_dpT always hold
// one raw tile per 32 rows, half the size), and state_fm must match the layout the path runs; 107: per-env scenario
// parameters (nmarl_cacc_env_par, nmarl_cacc_draw_par, nmarl_cacc_reset_pe / nmarl_cacc_step_pe); 108: envs sharded
// over processes: nmarl_fwd_args.env0 / B_total key the sampling lanes by the global env index, and
// nmarl_cacc_reset_shard / nmarl_cacc_reset_pe_shard / nmarl_cacc_draw_par_shard the env draws
extern "C" int nmarl_version(void) { return 108; }
extern "C" int nmarl_sizeof_model(void) { return (int)sizeof(nmarl_model); }
extern "C" int nmarl_sizeof_agent(void) { return (int)sizeof(nmarl_agent); }
extern "C" int nmarl_sizeof_cacc_cfg(void) { return (int)sizeof(nmarl_cacc_cfg); }
extern "C" int nmarl_sizeof_cacc_env_par(void) { return (int)sizeof(nmarl_cacc_env_par); }
extern "C" int nmarl_sizeof_cacc_par_ranges(void) { return (int)sizeof(nmarl_cacc_par_ranges); }
extern "C" int nmarl_sizeof_fwd_args(void) { return (int)sizeof(nmarl_fwd_args); }
extern "C" int nmarl_sizeof_bwd_args(void) { return (int)sizeof(nmarl_bwd_args); }
extern "C" int64_t nmarl_operand_tile_offset(int rows, int t, int n_agent, int B, int agent, int block) {
  return (int64_t)nmarl_tc_tile_offset(rows, t, n_agent, B / 32, agent, block);
}

bool nmarl_pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("NMARL_NO_PDL");
    on = (e != nullptr && e[0] == '1') ? 0 : 1;
  }
  return on != 0;
}

extern "C" int nmarl_create(nmarl_ctx** out) {
  NMARL_CHECK(out != nullptr, "nmarl_create: out is NULL");
  nmarl_ctx* c = new (std::nothrow) nmarl_ctx();
  NMARL_CHECK(c != nullptr, "nmarl_create: out of host memory");
  c->side = nullptr; c->fork = nullptr; c->join = nullptr; c->heads = nullptr;
  cudaError_t e = cudaGetDevice(&c->device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->join, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->heads, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    nmarl_set_error("nmarl_create: %s", cudaGetErrorString(e));
    nmarl_destroy(c);
    return 2;
  }
  *out = c;
  return 0;
}

extern "C" int nmarl_destroy(nmarl_ctx* c) {
  if (c == nullptr) return 0;
  if (c->fork) cudaEventDestroy(c->fork);
  if (c->join) cudaEventDestroy(c->join);
  if (c->heads) cudaEventDestroy(c->heads);
  if (c->side) cudaStreamDestroy(c->side);
  delete c;
  return 0;
}

// debug hook (not part of the public ABI): device buffer of >= 128 int64 receiving clock64() stamps from
// CTA (0,0) of the tensor-core forward kernel
long long* g_nmarl_prof = nullptr;
extern "C" __attribute__((visibility("default"))) void nmarl_debug_set_prof(long long* p) { g_nmarl_prof = p; }
