// Library-level plumbing: error string, launch counter, GEMM dispatch and the ase_gemm entry point.
#include <stdarg.h>
#include <atomic>
#include "common.cuh"
#include "kernels.h"

namespace ase {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

static int check_gemm(const AseGemmParams& p) {
  ASE_CHECK_ARG(p.A && p.B && p.C, "gemm: null operand");
  ASE_CHECK_ARG(p.M > 0 && p.N > 0 && p.K > 0, "gemm: non-positive dimension %d %d %d", p.M, p.N, p.K);
  ASE_CHECK_ARG(p.lda >= (p.a_trans ? p.M : p.K) && p.ldb >= (p.b_trans ? p.N : p.K) && p.ldc >= p.N, "gemm: leading dimension too small");
  ASE_CHECK_ARG(!(p.accumulate && (p.act || (p.mask_src && p.mask_mode))), "gemm: accumulate cannot be combined with act/mask");
  ASE_CHECK_ARG(!(p.accumulate && p.colsum_out), "gemm: colsum_out cannot be combined with accumulate");
  ASE_CHECK_ARG(p.act >= 0 && p.act <= 2 && p.mask_mode >= 0 && p.mask_mode <= 2, "gemm: bad act/mask mode");
  return ASE_OK;
}

int gemm_dispatch(const AseGemmParams& p, cudaStream_t st, PlaneRegistry* reg) {
  int rc = check_gemm(p);
  if (rc) return rc;
  if (p.backend == 1 || p.backend == 2) return gemm_tc(p, st, reg);
  return gemm_simt(p, st);
}

}  // namespace ase

using namespace ase;

extern "C" int ase_abi_version(void) { return ASE_ABI_VERSION; }
extern "C" const char* ase_last_error(void) { return g_err; }
extern "C" uint64_t ase_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

extern "C" int ase_gemm(const AseGemmParams* p, void* stream) {
  ASE_CHECK_ARG(p != nullptr, "ase_gemm: null params");
  return gemm_dispatch(*p, (cudaStream_t)stream);
}

extern "C" int64_t ase_gemm_tc_workspace_bytes(int M, int N, int K) { return gemm_tc_workspace_bytes(M, N, K); }
