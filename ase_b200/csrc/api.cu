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

// The learner's operand-plane registry behind a handle: every call maps onto one PlaneRegistry member or gemm_dispatch, so a
// test drives exactly the path calc_gradients / eval_* take, one GEMM at a time.
struct AseGemmPlanes { PlaneRegistry reg; };

extern "C" int64_t ase_gemm_planes_device_bytes(void) { return PlaneRegistry::device_bytes(); }

extern "C" int ase_gemm_planes_create(int backend, void* device_mem, AseGemmPlanes** out) {
  ASE_CHECK_ARG(out && (backend == 1 || backend == 2), "ase_gemm_planes_create: backend must be 1 or 2");
  ASE_CHECK_ARG(backend == 1 || device_mem, "ase_gemm_planes_create: backend 2 needs device memory");
  AseGemmPlanes* h = new AseGemmPlanes;
  if (backend == 2) {
    if (cudaMemset(device_mem, 0, (size_t)PlaneRegistry::device_bytes()) != cudaSuccess) {
      delete h; set_error("ase_gemm_planes_create: cudaMemset failed"); return ASE_ERR_CUDA;
    }
    h->reg.f16 = true; h->reg.attach_device(device_mem);
  }
  *out = h;
  return ASE_OK;
}

extern "C" void ase_gemm_planes_destroy(AseGemmPlanes* h) { delete h; }

extern "C" int ase_gemm_planes_add(AseGemmPlanes* h, const float* base, int64_t capacity_floats, float* hi, float* lo,
                                   int64_t plane_capacity_floats) {
  ASE_CHECK_ARG(h && base && hi && lo && capacity_floats > 0 && plane_capacity_floats > 0, "ase_gemm_planes_add: bad argument");
  ASE_CHECK_ARG(h->reg.n < PlaneRegistry::MAX, "ase_gemm_planes_add: more than %d buffers", PlaneRegistry::MAX);
  h->reg.add(base, capacity_floats, hi, lo, plane_capacity_floats);
  return ASE_OK;
}

extern "C" int ase_gemm_planes_begin_call(AseGemmPlanes* h, int site_base, void* stream) {
  ASE_CHECK_ARG(h && site_base >= 0 && site_base < PlaneRegistry::SITES, "ase_gemm_planes_begin_call: bad argument");
  return h->reg.begin_call((cudaStream_t)stream, site_base);
}

extern "C" int ase_gemm_planes_forget(AseGemmPlanes* h) {
  ASE_CHECK_ARG(h != nullptr, "ase_gemm_planes_forget: null handle");
  h->reg.forget_sites();
  return ASE_OK;
}

extern "C" int ase_gemm_planes_prep_weights(AseGemmPlanes* h, const float* const* srcs, const int* rows, const int* cols, int count,
                                            void* stream) {
  ASE_CHECK_ARG(h && srcs && rows && cols && count >= 0 && count <= TcPrepBatch::MAX, "ase_gemm_planes_prep_weights: bad argument");
  return h->reg.prep_weights(srcs, rows, cols, count, (cudaStream_t)stream);
}

extern "C" int ase_gemm_planes_gemm(AseGemmPlanes* h, const AseGemmParams* p, void* stream) {
  ASE_CHECK_ARG(h && p, "ase_gemm_planes_gemm: null argument");
  ASE_CHECK_ARG(p->backend == (h->reg.f16 ? 2 : 1), "ase_gemm_planes_gemm: backend %d does not match the registry", p->backend);
  return gemm_dispatch(*p, (cudaStream_t)stream, &h->reg);
}

extern "C" int ase_gemm_planes_info(AseGemmPlanes* h, const float* base, int64_t* out, float* scale_dst, void* stream) {
  ASE_CHECK_ARG(h && base && out, "ase_gemm_planes_info: null argument");
  const PlaneBuf* x = h->reg.find(base);
  ASE_CHECK_ARG(x && x->base == base, "ase_gemm_planes_info: %p is not the base of a registered buffer", (const void*)base);
  out[0] = x->valid; out[1] = x->fp32_stale; out[2] = x->rows; out[3] = x->cols; out[4] = x->ld; out[5] = x->ldp;
  if (scale_dst && h->reg.f16 && x->valid && x->scale_ptr)
    ASE_CUDA_OK(cudaMemcpyAsync(scale_dst, x->scale_ptr, 2 * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return ASE_OK;
}

extern "C" int ase_gemm_planes_status(AseGemmPlanes* h, int* flags, void* stream) {
  ASE_CHECK_ARG(h && flags, "ase_gemm_planes_status: null argument");
  *flags = 0;
  if (!h->reg.f16) return ASE_OK;
  unsigned f = 0;
  ASE_CUDA_OK(cudaMemcpyAsync(&f, h->reg.flag, sizeof(f), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  ASE_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  *flags = (int)f;
  return ASE_OK;
}

extern "C" int ase_gemm_planes_clear(AseGemmPlanes* h, void* stream) {
  ASE_CHECK_ARG(h != nullptr, "ase_gemm_planes_clear: null handle");
  if (h->reg.f16) ASE_CUDA_OK(cudaMemsetAsync(h->reg.flag, 0, sizeof(unsigned), (cudaStream_t)stream));
  return ASE_OK;
}
