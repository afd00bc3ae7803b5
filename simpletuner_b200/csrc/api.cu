// simpletuner_b200 — C-ABI entry points (include/stb200.h): argument checking, TMA tensor-map
// construction and kernel launches.  No torch types here; the Python host passes raw pointers.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>

#include <climits>
#include "../../include/stb200.h"
#include "attn_bwd.cuh"
#include "attn_fwd.cuh"
#include "optim.cuh"
#include "elementwise.cuh"
#include "gemm.cuh"
#include "wgrad_full.cuh"
#include "lokr.cuh"
#include "vae.cuh"
#include "wgrad.cuh"

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define STB_CUDA(expr)                                                                       \
  do {                                                                                       \
    cudaError_t e_ = (expr);                                                                 \
    if (e_ != cudaSuccess) return fail(STB_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

#define STB_LAUNCH_CHECK(name)                                                                  \
  do {                                                                                          \
    cudaError_t e_ = cudaGetLastError();                                                        \
    if (e_ != cudaSuccess) return fail(STB_ERR_CUDA, "launch %s: %s", name, cudaGetErrorString(e_)); \
    g_launches.fetch_add(1, std::memory_order_relaxed);                                         \
  } while (0)

// ---------------------------------------------------------------- device / driver helpers
int num_sms() {
  static int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return v;
  }();
  return n;
}

int check_device() {
  static int ok = [] {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
    int minor = 0;
    if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
    return major == 9 && minor == 0 ? 1 : 0;
  }();
  if (!ok) return fail(STB_ERR_UNSUPPORTED, "libstb200 needs an sm_90 (H100) device; there is no CPU or other-arch fallback");
  return 0;
}

PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

struct MapKey {
  const void* ptr;
  int rank;
  unsigned long long dims[4];
  unsigned long long strides[3];
  unsigned box[4];
  bool operator==(const MapKey& o) const { return std::memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    const unsigned char* p = reinterpret_cast<const unsigned char*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(MapKey); ++i) h = (h ^ p[i]) * 1099511628211ull;
    return h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// bf16 tensor map, SWIZZLE_128B, dims/strides innermost-first (strides in BYTES for dims 1..rank-1)
int make_map(CUtensorMap* out, const void* ptr, int rank, const unsigned long long* dims,
             const unsigned long long* strides_bytes, const unsigned* box) {
  MapKey key;
  std::memset(&key, 0, sizeof key);
  key.ptr = ptr;
  key.rank = rank;
  for (int i = 0; i < rank; ++i) key.dims[i] = dims[i], key.box[i] = box[i];
  for (int i = 0; i + 1 < rank; ++i) key.strides[i] = strides_bytes[i];
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) {
      *out = it->second;
      return 0;
    }
  }
  auto fn = encode_fn();
  if (!fn) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if (reinterpret_cast<uintptr_t>(ptr) & 15) return fail(STB_ERR_ARG, "tensor base pointer must be 16-byte aligned");
  for (int i = 0; i + 1 < rank; ++i)
    if (strides_bytes[i] & 15) return fail(STB_ERR_ARG, "tensor stride %d (%llu bytes) must be a multiple of 16 bytes", i, strides_bytes[i]);
  cuuint64_t gdim[4];
  cuuint64_t gstr[3];
  cuuint32_t bx[4], es[4];
  for (int i = 0; i < rank; ++i) gdim[i] = dims[i], bx[i] = box[i], es[i] = 1;
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", int(r));
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    if (g_maps.size() > 65536) g_maps.clear();
    g_maps.emplace(key, *out);
  }
  return 0;
}

// fp32 map without swizzle (dq accumulator reduce-add)
int make_map_f32(CUtensorMap* out, const void* ptr, int rank, const unsigned long long* dims,
                 const unsigned long long* strides_bytes, const unsigned* box) {
  auto fn = encode_fn();
  if (!fn) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[4];
  cuuint64_t gstr[3];
  cuuint32_t bx[4], es[4];
  for (int i = 0; i < rank; ++i) gdim[i] = dims[i], bx[i] = box[i], es[i] = 1;
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled(f32) failed with CUresult %d", int(r));
  return 0;
}

// bf16 SWIZZLE_128B map with per-dimension traversal strides (strided conv windows); not cached
int make_map_strided(CUtensorMap* out, const void* ptr, int rank, const unsigned long long* dims,
                     const unsigned long long* strides_bytes, const unsigned* box, const unsigned* estrides) {
  auto fn = encode_fn();
  if (!fn) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if (reinterpret_cast<uintptr_t>(ptr) & 15) return fail(STB_ERR_ARG, "tensor base pointer must be 16-byte aligned");
  cuuint64_t gdim[4];
  cuuint64_t gstr[3];
  cuuint32_t bx[4], es[4];
  for (int i = 0; i < rank; ++i) gdim[i] = dims[i], bx[i] = box[i], es[i] = estrides[i];
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled(strided) failed with CUresult %d", int(r));
  return 0;
}

template <typename K>
int set_smem(K kernel, int bytes) {
  STB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return 0;
}

// ---------------------------------------------------------------- GEMM
template <int BN>
int launch_gemm(const stb_gemm_args* a, cudaStream_t st) {
  using Cfg = stb::GemmCfg<BN>;
  stb::GemmMaps maps;
  std::memset(&maps, 0, sizeof maps);
  stb::GemmParams p;
  std::memset(&p, 0, sizeof p);
  for (int s = 0; s < a->nseg; ++s) {
    const stb_gemm_seg& g = a->seg[s];
    if (g.K <= 0 || (g.K & 7)) return fail(STB_ERR_ARG, "segment %d: K=%d must be a positive multiple of 8", s, g.K);
    unsigned long long ad[3] = {(unsigned long long)g.K, (unsigned long long)a->rows_per_batch,
                                (unsigned long long)a->num_batches};
    unsigned long long as[2] = {(unsigned long long)g.a_row_stride * 2ull, (unsigned long long)g.a_batch_stride * 2ull};
    if (a->num_batches == 1) as[1] = as[0] * (unsigned long long)a->rows_per_batch;
    unsigned ab[3] = {64, 128, 1};
    if (int r = make_map(&maps.a[s], g.a, 3, ad, as, ab)) return r;
    if (g.w_kn) {   // [K, N] row-major: contraction index = row; staged as 64 x 64 MN-major boxes
      unsigned long long wd[2] = {(unsigned long long)a->N, (unsigned long long)g.K};
      unsigned long long ws[1] = {(unsigned long long)g.w_row_stride * 2ull};
      unsigned wb[2] = {64, 64};
      if (int r = make_map(&maps.w[s], g.w, 2, wd, ws, wb)) return r;
    } else {
      unsigned long long wd[2] = {(unsigned long long)g.K, (unsigned long long)a->N};
      unsigned long long ws[1] = {(unsigned long long)g.w_row_stride * 2ull};
      unsigned wb[2] = {64, (unsigned)BN};
      if (int r = make_map(&maps.w[s], g.w, 2, wd, ws, wb)) return r;
    }
    p.w_kn[s] = g.w_kn ? 1 : 0;
    p.kblocks[s] = (g.K + 63) / 64;
  }
  p.rows_per_batch = a->rows_per_batch;
  p.num_batches = a->num_batches;
  p.N = a->N;
  p.nseg = a->nseg;
  p.epi = a->epi;
  p.nan_to_num = a->nan_to_num;
  p.D = static_cast<__nv_bfloat16*>(a->d);
  p.d_batch_stride = a->d_batch_stride;
  p.d_row_stride = a->d_row_stride;
  p.bias = static_cast<const __nv_bfloat16*>(a->bias);
  p.gate = static_cast<const __nv_bfloat16*>(a->gate);
  p.gate_batch_stride = a->gate_batch_stride;
  p.res = static_cast<const __nv_bfloat16*>(a->res);
  p.res_batch_stride = a->res_batch_stride;
  p.res_row_stride = a->res_row_stride;
  p.aux = static_cast<__nv_bfloat16*>(a->aux);
  p.aux_batch_stride = a->aux_batch_stride;
  p.aux_row_stride = a->aux_row_stride;

  auto kernel = stb::gemm_bf16_tn_kernel<BN, false>;
  static bool configured = false;
  if (!configured) {
    if (int r = set_smem(kernel, Cfg::SMEM_BYTES)) return r;
    configured = true;
  }
  const long long tiles = (long long)((a->rows_per_batch + Cfg::BM - 1) / Cfg::BM) * a->num_batches * ((a->N + BN - 1) / BN);
  const int grid = (int)std::min<long long>(tiles, num_sms());
  kernel<<<grid, 384, Cfg::SMEM_BYTES, st>>>(maps, p);
  STB_LAUNCH_CHECK("gemm_bf16_tn");
  return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

template <int HD>
static int launch_attn_bwd(const stb_attn_bwd_args* a, const stb::AttnBwdMaps& maps, const stb::AttnBwdParams& p,
                           cudaStream_t st) {
  {
    const long long warps = (long long)a->B * a->Sq * a->H;
    stb::attn_bwd_delta_kernel<HD><<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(a->o), a->o_b, a->o_s, a->o_h,
        static_cast<const __nv_bfloat16*>(a->d_o), a->do_b, a->do_s, a->do_h, a->delta, a->B, a->H, a->Sq);
    STB_LAUNCH_CHECK("attn_bwd_delta");
  }
  constexpr int SMEM = stb::AttnBwdCfg<HD>::SMEM_BYTES;
  auto k1 = stb::attn_bwd_dkdv_kernel<HD>;
  auto k2 = stb::attn_bwd_dq_kernel<HD>;
  static bool configured = false;
  if (!configured) {
    if (int r = set_smem(k1, SMEM)) return r;
    if (int r = set_smem(k2, SMEM)) return r;
    configured = true;
  }
  k1<<<dim3((a->Sk + 127) / 128, a->H, a->B), 384, SMEM, st>>>(maps, p);
  STB_LAUNCH_CHECK("attn_bwd_dkdv");
  k2<<<dim3((a->Sq + 127) / 128, a->H, a->B), 384, SMEM, st>>>(maps, p);
  STB_LAUNCH_CHECK("attn_bwd_dq");
  return 0;
}

extern "C" {

const char* stb_last_error(void) { return g_err.c_str(); }
int stb_version(void) { return 100; }
long long stb_launch_count(void) { return g_launches.load(); }
void stb_reset_launch_count(void) { g_launches.store(0); }

int stb_gemm_bf16(const stb_gemm_args* a, void* stream) {
  if (int r = check_device()) return r;
  if (!a || a->nseg < 1 || a->nseg > 3) return fail(STB_ERR_ARG, "nseg must be 1..3");
  if (a->num_batches < 1 || a->rows_per_batch < 1 || a->N < 1) return fail(STB_ERR_ARG, "empty problem");
  if (!aligned16(a->d) || (a->d_row_stride & 7) || (a->d_batch_stride & 7))
    return fail(STB_ERR_ARG, "D must be 16-byte aligned with strides multiple of 8 elements");
  if (a->bias && !aligned16(a->bias)) return fail(STB_ERR_ARG, "bias must be 16-byte aligned");
  if (a->epi == STB_EPI_GATE_RES && (!a->gate || !a->res)) return fail(STB_ERR_ARG, "GATE_RES needs gate and res");
  if (a->epi == STB_EPI_GATE_RES && (!aligned16(a->gate) || (a->gate_batch_stride & 7)))
    return fail(STB_ERR_ARG, "gate must be 16-byte aligned");
  if ((a->epi == STB_EPI_GATE_RES || a->epi == STB_EPI_ADD_RES) &&
      (!a->res || !aligned16(a->res) || (a->res_row_stride & 7) || (a->res_batch_stride & 7)))
    return fail(STB_ERR_ARG, "res must be given, 16-byte aligned, strides multiple of 8");
  if ((a->epi == STB_EPI_MUL_DGELU || a->epi == STB_EPI_MUL) && !a->aux) return fail(STB_ERR_ARG, "MUL_DGELU / MUL need aux");
  if (a->aux && (!aligned16(a->aux) || (a->aux_row_stride & 7) || (a->aux_batch_stride & 7)))
    return fail(STB_ERR_ARG, "aux must be 16-byte aligned, strides multiple of 8");
  if (a->epi < 0 || a->epi > 6) return fail(STB_ERR_ARG, "unknown epilogue %d", a->epi);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // every sm_90a tile is 128 rows (two 64-row consumer warpgroups); the row-tile request tile_mt is accepted and ignored
  if (a->tile_mt < 0 || a->tile_mt > 3) return fail(STB_ERR_ARG, "unsupported tile config MT=%d", a->tile_mt);
  int bn = a->tile_bn;
  if (bn == 0) {
    bn = a->N > 128 ? 256 : (a->N > 64 ? 128 : 64);
    // skinny-M problems (conditioning / modulation GEMMs, M = batch) and short grids: spread the weight stream over
    // more SMs with narrower tiles while 256-wide tiles would leave SMs idle
    const long long t256 = (long long)((a->rows_per_batch + 127) / 128) * a->num_batches * ((a->N + 255) / 256);
    if (bn == 256 && t256 < num_sms()) bn = 128;
  }
  if (bn == 256) return launch_gemm<256>(a, st);
  if (bn == 128) return launch_gemm<128>(a, st);
  if (bn == 64) return launch_gemm<64>(a, st);
  return fail(STB_ERR_ARG, "unsupported tile config BN=%d", bn);
}

int stb_attn_fwd(const stb_attn_fwd_args* a, void* stream) {
  if (int r = check_device()) return r;
  if (!a || a->B < 1 || a->H < 1 || a->Sq < 1 || a->Sk < 1) return fail(STB_ERR_ARG, "empty attention problem");
  if (a->HD != 128 && a->HD != 64) return fail(STB_ERR_UNSUPPORTED, "head_dim %d not supported (64 or 128)", a->HD);
  if (!aligned16(a->o) || (a->o_s & 7) || (a->o_h & 7) || (a->o_b & 7)) return fail(STB_ERR_ARG, "O alignment");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  stb::AttnFwdMaps maps;
  auto mk = [&](CUtensorMap* m, const void* ptr, long long sb, long long ss, long long sh, int S) {
    unsigned long long d[4] = {(unsigned long long)a->HD, (unsigned long long)a->H, (unsigned long long)S,
                               (unsigned long long)a->B};
    unsigned long long s[3] = {(unsigned long long)sh * 2ull, (unsigned long long)ss * 2ull, (unsigned long long)sb * 2ull};
    unsigned bx[4] = {64, 1, 128, 1};
    return make_map(m, ptr, 4, d, s, bx);
  };
  if (int r = mk(&maps.q, a->q, a->q_b, a->q_s, a->q_h, a->Sq)) return r;
  if (int r = mk(&maps.k, a->k, a->k_b, a->k_s, a->k_h, a->Sk)) return r;
  if (int r = mk(&maps.v, a->v, a->v_b, a->v_s, a->v_h, a->Sk)) return r;
  stb::AttnFwdParams p;
  p.B = a->B; p.H = a->H; p.Sq = a->Sq; p.Sk = a->Sk;
  p.scale = a->scale;
  p.O = static_cast<__nv_bfloat16*>(a->o);
  p.o_b = a->o_b; p.o_s = a->o_s; p.o_h = a->o_h;
  p.lse = a->lse;
  p.bias = static_cast<const __nv_bfloat16*>(a->bias);
  p.bias_h = a->bias_h; p.bias_q = a->bias_q;
  p.inv_scale = a->scale != 0.f ? 1.f / a->scale : 0.f;
  dim3 grid((a->Sq + 127) / 128, a->H, a->B);
  if (a->bias) {   // text-encoder instantiation (additive bias / mask); never taken by the training step
    if (a->scale == 0.f || a->bias_q < a->Sk) return fail(STB_ERR_ARG, "attn_fwd bias: scale must be non-zero and bias_q >= Sk");
    if (a->HD == 128) {
      auto kernel = stb::attn_fwd_kernel<128, true>;
      static bool configured = false;
      if (!configured) {
        if (int r = set_smem(kernel, stb::AttnFwdCfg<128>::SMEM_BYTES)) return r;
        configured = true;
      }
      kernel<<<grid, 384, stb::AttnFwdCfg<128>::SMEM_BYTES, st>>>(maps, p);
    } else {
      auto kernel = stb::attn_fwd_kernel<64, true>;
      static bool configured = false;
      if (!configured) {
        if (int r = set_smem(kernel, stb::AttnFwdCfg<64>::SMEM_BYTES)) return r;
        configured = true;
      }
      kernel<<<grid, 384, stb::AttnFwdCfg<64>::SMEM_BYTES, st>>>(maps, p);
    }
    STB_LAUNCH_CHECK("attn_fwd_bias");
    return 0;
  }
  if (a->HD == 128) {
    auto kernel = stb::attn_fwd_kernel<128, false>;
    static bool configured = false;
    if (!configured) {
      if (int r = set_smem(kernel, stb::AttnFwdCfg<128>::SMEM_BYTES)) return r;
      configured = true;
    }
    kernel<<<grid, 384, stb::AttnFwdCfg<128>::SMEM_BYTES, st>>>(maps, p);
  } else {
    auto kernel = stb::attn_fwd_kernel<64, false>;
    static bool configured = false;
    if (!configured) {
      if (int r = set_smem(kernel, stb::AttnFwdCfg<64>::SMEM_BYTES)) return r;
      configured = true;
    }
    kernel<<<grid, 384, stb::AttnFwdCfg<64>::SMEM_BYTES, st>>>(maps, p);
  }
  STB_LAUNCH_CHECK("attn_fwd");
  return 0;
}

int stb_attn_bwd(const stb_attn_bwd_args* a, void* stream) {
  if (int r = check_device()) return r;
  if (!a || a->B < 1 || a->H < 1 || a->Sq < 1 || a->Sk < 1) return fail(STB_ERR_ARG, "empty attention problem");
  if (a->HD != 128 && a->HD != 64) return fail(STB_ERR_UNSUPPORTED, "head_dim %d not supported (64 or 128)", a->HD);
  if (!a->lse || !a->delta) return fail(STB_ERR_ARG, "attn_bwd needs lse and a delta scratch buffer");
  auto al = [&](const void* ptr, long long sb, long long ss, long long sh) {
    return aligned16(ptr) && !(sb & 7) && !(ss & 7) && !(sh & 7);
  };
  if (!al(a->dq, a->dq_b, a->dq_s, a->dq_h) || !al(a->dk, a->dk_b, a->dk_s, a->dk_h) ||
      !al(a->dv, a->dv_b, a->dv_s, a->dv_h))
    return fail(STB_ERR_ARG, "dq/dk/dv must be 16-byte aligned with strides multiple of 8 elements");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  stb::AttnBwdMaps maps;
  auto mk = [&](CUtensorMap* m, const void* ptr, long long sb, long long ss, long long sh, int S, unsigned rows) {
    unsigned long long d[4] = {(unsigned long long)a->HD, (unsigned long long)a->H, (unsigned long long)S,
                               (unsigned long long)a->B};
    unsigned long long s[3] = {(unsigned long long)sh * 2ull, (unsigned long long)ss * 2ull, (unsigned long long)sb * 2ull};
    unsigned bx[4] = {64, 1, rows, 1};
    return make_map(m, ptr, 4, d, s, bx);
  };
  if (int r = mk(&maps.q128, a->q, a->q_b, a->q_s, a->q_h, a->Sq, 128)) return r;
  if (int r = mk(&maps.k128, a->k, a->k_b, a->k_s, a->k_h, a->Sk, 128)) return r;
  if (int r = mk(&maps.v128, a->v, a->v_b, a->v_s, a->v_h, a->Sk, 128)) return r;
  if (int r = mk(&maps.do128, a->d_o, a->do_b, a->do_s, a->do_h, a->Sq, 128)) return r;
  if (int r = mk(&maps.q64, a->q, a->q_b, a->q_s, a->q_h, a->Sq, 64)) return r;
  if (int r = mk(&maps.k64, a->k, a->k_b, a->k_s, a->k_h, a->Sk, 64)) return r;
  if (int r = mk(&maps.v64, a->v, a->v_b, a->v_s, a->v_h, a->Sk, 64)) return r;
  if (int r = mk(&maps.do64, a->d_o, a->do_b, a->do_s, a->do_h, a->Sq, 64)) return r;
  stb::AttnBwdParams p;
  p.B = a->B; p.H = a->H; p.Sq = a->Sq; p.Sk = a->Sk;
  p.scale = a->scale;
  p.lse = a->lse;
  p.delta = a->delta;
  p.dq = static_cast<__nv_bfloat16*>(a->dq);
  p.dk = static_cast<__nv_bfloat16*>(a->dk);
  p.dv = static_cast<__nv_bfloat16*>(a->dv);
  p.dq_b = a->dq_b; p.dq_s = a->dq_s; p.dq_h = a->dq_h;
  p.dk_b = a->dk_b; p.dk_s = a->dk_s; p.dk_h = a->dk_h;
  p.dv_b = a->dv_b; p.dv_s = a->dv_s; p.dv_h = a->dv_h;
  p.fuse_prep = 0;
  if (const stb_qk_prep* f = a->qk_prep) {
    if (a->Sq != a->Sk) return fail(STB_ERR_ARG, "qk_prep fusion needs self-attention (Sq == Sk)");
    if (!f->src || !aligned16(f->src) || (f->src_b & 7) || (f->src_s & 7) || (f->k_off & 7))
      return fail(STB_ERR_ARG, "qk_prep.src must be 16-byte aligned with strides / k_off multiple of 8 elements");
    if ((f->cos_t == nullptr) != (f->sin_t == nullptr)) return fail(STB_ERR_ARG, "qk_prep: give both cos_t and sin_t or neither");
    p.fuse_prep = 1;
    p.src = static_cast<const __nv_bfloat16*>(f->src);
    p.src_b = f->src_b; p.src_s = f->src_s; p.k_off = f->k_off;
    p.wq0 = static_cast<const __nv_bfloat16*>(f->wq); p.wk0 = static_cast<const __nv_bfloat16*>(f->wk);
    p.wq1 = static_cast<const __nv_bfloat16*>(f->wq_added); p.wk1 = static_cast<const __nv_bfloat16*>(f->wk_added);
    p.s_split = f->s_split;
    p.cosT = f->cos_t; p.sinT = f->sin_t;
    p.eps = f->eps;
  }
  p.q = static_cast<const __nv_bfloat16*>(a->q);
  p.d_o = static_cast<const __nv_bfloat16*>(a->d_o);
  p.q_b = a->q_b; p.q_s = a->q_s; p.q_h = a->q_h;
  p.do_b = a->do_b; p.do_s = a->do_s; p.do_h = a->do_h;
  if (a->HD == 128) return launch_attn_bwd<128>(a, maps, p, st);
  return launch_attn_bwd<64>(a, maps, p, st);
}

int stb_ln_modulate_fwd(const void* x, long long x_b, long long x_s, const void* shift, const void* scale,
                        long long mod_b, void* out, long long o_b, long long o_s, int B, int S, int D,
                        float eps, void* stream) {
  if (int r = check_device()) return r;
  if ((D & 7) || D > 8192) return fail(STB_ERR_ARG, "D=%d must be a multiple of 8 and <= 8192", D);
  if (!aligned16(x) || !aligned16(out) || !aligned16(shift) || !aligned16(scale) || (x_s & 7) || (x_b & 7) ||
      (o_s & 7) || (o_b & 7) || (mod_b & 7))
    return fail(STB_ERR_ARG, "ln_modulate_fwd alignment");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rows = B * S;
  const int vpt = (D + 1023) / 1024;
  auto X = static_cast<const __nv_bfloat16*>(x);
  auto SH = static_cast<const __nv_bfloat16*>(shift);
  auto SC = static_cast<const __nv_bfloat16*>(scale);
  auto O = static_cast<__nv_bfloat16*>(out);
#define STB_LN_F(V) stb::ln_modulate_fwd_kernel<V><<<rows, 128, 0, st>>>(X, x_b, x_s, SH, SC, mod_b, O, o_b, o_s, S, D, eps)
  switch (vpt) {
    case 1: STB_LN_F(1); break;
    case 2: STB_LN_F(2); break;
    case 3: STB_LN_F(3); break;
    case 4: STB_LN_F(4); break;
    default: STB_LN_F(8); break;
  }
#undef STB_LN_F
  STB_LAUNCH_CHECK("ln_modulate_fwd");
  return 0;
}

int stb_ln_modulate_bwd(const void* dy, long long dy_b, long long dy_s, const void* x, long long x_b,
                        long long x_s, const void* scale, long long mod_b, const void* add, long long add_b,
                        long long add_s, void* dx, long long dx_b, long long dx_s, int B, int S, int D,
                        float eps, void* stream) {
  if (int r = check_device()) return r;
  if ((D & 7) || D > 4096) return fail(STB_ERR_ARG, "D=%d must be a multiple of 8 and <= 4096", D);
  if (!aligned16(x) || !aligned16(dy) || !aligned16(dx) || !aligned16(scale) || (add && !aligned16(add)))
    return fail(STB_ERR_ARG, "ln_modulate_bwd alignment");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rows = B * S;
  const int vpt = (D + 1023) / 1024;
  auto DY = static_cast<const __nv_bfloat16*>(dy);
  auto X = static_cast<const __nv_bfloat16*>(x);
  auto SC = static_cast<const __nv_bfloat16*>(scale);
  auto AD = static_cast<const __nv_bfloat16*>(add);
  auto DX = static_cast<__nv_bfloat16*>(dx);
#define STB_LN_B(V) \
  stb::ln_modulate_bwd_kernel<V><<<rows, 128, 0, st>>>(DY, dy_b, dy_s, X, x_b, x_s, SC, mod_b, AD, add_b, add_s, DX, dx_b, dx_s, S, D, eps)
  switch (vpt) {
    case 1: STB_LN_B(1); break;
    case 2: STB_LN_B(2); break;
    case 3: STB_LN_B(3); break;
    default: STB_LN_B(4); break;
  }
#undef STB_LN_B
  STB_LAUNCH_CHECK("ln_modulate_bwd");
  return 0;
}

int stb_qk_rmsnorm_rope_fwd(const void* src, long long src_b, long long src_s, int k_off, const void* wq,
                            const void* wk, const void* wq_added, const void* wk_added, int s_split,
                            const float* cos_t, const float* sin_t, void* q_out, void* k_out,
                            long long dst_b, long long dst_s, int B, int S, int H, int HD, float eps,
                            void* stream) {
  if (int r = check_device()) return r;
  if (HD != 128 && HD != 64) return fail(STB_ERR_UNSUPPORTED, "head_dim %d not supported", HD);
  if ((src_s & 3) || (src_b & 3) || (k_off & 3) || (dst_s & 3) || (dst_b & 3)) return fail(STB_ERR_ARG, "qk_rmsnorm_rope alignment");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long warps = (long long)B * S;  // one warp per token
  const unsigned grid = (unsigned)((warps + 7) / 8);
  auto SRC = static_cast<const __nv_bfloat16*>(src);
  auto cast = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
  if (HD == 128)
    stb::qk_rmsnorm_rope_fwd_kernel<128><<<grid, 256, 0, st>>>(SRC, src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t, static_cast<__nv_bfloat16*>(q_out), static_cast<__nv_bfloat16*>(k_out), dst_b, dst_s, B, S, H, eps);
  else
    stb::qk_rmsnorm_rope_fwd_kernel<64><<<grid, 256, 0, st>>>(SRC, src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t, static_cast<__nv_bfloat16*>(q_out), static_cast<__nv_bfloat16*>(k_out), dst_b, dst_s, B, S, H, eps);
  STB_LAUNCH_CHECK("qk_rmsnorm_rope_fwd");
  return 0;
}

int stb_qk_rmsnorm_rope_bwd(const void* dq, const void* dk, long long d_b, long long d_s, const void* src,
                            long long src_b, long long src_s, int k_off, const void* wq, const void* wk,
                            const void* wq_added, const void* wk_added, int s_split, const float* cos_t,
                            const float* sin_t, void* dsrc, long long ds_b, long long ds_s, int B, int S,
                            int H, int HD, float eps, float* dw, void* stream) {
  if (int r = check_device()) return r;
  if (HD != 128 && HD != 64) return fail(STB_ERR_UNSUPPORTED, "head_dim %d not supported", HD);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long warps = (long long)B * S;  // one warp per token
  const unsigned grid = (unsigned)((warps + 7) / 8);
  auto cast = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
  if (HD == 128) {
    if (dw) stb::qk_rmsnorm_rope_bwd_kernel<128, true><<<grid, 256, 0, st>>>(cast(dq), cast(dk), d_b, d_s, cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t, static_cast<__nv_bfloat16*>(dsrc), ds_b, ds_s, B, S, H, eps, dw);
    else {
      static const bool loop_kernel = [] { const char* e = std::getenv("STB_ROPE_BWD_LOOP"); return e && e[0] == '1'; }();
      const bool flat_ok = aligned16(dq) && aligned16(dk) && aligned16(src) && aligned16(dsrc) && !(d_b & 7) && !(d_s & 7) && !(src_s & 7) &&
                           !(src_b & 7) && !(k_off & 7) && !(ds_s & 7) && !(ds_b & 7) && (!cos_t || (aligned16(cos_t) && aligned16(sin_t))) &&
                           (!wq || aligned16(wq)) && (!wk || aligned16(wk)) && (!wq_added || aligned16(wq_added)) && (!wk_added || aligned16(wk_added));
      if (flat_ok && !loop_kernel) {   // one 16-byte chunk per thread: 4.0 TB/s vs 2.7 for the warp-per-token loop
        const long long threads = (long long)B * S * 2 * H * 16;
        stb::qk_rmsnorm_rope_flat128_kernel<true><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(
            cast(dq), cast(dk), d_b, d_s, cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split,
            cos_t, sin_t, static_cast<__nv_bfloat16*>(dsrc), nullptr, ds_b, ds_s, B, S, H, eps);
      } else {
        stb::qk_rmsnorm_rope_bwd_kernel<128, false><<<grid, 256, 0, st>>>(cast(dq), cast(dk), d_b, d_s, cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t, static_cast<__nv_bfloat16*>(dsrc), ds_b, ds_s, B, S, H, eps, dw);
      }
    }
  } else {
    if (dw) stb::qk_rmsnorm_rope_bwd_kernel<64, true><<<grid, 256, 0, st>>>(cast(dq), cast(dk), d_b, d_s, cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t, static_cast<__nv_bfloat16*>(dsrc), ds_b, ds_s, B, S, H, eps, dw);
    else stb::qk_rmsnorm_rope_bwd_kernel<64, false><<<grid, 256, 0, st>>>(cast(dq), cast(dk), d_b, d_s, cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t, static_cast<__nv_bfloat16*>(dsrc), ds_b, ds_s, B, S, H, eps, dw);
  }
  STB_LAUNCH_CHECK("qk_rmsnorm_rope_bwd");
  return 0;
}

int stb_flow_prep_pack(const void* latents, const void* noise, const float* sigmas, void* noisy,
                       void* packed, int B, int C, int Hh, int Ww, void* stream) {
  if (int r = check_device()) return r;
  if ((Hh & 1) || (Ww & 1)) return fail(STB_ERR_ARG, "latent H and W must be even for 2x2 patchify");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = (long long)B * C * Hh * Ww;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)num_sms() * 16);
  stb::flow_prep_pack_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(latents), static_cast<const __nv_bfloat16*>(noise), sigmas, static_cast<__nv_bfloat16*>(noisy), static_cast<__nv_bfloat16*>(packed), B, C, Hh, Ww);
  STB_LAUNCH_CHECK("flow_prep_pack");
  return 0;
}

// the loss kernels run as one fixed cluster (deterministic reduction, elementwise.cuh loss_cluster_store)
static void loss_cluster_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute (&attr)[1], cudaStream_t st) {
  std::memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(stb::LOSS_CTAS);
  cfg.blockDim = dim3(stb::LOSS_THREADS);
  cfg.stream = st;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = stb::LOSS_CTAS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
}

static int check_loss_type(int loss_type, const float* huber_c) {
  if (loss_type < 0 || loss_type > 2) return fail(STB_ERR_ARG, "loss_type must be 0 (l2), 1 (huber) or 2 (smooth_l1)");
  if (loss_type != 0 && !huber_c) return fail(STB_ERR_ARG, "huber / smooth_l1 need the per-sample huber_c array");
  return 0;
}

int stb_flow_mse_loss(const void* pred_packed, const void* latents, const void* noise, float* loss_out,
                      void* dpred_packed, float grad_scale, int B, int C, int Hh, int Ww, int layout, int loss_type,
                      const float* huber_c, void* stream) {
  if (int r = check_device()) return r;
  if (int r = check_loss_type(loss_type, huber_c)) return r;
  if (layout < 0 || layout > 2) return fail(STB_ERR_ARG, "flow_mse_loss layout must be 0 (Flux), 1 (SD3) or 2 (NCHW)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  loss_cluster_config(cfg, attr, st);
  STB_CUDA(cudaLaunchKernelEx(&cfg, stb::flow_mse_loss_kernel, static_cast<const __nv_bfloat16*>(pred_packed), static_cast<const __nv_bfloat16*>(latents),
                              static_cast<const __nv_bfloat16*>(noise), loss_out, static_cast<__nv_bfloat16*>(dpred_packed), grad_scale, B, C, Hh,
                              Ww, layout, loss_type, huber_c));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

int stb_ddpm_prep_pack(const void* latents, const void* noise, const float* coef_a, const float* coef_b, void* noisy,
                       void* packed, int B, int C, int Hh, int Ww, void* stream) {
  if (int r = check_device()) return r;
  if (packed && ((Hh & 1) || (Ww & 1))) return fail(STB_ERR_ARG, "latent H and W must be even for 2x2 patchify");
  if (!noisy && !packed) return fail(STB_ERR_ARG, "ddpm_prep_pack: no output requested");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = (long long)B * C * Hh * Ww;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)num_sms() * 16);
  stb::ddpm_prep_pack_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(latents), static_cast<const __nv_bfloat16*>(noise), coef_a, coef_b, static_cast<__nv_bfloat16*>(noisy), static_cast<__nv_bfloat16*>(packed), B, C, Hh, Ww);
  STB_LAUNCH_CHECK("ddpm_prep_pack");
  return 0;
}

int stb_target_mse_loss(const void* pred_packed, const void* target, const float* weights, float* loss_out,
                        void* dpred_packed, float grad_scale, int B, int C, int Hh, int Ww, int layout, int loss_type,
                        const float* huber_c, void* stream) {
  if (int r = check_device()) return r;
  if (int r = check_loss_type(loss_type, huber_c)) return r;
  if (layout < 0 || layout > 2) return fail(STB_ERR_ARG, "target_mse_loss layout must be 0 (c,dy,dx), 1 (dy,dx,c) or 2 (NCHW)");
  if (layout != 2 && ((Hh & 1) || (Ww & 1))) return fail(STB_ERR_ARG, "latent H and W must be even for 2x2 patchify");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  loss_cluster_config(cfg, attr, st);
  STB_CUDA(cudaLaunchKernelEx(&cfg, stb::target_mse_loss_kernel, static_cast<const __nv_bfloat16*>(pred_packed), static_cast<const __nv_bfloat16*>(target),
                              weights, loss_out, static_cast<__nv_bfloat16*>(dpred_packed), grad_scale, B, C, Hh, Ww, layout, loss_type, huber_c));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

int stb_adamw_bf16_multi(const long long* ptrs, const long long* sizes, const float* decay, const int* blk_tensor,
                         const long long* blk_off, int num_blocks, int T, double beta1, double beta2, double step, double lr,
                         double eps, const int* rnd, const long long* rnd_off, long long rnd_plane, unsigned long long seed,
                         double grad_clamp, const long long* ema_shadow, double ema_one_minus_decay, void* stream) {
  if (int r = check_device()) return r;
  if (!ptrs || !sizes || !decay || !blk_tensor || !blk_off || num_blocks < 1 || T < 1) return fail(STB_ERR_ARG, "adamw_bf16_multi: bad tables");
  if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0) || eps < 0.0) return fail(STB_ERR_ARG, "adamw_bf16_multi: bad hyper-parameters");
  // hyper-parameters arrive as the reference's Python floats (doubles): `1 - beta` and `-lr * (1 - beta2 ** step) ** 0.5`
  // are formed in double there and only then become the fp32 scalars of the eager kernels
  const float alpha1 = float(1.0 - beta1), alpha2 = float(1.0 - beta2);
  const float value = float(-lr * std::sqrt(1.0 - std::pow(beta2, step)));
  if (!(grad_clamp >= 0.0) || !(ema_one_minus_decay >= 0.0 && ema_one_minus_decay <= 1.0))
    return fail(STB_ERR_ARG, "adamw_bf16_multi: grad_clamp must be >= 0 (0 = off) and 1 - ema decay in [0, 1]");
  stb::adamw_bf16_multi_kernel<<<num_blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      ptrs, sizes, decay, blk_tensor, blk_off, T, float(beta1), float(beta2), alpha1, alpha2, value, float(eps), rnd, rnd_off, rnd_plane, seed,
      float(grad_clamp), ema_shadow, float(ema_one_minus_decay));
  STB_LAUNCH_CHECK("adamw_bf16_multi");
  return 0;
}

int stb_adamw_bf16_chunk(void) { return stb::OPT_CHUNK; }

int stb_gate_mul(const void* x, long long x_b, long long x_s, const void* gate, long long g_b, void* y,
                 long long y_b, long long y_s, int B, int S, int D, void* stream) {
  if (int r = check_device()) return r;
  if ((D & 7) || !aligned16(x) || !aligned16(y) || !aligned16(gate) || (x_s & 7) || (x_b & 7) || (y_s & 7) ||
      (y_b & 7) || (g_b & 7))
    return fail(STB_ERR_ARG, "gate_mul alignment");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = (long long)B * S * (D >> 3);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  stb::gate_mul_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), x_b, x_s, static_cast<const __nv_bfloat16*>(gate), g_b, static_cast<__nv_bfloat16*>(y), y_b, y_s, B, S, D);
  STB_LAUNCH_CHECK("gate_mul");
  return 0;
}

int stb_lokr_rebuild(const void* W, long long w_row_stride, const void* w1, const void* w2, float scale, void* out,
                     long long out_row_stride, void* out_t, long long out_t_row_stride, int a, int b, int c, int d, void* stream) {
  if (int r = check_device()) return r;
  if (!W || !w1 || !w2 || !out || a < 1 || b < 1 || c < 1 || d < 1) return fail(STB_ERR_ARG, "lokr_rebuild: bad arguments");
  const long long N = (long long)a * b, K = (long long)c * d;
  if (N > INT_MAX || K > INT_MAX) return fail(STB_ERR_ARG, "lokr_rebuild: shape too large");
  if (!aligned16(W) || !aligned16(out) || (out_t && !aligned16(out_t))) return fail(STB_ERR_ARG, "lokr_rebuild: pointers must be 16-byte aligned");
  dim3 grid((unsigned)((K + stb::LOKR_TILE - 1) / stb::LOKR_TILE), (unsigned)((N + stb::LOKR_TILE - 1) / stb::LOKR_TILE));
  stb::lokr_rebuild_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(W), w_row_stride, static_cast<const __nv_bfloat16*>(w1), static_cast<const __nv_bfloat16*>(w2),
      scale, static_cast<__nv_bfloat16*>(out), out_row_stride, static_cast<__nv_bfloat16*>(out_t), out_t_row_stride, (int)N, (int)K, b, c, d);
  STB_LAUNCH_CHECK("lokr_rebuild");
  return 0;
}

int stb_lokr_factor_grads(const void* dW, long long dw_row_stride, const void* w1, const void* w2, float scale, float* dw1,
                          float* dw2, int a, int b, int c, int d, void* stream) {
  if (int r = check_device()) return r;
  if (!dW || !w1 || !w2 || !dw1 || !dw2 || a < 1 || b < 1 || c < 1 || d < 8) return fail(STB_ERR_ARG, "lokr_factor_grads: bad arguments");
  if ((d & 7) || (dw_row_stride & 7) || !aligned16(dW) || !aligned16(w2) || !aligned16(dw2))
    return fail(STB_ERR_ARG, "lokr_factor_grads: d and the dW row stride must be multiples of 8, pointers 16-byte aligned");
  if ((long long)a * c * 4 > 48 * 1024) return fail(STB_ERR_ARG, "lokr_factor_grads: a * c too large for the partial-sum buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  STB_CUDA(cudaMemsetAsync(dw1, 0, sizeof(float) * (size_t)a * c, st));
  const long long vecs = ((long long)b * d) / 8;
  const int grid = (int)((vecs + 255) / 256);
  stb::lokr_factor_grad_kernel<<<grid, 256, sizeof(float) * (size_t)a * c, st>>>(
      static_cast<const __nv_bfloat16*>(dW), dw_row_stride, static_cast<const __nv_bfloat16*>(w1), static_cast<const __nv_bfloat16*>(w2),
      scale, dw1, dw2, a, b, c, d);
  STB_LAUNCH_CHECK("lokr_factor_grads");
  return 0;
}

int stb_rmsnorm_fwd(const void* x, long long x_b, long long x_s, const void* w, void* out, long long o_b, long long o_s,
                    int B, int S, int D, float eps, void* stream) {
  if (int r = check_device()) return r;
  if (!x || !w || !out || B < 1 || S < 1 || D < 8 || (D & 7)) return fail(STB_ERR_ARG, "rmsnorm_fwd: bad shape (D multiple of 8)");
  if (!aligned16(x) || !aligned16(out) || !aligned16(w) || (x_b & 7) || (x_s & 7) || (o_b & 7) || (o_s & 7))
    return fail(STB_ERR_ARG, "rmsnorm_fwd alignment");
  const long long rows = (long long)B * S;
  stb::rmsnorm_fwd_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), x_b, x_s, static_cast<const __nv_bfloat16*>(w), static_cast<__nv_bfloat16*>(out), o_b,
      o_s, B, S, D, eps);
  STB_LAUNCH_CHECK("rmsnorm_fwd");
  return 0;
}

int stb_gelu_tanh(const void* pre, long long p_b, long long p_s, const void* g, long long g_b, long long g_s, void* y,
                  long long y_b, long long y_s, int B, int S, int D, int mode, void* stream) {
  if (int r = check_device()) return r;
  if (mode != 0 && mode != 1) return fail(STB_ERR_ARG, "gelu_tanh: mode 0 (gelu) or 1 (g * gelu')");
  if (!pre || !y || (mode == 1 && !g) || B < 1 || S < 1 || D < 8) return fail(STB_ERR_ARG, "gelu_tanh: bad arguments");
  if ((D & 7) || !aligned16(pre) || !aligned16(y) || (p_s & 7) || (p_b & 7) || (y_s & 7) || (y_b & 7) ||
      (mode == 1 && (!aligned16(g) || (g_s & 7) || (g_b & 7))))
    return fail(STB_ERR_ARG, "gelu_tanh alignment");
  const long long total = (long long)B * S * (D >> 3);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  stb::gelu_tanh_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(pre), p_b, p_s, static_cast<const __nv_bfloat16*>(g), g_b, g_s,
      static_cast<__nv_bfloat16*>(y), y_b, y_s, B, S, D, mode);
  STB_LAUNCH_CHECK("gelu_tanh");
  return 0;
}

static int dropout_args(const void* a, const void* b, int members, int B, int S, int K, float p) {
  if (!a || !b || members < 1 || members > 8 || B < 1 || S < 1 || K < 8 || (K & 7)) return fail(STB_ERR_ARG, "dropout: bad shape (K multiple of 8, 1..8 members)");
  if (!(p >= 0.f && p < 1.f)) return fail(STB_ERR_ARG, "dropout: p must be in [0, 1)");
  if (!aligned16(a) || !aligned16(b)) return fail(STB_ERR_ARG, "dropout: pointers must be 16-byte aligned");
  return 0;
}

int stb_dropout_expand(const void* x, long long x_b, long long x_s, void* out, int members, int B, int S, int K, float p,
                       unsigned int seed, unsigned int stream0, void* stream) {
  if (int r = check_device()) return r;
  if (int r = dropout_args(x, out, members, B, S, K, p)) return r;
  if ((x_b & 7) || (x_s & 7)) return fail(STB_ERR_ARG, "dropout_expand: strides must be multiples of 8 elements");
  const long long total = (long long)B * S * (K >> 3);
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  const uint32_t thresh = (uint32_t)std::llround(double(p) * 16777216.0);
  stb::dropout_expand_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), x_b, x_s, static_cast<__nv_bfloat16*>(out), members, B, S, K, 1.f / (1.f - p), thresh, seed, stream0);
  STB_LAUNCH_CHECK("dropout_expand");
  return 0;
}

int stb_dropout_accum(const void* d, void* dx, long long dx_b, long long dx_s, int members, int B, int S, int K, float p,
                      unsigned int seed, unsigned int stream0, void* stream) {
  if (int r = check_device()) return r;
  if (int r = dropout_args(d, dx, members, B, S, K, p)) return r;
  if ((dx_b & 7) || (dx_s & 7)) return fail(STB_ERR_ARG, "dropout_accum: strides must be multiples of 8 elements");
  const long long total = (long long)B * S * (K >> 3);
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
  const uint32_t thresh = (uint32_t)std::llround(double(p) * 16777216.0);
  stb::dropout_accum_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(d), static_cast<__nv_bfloat16*>(dx), dx_b, dx_s, members, B, S, K, 1.f / (1.f - p), thresh, seed, stream0);
  STB_LAUNCH_CHECK("dropout_accum");
  return 0;
}

int stb_wgrad_full(const void* dy, long long dy_b, long long dy_s, const void* x, long long x_b, long long x_s, void* dw,
                   long long dw_row_stride, int B, int S, int N, int K, float alpha, int accumulate, void* stream) {
  if (int r = check_device()) return r;
  if (!dy || !x || !dw || B < 1 || S < 1 || N < 8 || K < 8 || (N & 7) || (K & 7)) return fail(STB_ERR_ARG, "wgrad_full: N, K must be positive multiples of 8");
  if (!aligned16(dw) || (dw_row_stride & 7)) return fail(STB_ERR_ARG, "wgrad_full: dW must be 16-byte aligned with a row stride multiple of 8");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  stb::WgradFullMaps maps;
  unsigned bx[3] = {64, 64, 1};
  {
    unsigned long long d[3] = {(unsigned long long)N, (unsigned long long)S, (unsigned long long)B};
    unsigned long long sb[2] = {(unsigned long long)dy_s * 2ull, (unsigned long long)(B == 1 ? dy_s * (long long)S : dy_b) * 2ull};
    if (int r = make_map(&maps.dy, dy, 3, d, sb, bx)) return r;
  }
  {
    unsigned long long d[3] = {(unsigned long long)K, (unsigned long long)S, (unsigned long long)B};
    unsigned long long sb[2] = {(unsigned long long)x_s * 2ull, (unsigned long long)(B == 1 ? x_s * (long long)S : x_b) * 2ull};
    if (int r = make_map(&maps.x, x, 3, d, sb, bx)) return r;
  }
  stb::WgradFullParams p;
  p.S = S; p.B = B; p.N = N; p.K = K;
  p.alpha = alpha;
  p.accumulate = accumulate;
  p.out = static_cast<__nv_bfloat16*>(dw);
  p.out_row_stride = dw_row_stride;
  const int tiles_n = (N + 127) / 128;
  const int sms = num_sms();
  // 256-wide tiles unless they leave more than half of the SMs idle
  const bool wide = tiles_n * ((K + 255) / 256) >= sms / 2 || K <= 128;
  if (wide) {
    auto kern = stb::wgrad_full_kernel<256>;
    constexpr int SMEM = stb::WgradFullCfg<256>::SMEM_BYTES;
    static bool configured = false;
    if (!configured) { if (int r = set_smem(kern, SMEM)) return r; configured = true; }
    const int tiles = tiles_n * ((K + 255) / 256);
    kern<<<std::min(tiles, sms), 384, SMEM, st>>>(maps, p);
  } else {
    auto kern = stb::wgrad_full_kernel<128>;
    constexpr int SMEM = stb::WgradFullCfg<128>::SMEM_BYTES;
    static bool configured = false;
    if (!configured) { if (int r = set_smem(kern, SMEM)) return r; configured = true; }
    const int tiles = tiles_n * ((K + 127) / 128);
    kern<<<std::min(tiles, sms), 384, SMEM, st>>>(maps, p);
  }
  STB_LAUNCH_CHECK("wgrad_full");
  return 0;
}

int stb_colsum2(const void* dy, long long dy_b, long long dy_s, const void* z, long long z_b, long long z_s, float* sum,
                float* dot, int B, int S, int D, void* stream) {
  if (int r = check_device()) return r;
  if (!dy || (!sum && !dot) || B < 1 || S < 1 || D < 8 || (D & 7)) return fail(STB_ERR_ARG, "colsum2: bad arguments (D multiple of 8)");
  if (dot && !z) return fail(STB_ERR_ARG, "colsum2: dot needs z");
  if (!aligned16(dy) || (dy_b & 7) || (dy_s & 7) || (z && (!aligned16(z) || (z_b & 7) || (z_s & 7))))
    return fail(STB_ERR_ARG, "colsum2: operands must be 16-byte aligned with strides multiple of 8");
  const int vecs = D >> 3;
  const int gx = (vecs + 255) / 256;
  int rows = std::max(8, (int)(((long long)S * B * gx + (long long)num_sms() * 8 - 1) / ((long long)num_sms() * 8)));
  dim3 grid(gx, (S + rows - 1) / rows, B);
  stb::colsum2_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(dy), dy_b, dy_s, static_cast<const __nv_bfloat16*>(z), z_b, z_s, sum, dot, B, S, D, rows);
  STB_LAUNCH_CHECK("colsum2");
  return 0;
}

static void skinny_split(int B, int S, int N, int& rows, int& spb) {
  const int n_tiles = (N + 127) / 128;
  spb = std::max(1, (2 * num_sms()) / std::max(1, n_tiles * B));     // ~2 CTAs' worth of work per SM
  rows = ((S + spb - 1) / spb + 63) / 64 * 64;
  spb = (S + rows - 1) / rows;
}

long long stb_skinny_tn_workspace(int B, int S, int R, int N) {
  if (B < 1 || S < 1 || R < 1 || N < 1 || check_device()) return 0;
  int rows, spb;
  skinny_split(B, S, N, rows, spb);
  return (long long)spb * B * R * N;
}

int stb_skinny_tn(const void* L, long long l_b, long long l_s, const void* Rm, long long r_b, long long r_s,
                  float* out, int B, int S, int R, int N, float alpha, void* stream) {
  return stb_skinny_tn_ws(L, l_b, l_s, Rm, r_b, r_s, out, B, S, R, N, alpha, nullptr, 0, stream);
}

int stb_skinny_tn_ws(const void* L, long long l_b, long long l_s, const void* Rm, long long r_b, long long r_s,
                     float* out, int B, int S, int R, int N, float alpha, float* workspace, long long workspace_elems,
                     void* stream) {
  if (int r = check_device()) return r;
  if (N & 1) return fail(STB_ERR_ARG, "N must be even");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // tensor-core path: both operands TMA-able (16-byte aligned rows), rank block <= 128
  if (R % 8 == 0 && R <= 128 && N % 8 == 0 && aligned16(L) && aligned16(Rm) && !(l_s & 7) && !(r_s & 7) &&
      (B == 1 || (!(l_b & 7) && !(r_b & 7)))) {
    stb::WgradMaps maps;
    unsigned bx[3] = {64, 64, 1};
    {
      unsigned long long d[3] = {(unsigned long long)N, (unsigned long long)S, (unsigned long long)B};
      unsigned long long sb[2] = {(unsigned long long)r_s * 2ull, (unsigned long long)(B == 1 ? r_s * (long long)S : r_b) * 2ull};
      if (int r = make_map(&maps.rm, Rm, 3, d, sb, bx)) return r;
    }
    {
      unsigned long long d[3] = {(unsigned long long)R, (unsigned long long)S, (unsigned long long)B};
      unsigned long long sb[2] = {(unsigned long long)l_s * 2ull, (unsigned long long)(B == 1 ? l_s * (long long)S : l_b) * 2ull};
      if (int r = make_map(&maps.l, L, 3, d, sb, bx)) return r;
    }
    stb::WgradParams p;
    p.S = S; p.B = B; p.N = N; p.R = R;
    p.alpha = alpha;
    p.out = out;
    const int n_tiles = (N + 127) / 128;
    int spb, rows;
    skinny_split(B, S, N, rows, spb);
    p.partial = nullptr;
    if (workspace) {
      if (workspace_elems < (long long)spb * B * R * N) return fail(STB_ERR_ARG, "skinny_tn workspace too small (stb_skinny_tn_workspace)");
      p.partial = workspace;
    }
    p.rows_per_split = rows;
    p.splits_per_batch = spb;
    dim3 grid(n_tiles, spb * B);
    if (R <= 64) {
      auto kern = stb::wgrad_tn_kernel<64>;
      static bool configured = false;
      if (!configured) {
        if (int r = set_smem(kern, stb::WgradCfg<64>::SMEM_BYTES)) return r;
        configured = true;
      }
      kern<<<grid, 384, stb::WgradCfg<64>::SMEM_BYTES, st>>>(maps, p);
    } else {
      auto kern = stb::wgrad_tn_kernel<128>;
      static bool configured = false;
      if (!configured) {
        if (int r = set_smem(kern, stb::WgradCfg<128>::SMEM_BYTES)) return r;
        configured = true;
      }
      kern<<<grid, 384, stb::WgradCfg<128>::SMEM_BYTES, st>>>(maps, p);
    }
    STB_LAUNCH_CHECK("wgrad_tn");
    if (workspace) {
      const long long n = (long long)R * N;
      stb::wgrad_reduce_slabs_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, (long long)num_sms() * 8), 256, 0, st>>>(
          workspace, out, spb * B, n, alpha);
      STB_LAUNCH_CHECK("wgrad_reduce_slabs");
    }
    return 0;
  }
  if (workspace) return fail(STB_ERR_UNSUPPORTED, "deterministic skinny_tn needs the tensor-core path (R % 8 == 0, R <= 128, N % 8 == 0, 16-byte aligned operands)");
  const long long M = (long long)B * S;
  const int col_blocks = (N / 2 + 255) / 256;
  // enough row chunks to fill the machine ~4x
  int chunks = std::max(1, (num_sms() * 4) / col_blocks);
  long long mchunk = ((M + chunks - 1) / chunks + 63) / 64 * 64;
  chunks = (int)((M + mchunk - 1) / mchunk);
  dim3 grid(col_blocks, chunks);
  auto LL = static_cast<const __nv_bfloat16*>(L);
  auto RR = static_cast<const __nv_bfloat16*>(Rm);
  switch (R) {
    case 16: stb::skinny_tn_kernel<16><<<grid, 256, 0, st>>>(LL, l_b, l_s, RR, r_b, r_s, out, B, S, N, alpha, (int)mchunk); break;
    case 32: stb::skinny_tn_kernel<32><<<grid, 256, 0, st>>>(LL, l_b, l_s, RR, r_b, r_s, out, B, S, N, alpha, (int)mchunk); break;
    case 48: stb::skinny_tn_kernel<48><<<grid, 256, 0, st>>>(LL, l_b, l_s, RR, r_b, r_s, out, B, S, N, alpha, (int)mchunk); break;
    case 64: stb::skinny_tn_kernel<64><<<grid, 256, 0, st>>>(LL, l_b, l_s, RR, r_b, r_s, out, B, S, N, alpha, (int)mchunk); break;
    default: return fail(STB_ERR_UNSUPPORTED, "LoRA rank block R=%d not supported (16/32/48/64)", R);
  }
  STB_LAUNCH_CHECK("skinny_tn");
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------- VAE latent encode
template <int BN>
static int launch_conv3x3(const void* x, const void* w, const void* bias, const void* res, void* out, int B, int H,
                          int W, int C_in, int C_out, int stride, cudaStream_t st) {
  using Cfg = stb::GemmCfg<BN>;
  const int H_out = stride == 1 ? H : H / 2, W_out = stride == 1 ? W : W / 2;
  stb::GemmMaps maps;
  std::memset(&maps, 0, sizeof maps);
  {
    unsigned long long d[4] = {(unsigned long long)C_in, (unsigned long long)W, (unsigned long long)H, (unsigned long long)B};
    unsigned long long sb[3] = {(unsigned long long)C_in * 2ull, (unsigned long long)W * C_in * 2ull,
                                (unsigned long long)H * W * C_in * 2ull};
    unsigned bx[4] = {64, (unsigned)(128 * stride), 1, 1};  // traversed span: 128 elements at stride `stride`
    unsigned es[4] = {1, (unsigned)stride, 1, 1};
    if (int r = make_map_strided(&maps.a[0], x, 4, d, sb, bx, es)) return r;
  }
  {
    unsigned long long d[2] = {(unsigned long long)9 * C_in, (unsigned long long)C_out};
    unsigned long long sb[1] = {(unsigned long long)9 * C_in * 2ull};
    unsigned bx[2] = {64, (unsigned)BN};
    if (int r = make_map(&maps.w[0], w, 2, d, sb, bx)) return r;
  }
  stb::GemmParams p;
  std::memset(&p, 0, sizeof p);
  p.rows_per_batch = W_out;
  p.num_batches = B * H_out;
  p.N = C_out;
  p.nseg = 1;
  p.kblocks[0] = 9 * (C_in / 64);
  p.epi = res ? stb::EPI_ADD_RES : stb::EPI_STORE;
  p.D = static_cast<__nv_bfloat16*>(out);
  p.d_batch_stride = (long long)W_out * C_out;
  p.d_row_stride = C_out;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.res = static_cast<const __nv_bfloat16*>(res);
  p.res_batch_stride = p.d_batch_stride;
  p.res_row_stride = C_out;
  p.conv_h_out = H_out;
  p.conv_stride = stride;
  p.conv_pad = stride == 1 ? 1 : 0;
  p.conv_cblocks = C_in / 64;
  auto kernel = stb::gemm_bf16_tn_kernel<BN, true>;
  static bool configured = false;
  if (!configured) {
    if (int r = set_smem(kernel, Cfg::SMEM_BYTES)) return r;
    configured = true;
  }
  const long long tiles = (long long)((W_out + 127) / 128) * p.num_batches * ((C_out + BN - 1) / BN);
  const int grid = (int)std::min<long long>(tiles, num_sms());
  kernel<<<grid, 384, Cfg::SMEM_BYTES, st>>>(maps, p);
  STB_LAUNCH_CHECK("conv3x3_nhwc");
  return 0;
}

extern "C" {

int stb_conv3x3_nhwc(const void* x, const void* w, const void* bias, const void* res, void* out, int B, int H, int W,
                     int C_in, int C_out, int stride, void* stream) {
  if (int r = check_device()) return r;
  if (C_in % 64 || C_out % 8) return fail(STB_ERR_ARG, "conv3x3_nhwc needs C_in %% 64 == 0 and C_out %% 8 == 0 (got %d, %d)", C_in, C_out);
  if (stride != 1 && stride != 2) return fail(STB_ERR_ARG, "conv3x3_nhwc stride must be 1 or 2");
  if (stride == 2 && ((H | W) & 1)) return fail(STB_ERR_ARG, "stride-2 conv needs even H, W");
  if (!aligned16(x) || !aligned16(w) || !aligned16(out) || (res && !aligned16(res)) || (bias && !aligned16(bias)))
    return fail(STB_ERR_ARG, "conv3x3_nhwc alignment");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (C_out > 128) return launch_conv3x3<256>(x, w, bias, res, out, B, H, W, C_in, C_out, stride, st);
  if (C_out > 64) return launch_conv3x3<128>(x, w, bias, res, out, B, H, W, C_in, C_out, stride, st);
  return launch_conv3x3<64>(x, w, bias, res, out, B, H, W, C_in, C_out, stride, st);
}

int stb_conv_in_3ch(const void* pixels, const void* w, const void* bias, void* out, int B, int H, int W, int C,
                    void* stream) {
  if (int r = check_device()) return r;
  if (C % 8 || C > 512) return fail(STB_ERR_ARG, "conv_in_3ch: C must be a multiple of 8, <= 512");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((C == 64 || C == 128 || C == 256) && aligned16(bias) && aligned16(out)) {
    // tensor-core path: im2col tiles built in shared memory, K = 27 padded to 32
    constexpr int SMEM = 32768 + 16384 + 1024;
    const long long tiles = (long long)B * H * ((W + 127) / 128);
    const int grid = (int)std::min<long long>(tiles, 2LL * num_sms());
    auto px = static_cast<const __nv_bfloat16*>(pixels);
    auto wt = static_cast<const __nv_bfloat16*>(w);
    auto bs = static_cast<const __nv_bfloat16*>(bias);
    auto o = static_cast<__nv_bfloat16*>(out);
    static bool configured = false;
    if (!configured) {
      if (int r = set_smem(stb::conv_in_3ch_mma_kernel<256>, SMEM)) return r;
      if (int r = set_smem(stb::conv_in_3ch_mma_kernel<128>, SMEM)) return r;
      if (int r = set_smem(stb::conv_in_3ch_mma_kernel<64>, SMEM)) return r;
      configured = true;
    }
    if (C == 256) stb::conv_in_3ch_mma_kernel<256><<<grid, 256, SMEM, st>>>(px, wt, bs, o, B, H, W);
    else if (C == 128) stb::conv_in_3ch_mma_kernel<128><<<grid, 256, SMEM, st>>>(px, wt, bs, o, B, H, W);
    else stb::conv_in_3ch_mma_kernel<64><<<grid, 256, SMEM, st>>>(px, wt, bs, o, B, H, W);
    STB_LAUNCH_CHECK("conv_in_3ch_mma");
    return 0;
  }
  const long long total = (long long)B * H * W * (C / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  const int smem = (C * 27 + C) * (int)sizeof(float);
  auto kernel = stb::conv_in_3ch_kernel;
  static bool configured = false;
  if (!configured) {
    if (int r = set_smem(kernel, 512 * 28 * (int)sizeof(float))) return r;
    configured = true;
  }
  kernel<<<grid, 256, smem, st>>>(static_cast<const __nv_bfloat16*>(pixels), static_cast<const __nv_bfloat16*>(w),
                                  static_cast<const __nv_bfloat16*>(bias), static_cast<__nv_bfloat16*>(out), B, H, W, C);
  STB_LAUNCH_CHECK("conv_in_3ch");
  return 0;
}

int stb_groupnorm_nhwc(const void* x, const void* gamma, const void* beta, void* out, float* stats, int B, int HW,
                       int C, int G, float eps, int silu, void* stream) {
  if (int r = check_device()) return r;
  if (C % 8 || C > 512 || G > 64 || C % G || (8 % (C / G) && (C / G) % 8)) return fail(STB_ERR_ARG, "groupnorm_nhwc: unsupported C=%d G=%d", C, G);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  STB_CUDA(cudaMemsetAsync(stats, 0, sizeof(float) * 2 * B * G, st));
  const int chunks = std::max(1, std::min((HW + 255) / 256, (num_sms() * 4 + B - 1) / B));
  const int ppc = (HW + chunks - 1) / chunks;
  stb::groupnorm_stats_kernel<<<dim3((HW + ppc - 1) / ppc, B), 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), stats, HW, C, G, ppc);
  STB_LAUNCH_CHECK("groupnorm_stats");
  const int achunks = std::max(1, std::min((HW + 63) / 64, (num_sms() * 16 + B - 1) / B));
  const int appc = (HW + achunks - 1) / achunks;
  stb::groupnorm_apply_kernel<<<dim3((HW + appc - 1) / appc, B), 256, 0, st>>>(
      static_cast<const __nv_bfloat16*>(x), stats, static_cast<const __nv_bfloat16*>(gamma), static_cast<const __nv_bfloat16*>(beta),
      static_cast<__nv_bfloat16*>(out), B, HW, C, G, eps, silu, appc);
  STB_LAUNCH_CHECK("groupnorm_apply");
  return 0;
}

int stb_softmax_rows(void* s, long long row_stride, int rows, int cols, float scale, void* stream) {
  if (int r = check_device()) return r;
  if (cols % 8 || (row_stride & 7) || !aligned16(s)) return fail(STB_ERR_ARG, "softmax_rows alignment");
  stb::softmax_rows_kernel<<<rows, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<__nv_bfloat16*>(s), row_stride, cols, scale);
  STB_LAUNCH_CHECK("softmax_rows");
  return 0;
}

int stb_gaussian_sample_scale(const void* moments, const void* eps, void* out, int B, int L, int hw, float shift,
                              float scale, int has_shift, void* stream) {
  if (int r = check_device()) return r;
  const long long total = (long long)B * L * hw;
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  stb::gaussian_sample_scale_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(moments), static_cast<const __nv_bfloat16*>(eps), static_cast<__nv_bfloat16*>(out), B, L, hw, shift, scale, has_shift);
  STB_LAUNCH_CHECK("gaussian_sample_scale");
  return 0;
}

}  // extern "C"
