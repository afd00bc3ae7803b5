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
  // The tensor-map encoder is a driver call and needs a context current on the calling thread.  A thread whose first CUDA
  // work is a libstb200 call has none (the autograd engine's device thread, when an attention backward is the first op
  // it runs); cudaSetDevice makes the primary context of the thread's device current.
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaSetDevice(dev) != cudaSuccess)
    return fail(STB_ERR_CUDA, "no CUDA context for the calling thread");
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

// bf16 SWIZZLE_128B map, dims / box / per-dimension traversal strides innermost-first, strides in BYTES for dims
// 1..rank-1; not cached (the strided conv windows use it directly)
int make_map_strided(CUtensorMap* out, const void* ptr, int rank, const unsigned long long* dims,
                     const unsigned long long* strides_bytes, const unsigned* box, const unsigned* estrides) {
  auto fn = encode_fn();
  if (!fn) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if (reinterpret_cast<uintptr_t>(ptr) & 15) return fail(STB_ERR_ARG, "tensor base pointer must be 16-byte aligned");
  for (int i = 0; i + 1 < rank; ++i)
    if (strides_bytes[i] & 15) return fail(STB_ERR_ARG, "tensor stride %d (%llu bytes) must be a multiple of 16 bytes", i, strides_bytes[i]);
  cuuint64_t gdim[4];
  cuuint64_t gstr[3];
  cuuint32_t bx[4], es[4];
  for (int i = 0; i < rank; ++i) gdim[i] = dims[i], bx[i] = box[i], es[i] = estrides[i];
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(STB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", int(r));
  return 0;
}

// make_map_strided with unit traversal strides, cached by (pointer, shape, strides, box)
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
  static const unsigned unit[4] = {1, 1, 1, 1};
  if (int r = make_map_strided(out, ptr, rank, dims, strides_bytes, box, unit)) return r;
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    if (g_maps.size() > 65536) g_maps.clear();
    g_maps.emplace(key, *out);
  }
  return 0;
}

// Token-major operand [B, S, C] (row stride s_stride, batch stride b_stride, in elements) as the 3-D map (C, S, B) with
// box (64, rows, 1).  With one batch the batch stride addresses nothing, so S rows stand in for it: views of a larger
// buffer then encode whatever batch stride they carry.
int make_token_map(CUtensorMap* out, const void* ptr, int C, int S, int B, long long s_stride, long long b_stride,
                   unsigned rows) {
  const unsigned long long d[3] = {(unsigned long long)C, (unsigned long long)S, (unsigned long long)B};
  const unsigned long long sb[2] = {(unsigned long long)s_stride * 2ull,
                                    (unsigned long long)(B == 1 ? s_stride * (long long)S : b_stride) * 2ull};
  const unsigned bx[3] = {64, rows, 1};
  return make_map(out, ptr, 3, d, sb, bx);
}

// Attention operand [B, S, H, HD] with element strides (sb, ss, sh) as the 4-D map (HD, H, S, B), box (64, 1, rows, 1):
// one head's rows of one batch per load
int make_head_map(CUtensorMap* out, const void* ptr, int HD, int H, int S, int B, long long sb, long long ss,
                  long long sh, unsigned rows) {
  const unsigned long long d[4] = {(unsigned long long)HD, (unsigned long long)H, (unsigned long long)S, (unsigned long long)B};
  const unsigned long long s[3] = {(unsigned long long)sh * 2ull, (unsigned long long)ss * 2ull, (unsigned long long)sb * 2ull};
  const unsigned bx[4] = {64, 1, rows, 1};
  return make_map(out, ptr, 4, d, s, bx);
}

// Raises Kernel's dynamic shared-memory limit before its first launch.  Thread-safe: concurrent first calls both set
// the same value; a failed call is reported and retried on the next launch.
template <auto Kernel>
int set_smem(int bytes) {
  static std::atomic<bool> done{false};
  if (done.load(std::memory_order_acquire)) return 0;
  STB_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.store(true, std::memory_order_release);
  return 0;
}

// ---------------------------------------------------------------- GEMM
// One launch of the persistent GEMM for GEMM and conv3x3 alike: one CTA per SM, or one per tile when there are fewer.
// CLUSTER = 2: one 2-CTA cluster per pair tile, at most as many as the device can hold at once (the GPCs' SM counts
// decide how many pairs of SMs there are, so it is asked, once per kernel).
template <int BN, int EPI, bool CONV, int CLUSTER = 1>
int launch_gemm_kernel(const stb::GemmMaps& maps, const stb::GemmParams& p, cudaStream_t st, const char* name) {
  using Cfg = stb::GemmCfg<BN>;
  constexpr auto kernel = stb::gemm_bf16_tn_kernel<BN, EPI, CONV, CLUSTER>;
  if (int r = set_smem<kernel>(Cfg::SMEM_BYTES)) return r;
  const long long tiles_m = (long long)((p.rows_per_batch + Cfg::BM - 1) / Cfg::BM) * p.num_batches;
  const long long units = (tiles_m + CLUSTER - 1) / CLUSTER * ((p.N + BN - 1) / BN);
  if constexpr (CLUSTER == 1) {
    const int grid = (int)std::min<long long>(units, num_sms());
    kernel<<<grid, 384, Cfg::SMEM_BYTES, st>>>(maps, p);
  } else {
    cudaLaunchConfig_t cfg;
    std::memset(&cfg, 0, sizeof cfg);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CLUSTER;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3(384);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    static std::atomic<int> max_clusters{0};
    int mc = max_clusters.load(std::memory_order_acquire);
    if (mc == 0) {
      cfg.gridDim = dim3(CLUSTER * (num_sms() / CLUSTER));
      STB_CUDA(cudaOccupancyMaxActiveClusters(&mc, kernel, &cfg));
      if (mc < 1) return fail(STB_ERR_CUDA, "%s: no %d-CTA cluster of this kernel fits on the device", name, CLUSTER);
      max_clusters.store(mc, std::memory_order_release);
    }
    cfg.gridDim = dim3((unsigned)(CLUSTER * std::min<long long>(units, mc)));
    STB_CUDA(cudaLaunchKernelEx(&cfg, kernel, maps, p));
  }
  STB_LAUNCH_CHECK(name);
  return 0;
}

template <int BN>
int launch_gemm(const stb_gemm_args* a, cudaStream_t st, bool cluster) {
  stb::GemmMaps maps;
  std::memset(&maps, 0, sizeof maps);
  stb::GemmParams p;
  std::memset(&p, 0, sizeof p);
  for (int s = 0; s < a->nseg; ++s) {
    const stb_gemm_seg& g = a->seg[s];
    if (g.K <= 0 || (g.K & 7)) return fail(STB_ERR_ARG, "segment %d: K=%d must be a positive multiple of 8", s, g.K);
    if (int r = make_token_map(&maps.a[s], g.a, g.K, a->rows_per_batch, a->num_batches, g.a_row_stride, g.a_batch_stride,
                               stb::GemmCfg<BN>::BM))
      return r;
    if (g.w_kn) {   // [K, N] row-major: contraction index = row; staged as 64 x 64 MN-major boxes
      unsigned long long wd[2] = {(unsigned long long)a->N, (unsigned long long)g.K};
      unsigned long long ws[1] = {(unsigned long long)g.w_row_stride * 2ull};
      unsigned wb[2] = {64, 64};
      if (int r = make_map(&maps.w[s], g.w, 2, wd, ws, wb)) return r;
    } else {
      unsigned long long wd[2] = {(unsigned long long)g.K, (unsigned long long)a->N};
      unsigned long long ws[1] = {(unsigned long long)g.w_row_stride * 2ull};
      unsigned wb[2] = {64, cluster ? 64u : (unsigned)BN};   // a cluster CTA loads half of the W tile's rows
      if (int r = make_map(&maps.w[s], g.w, 2, wd, ws, wb)) return r;
    }
    p.w_kn[s] = g.w_kn ? 1 : 0;
    p.kblocks[s] = (g.K + 63) / 64;
  }
  p.rows_per_batch = a->rows_per_batch;
  p.num_batches = a->num_batches;
  p.N = a->N;
  p.nseg = a->nseg;
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
  // the 2-CTA cluster kernels exist at BN 128 only
  auto go = [&](auto epi) -> int {
    constexpr int EPI = decltype(epi)::value;
    if constexpr (BN == 128)
      if (cluster) return launch_gemm_kernel<BN, EPI, false, 2>(maps, p, st, "gemm_bf16_tn_cluster");
    return launch_gemm_kernel<BN, EPI, false>(maps, p, st, "gemm_bf16_tn");
  };
  switch (a->epi) {
    case stb::EPI_STORE: return go(std::integral_constant<int, stb::EPI_STORE>{});
    case stb::EPI_GELU: return go(std::integral_constant<int, stb::EPI_GELU>{});
    case stb::EPI_GATE_RES: return go(std::integral_constant<int, stb::EPI_GATE_RES>{});
    case stb::EPI_MUL_DGELU: return go(std::integral_constant<int, stb::EPI_MUL_DGELU>{});
    case stb::EPI_ADD_RES: return go(std::integral_constant<int, stb::EPI_ADD_RES>{});
    case stb::EPI_MUL: return go(std::integral_constant<int, stb::EPI_MUL>{});
    case stb::EPI_QUICK_GELU: return go(std::integral_constant<int, stb::EPI_QUICK_GELU>{});
  }
  return fail(STB_ERR_ARG, "unknown epilogue %d", a->epi);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

template <int HD, bool BIAS, bool KEY = false>
static int launch_attn_fwd(const stb::AttnFwdMaps& maps, const stb::AttnFwdParams& p, dim3 grid, cudaStream_t st) {
  using Cfg = stb::AttnFwdCfg<HD>;
  constexpr int SMEM = Cfg::SMEM_BYTES + (KEY ? Cfg::KV_STAGES * 128 * 4 : 0);
  if (int r = set_smem<stb::attn_fwd_kernel<HD, BIAS, KEY>>(SMEM)) return r;
  stb::attn_fwd_kernel<HD, BIAS, KEY><<<grid, 384, SMEM, st>>>(maps, p);
  STB_LAUNCH_CHECK(KEY ? "attn_fwd_key_bias" : (BIAS ? "attn_fwd_bias" : "attn_fwd"));
  return 0;
}

template <int HD, bool BIAS>
static int launch_attn_bwd(const stb_attn_bwd_args* a, const stb::AttnBwdMaps& maps, const stb::AttnBwdParams& p,
                           cudaStream_t st) {
  {
    const long long warps = (long long)a->B * a->Sq * a->H;
    stb::attn_bwd_delta_kernel<HD><<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(a->o), a->o_b, a->o_s, a->o_h,
        static_cast<const __nv_bfloat16*>(a->d_o), a->do_b, a->do_s, a->do_h, a->delta, a->B, a->H, a->Sq);
    STB_LAUNCH_CHECK("attn_bwd_delta");
  }
  using Cfg = stb::AttnBwdCfg<HD>;
  constexpr int SMEM1 = Cfg::DKDV_SMEM_BYTES, SMEM2 = Cfg::DQ_SMEM_BYTES + (BIAS ? Cfg::STAGES * Cfg::KB : 0);
  if (int r = set_smem<stb::attn_bwd_dkdv_kernel<HD, BIAS>>(SMEM1)) return r;
  if (int r = set_smem<stb::attn_bwd_dq_kernel<HD, BIAS>>(SMEM2)) return r;
  stb::attn_bwd_dkdv_kernel<HD, BIAS><<<dim3((a->Sk + 63) / 64, a->H, a->B), 384, SMEM1, st>>>(maps, p);
  STB_LAUNCH_CHECK(BIAS ? "attn_bwd_dkdv_bias" : "attn_bwd_dkdv");
  stb::attn_bwd_dq_kernel<HD, BIAS><<<dim3((a->Sq + 127) / 128, a->H, a->B), 384, SMEM2, st>>>(maps, p);
  STB_LAUNCH_CHECK(BIAS ? "attn_bwd_dq_bias" : "attn_bwd_dq");
  return 0;
}

// Weight-gradient GEMM over p's work units: one CTA per unit, at most one per SM for the persistent full-rank grid.
template <int BN, int OUT>
static int launch_wgrad(const stb::WgradMaps& maps, stb::WgradParams p, cudaStream_t st) {
  constexpr int SMEM = stb::WgradCfg<BN, OUT>::SMEM_BYTES;
  if (int r = set_smem<stb::wgrad_kernel<BN, OUT>>(SMEM)) return r;
  p.col_tiles = (p.K + BN - 1) / BN;   // 1 for a LoRA rank (R <= BN)
  const int units = p.splits * ((p.N + 127) / 128) * p.col_tiles;
  const int grid = OUT == stb::WGRAD_OUT_BF16_NK ? std::min(units, num_sms()) : units;
  stb::wgrad_kernel<BN, OUT><<<grid, 384, SMEM, st>>>(maps, p);
  STB_LAUNCH_CHECK(OUT == stb::WGRAD_OUT_BF16_NK ? "wgrad_full" : "wgrad_tn");
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
  // a tile's height follows from its width (GemmCfg: 64 x 256, 128 x 128, 128 x 64); tile_mt = 1 / 2 forces single CTAs /
  // 2-CTA clusters at BN 128, the only width that has the cluster kernel
  if (a->tile_mt < 0 || a->tile_mt > 2) return fail(STB_ERR_ARG, "unsupported tile config MT=%d", a->tile_mt);
  int bn = a->tile_bn;
  if (bn == 0) {
    // 128 x 128 wherever N allows: on H100 it matched or beat 64 x 256 at every Flux projection shape, M = 512 included.
    // Skinny M (modulation / conditioning GEMMs, a few rows per batch) streams W: 64 x 256 tiles waste no rows.
    bn = a->N <= 64 ? 64 : (a->rows_per_batch <= 64 && a->N > 128 ? 256 : 128);
  }
  if (bn == 256) return launch_gemm<256>(a, st, false);
  // Automatic: clusters for the GELU and dGELU epilogues at 16 or more m-tiles, where they measured 7-9 % faster on H100
  // (Flux fc1 / d_pre at M = 4096 and 4608, DESIGN.md 2.1); single CTAs elsewhere, where clusters were up to 5 % slower.
  if (bn == 128) {
    const long long tiles_m = (long long)((a->rows_per_batch + 127) / 128) * a->num_batches;
    const bool cluster = a->tile_mt == 2 || (a->tile_mt == 0 && tiles_m >= 16 &&
                                             (a->epi == STB_EPI_GELU || a->epi == STB_EPI_MUL_DGELU));
    return launch_gemm<128>(a, st, cluster);
  }
  if (bn == 64) return launch_gemm<64>(a, st, false);
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
    return make_head_map(m, ptr, a->HD, a->H, S, a->B, sb, ss, sh, 128);
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
  p.bias_b = a->bias_b; p.bias_h = a->bias_h; p.bias_q = a->bias_q;
  p.inv_scale = a->scale != 0.f ? 1.f / a->scale : 0.f;
  const dim3 grid((a->Sq + 127) / 128, a->H, a->B);
  if (a->bias) {   // additive bias / mask: text encoders, and the per-key bias of Flux masked training
    const bool key_row = a->bias_q == 0 && a->bias_h == 0;
    if (a->scale == 0.f || a->bias_b < 0 || a->bias_h < 0 || (a->bias_q < a->Sk && !key_row))
      return fail(STB_ERR_ARG, "attn_fwd bias: scale must be non-zero, strides non-negative, and bias_q >= Sk "
                               "(or bias_q = bias_h = 0 for a per-key row)");
    if (key_row)   // one row per sample: staged per key tile in shared memory
      return a->HD == 128 ? launch_attn_fwd<128, true, true>(maps, p, grid, st) : launch_attn_fwd<64, true, true>(maps, p, grid, st);
    return a->HD == 128 ? launch_attn_fwd<128, true>(maps, p, grid, st) : launch_attn_fwd<64, true>(maps, p, grid, st);
  }
  return a->HD == 128 ? launch_attn_fwd<128, false>(maps, p, grid, st) : launch_attn_fwd<64, false>(maps, p, grid, st);
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
    return make_head_map(m, ptr, a->HD, a->H, S, a->B, sb, ss, sh, rows);
  };
  if (int r = mk(&maps.q128, a->q, a->q_b, a->q_s, a->q_h, a->Sq, 128)) return r;
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
  p.bias = static_cast<const __nv_bfloat16*>(a->bias);
  p.bias_b = a->bias_b;
  if (a->bias) {   // per-key only: [B, Sk] rows bias_b apart, or one row shared by the batch (bias_b = 0)
    if (a->bias_b < 0 || (a->bias_b != 0 && a->bias_b < a->Sk))
      return fail(STB_ERR_UNSUPPORTED, "attn_bwd bias: only a per-key bias [B or 1, Sk] (bias_b = 0 or >= Sk) is supported");
    return a->HD == 128 ? launch_attn_bwd<128, true>(a, maps, p, st) : launch_attn_bwd<64, true>(a, maps, p, st);
  }
  return a->HD == 128 ? launch_attn_bwd<128, false>(a, maps, p, st) : launch_attn_bwd<64, false>(a, maps, p, st);
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
  auto cast = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
  auto launch = [&](auto hd) {
    stb::qk_rmsnorm_rope_fwd_kernel<decltype(hd)::value><<<grid, 256, 0, st>>>(
        cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split, cos_t, sin_t,
        static_cast<__nv_bfloat16*>(q_out), static_cast<__nv_bfloat16*>(k_out), dst_b, dst_s, B, S, H, eps);
  };
  if (HD == 128) launch(std::integral_constant<int, 128>{});
  else launch(std::integral_constant<int, 64>{});
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
  // the warp-per-token kernel, with the RMSNorm weight gradient when dw is given
  auto launch = [&](auto hd, auto with_dw) {
    stb::qk_rmsnorm_rope_bwd_kernel<decltype(hd)::value, decltype(with_dw)::value><<<grid, 256, 0, st>>>(
        cast(dq), cast(dk), d_b, d_s, cast(src), src_b, src_s, k_off, cast(wq), cast(wk), cast(wq_added), cast(wk_added), s_split,
        cos_t, sin_t, static_cast<__nv_bfloat16*>(dsrc), ds_b, ds_s, B, S, H, eps, dw);
  };
  using HD128 = std::integral_constant<int, 128>;
  using HD64 = std::integral_constant<int, 64>;
  if (HD == 128 && !dw) {
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
      launch(HD128{}, std::false_type{});
    }
  } else if (HD == 128) {
    launch(HD128{}, std::true_type{});
  } else if (dw) {
    launch(HD64{}, std::true_type{});
  } else {
    launch(HD64{}, std::false_type{});
  }
  STB_LAUNCH_CHECK("qk_rmsnorm_rope_bwd");
  return 0;
}

int stb_flow_prep_pack(const void* latents, const void* noise, const float* sigmas, void* noisy,
                       void* packed, long long packed_b, int B, int C, int Hh, int Ww, void* stream) {
  if (int r = check_device()) return r;
  if ((Hh & 1) || (Ww & 1)) return fail(STB_ERR_ARG, "latent H and W must be even for 2x2 patchify");
  if (!noise && (sigmas || noisy)) return fail(STB_ERR_ARG, "flow_prep_pack: sigmas / noisy need noise");
  if (noise && !sigmas) return fail(STB_ERR_ARG, "flow_prep_pack: noise needs sigmas");
  if (packed_b < (long long)(Hh / 2) * (Ww / 2) * 4 * C) return fail(STB_ERR_ARG, "flow_prep_pack: packed_b below one sample's tokens");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = (long long)B * C * Hh * Ww;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)num_sms() * 16);
  stb::flow_prep_pack_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(latents), static_cast<const __nv_bfloat16*>(noise), sigmas, static_cast<__nv_bfloat16*>(noisy), static_cast<__nv_bfloat16*>(packed), packed_b, B, C, Hh, Ww);
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
  stb::WgradMaps maps;
  if (int r = make_token_map(&maps.a, dy, N, S, B, dy_s, dy_b, 64)) return r;
  if (int r = make_token_map(&maps.b, x, K, S, B, x_s, x_b, 64)) return r;
  stb::WgradParams p{};
  p.N = N;
  p.K = K;
  p.chunks = (S + 63) / 64;
  p.splits = p.splits_per_group = 1;   // one split: every tile sums all B x chunks k-blocks
  p.kb_per_group = p.kb_per_split = B * p.chunks;
  p.alpha = alpha;
  p.out = static_cast<__nv_bfloat16*>(dw);
  p.out_row_stride = dw_row_stride;
  p.accumulate = accumulate;
  // 256-wide tiles unless they leave more than half of the SMs idle
  if (((N + 127) / 128) * ((K + 255) / 256) >= num_sms() / 2 || K <= 128)
    return launch_wgrad<256, stb::WGRAD_OUT_BF16_NK>(maps, p, st);
  return launch_wgrad<128, stb::WGRAD_OUT_BF16_NK>(maps, p, st);
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
    if (int r = make_token_map(&maps.a, Rm, N, S, B, r_s, r_b, 64)) return r;
    if (int r = make_token_map(&maps.b, L, R, S, B, l_s, l_b, 64)) return r;
    int spb, rows;
    skinny_split(B, S, N, rows, spb);
    if (workspace && workspace_elems < (long long)spb * B * R * N)
      return fail(STB_ERR_ARG, "skinny_tn workspace too small (stb_skinny_tn_workspace)");
    stb::WgradParams p{};
    p.N = N;
    p.K = R;
    p.chunks = (S + 63) / 64;
    // spb splits of `rows` tokens per batch; split y is batch y / spb, slab y of the workspace
    p.splits = spb * B;
    p.splits_per_group = spb;
    p.kb_per_group = p.chunks;
    p.kb_per_split = rows / 64;
    p.alpha = alpha;
    p.partial = workspace;
    p.out_f32 = out;
    if (int r = R <= 64 ? launch_wgrad<64, stb::WGRAD_OUT_F32_RN>(maps, p, st) : launch_wgrad<128, stb::WGRAD_OUT_F32_RN>(maps, p, st))
      return r;
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
  const int H_out = stride == 1 ? H : H / 2, W_out = stride == 1 ? W : W / 2;
  stb::GemmMaps maps;
  std::memset(&maps, 0, sizeof maps);
  {
    unsigned long long d[4] = {(unsigned long long)C_in, (unsigned long long)W, (unsigned long long)H, (unsigned long long)B};
    unsigned long long sb[3] = {(unsigned long long)C_in * 2ull, (unsigned long long)W * C_in * 2ull,
                                (unsigned long long)H * W * C_in * 2ull};
    unsigned bx[4] = {64, (unsigned)(stb::GemmCfg<BN>::BM * stride), 1, 1};  // traversed span: BM elements at stride `stride`
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
  if (res) return launch_gemm_kernel<BN, stb::EPI_ADD_RES, true>(maps, p, st, "conv3x3_nhwc");
  return launch_gemm_kernel<BN, stb::EPI_STORE, true>(maps, p, st, "conv3x3_nhwc");
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
    if (int r = set_smem<stb::conv_in_3ch_mma_kernel<256>>(SMEM)) return r;
    if (int r = set_smem<stb::conv_in_3ch_mma_kernel<128>>(SMEM)) return r;
    if (int r = set_smem<stb::conv_in_3ch_mma_kernel<64>>(SMEM)) return r;
    if (C == 256) stb::conv_in_3ch_mma_kernel<256><<<grid, 256, SMEM, st>>>(px, wt, bs, o, B, H, W);
    else if (C == 128) stb::conv_in_3ch_mma_kernel<128><<<grid, 256, SMEM, st>>>(px, wt, bs, o, B, H, W);
    else stb::conv_in_3ch_mma_kernel<64><<<grid, 256, SMEM, st>>>(px, wt, bs, o, B, H, W);
    STB_LAUNCH_CHECK("conv_in_3ch_mma");
    return 0;
  }
  const long long total = (long long)B * H * W * (C / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 8);
  const int smem = (C * 27 + C) * (int)sizeof(float);
  if (int r = set_smem<stb::conv_in_3ch_kernel>(512 * 28 * (int)sizeof(float))) return r;
  stb::conv_in_3ch_kernel<<<grid, 256, smem, st>>>(static_cast<const __nv_bfloat16*>(pixels), static_cast<const __nv_bfloat16*>(w),
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
