// kp_api.cu -- the C ABI of include/karpsolve.h: device memory, transfers, kernel launches, result assembly.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <dlfcn.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "kp_consolidate.cuh"
#include "kp_gosort_host.hpp"
#include "kp_prep.hpp"

#define CK(call)                                                                                     \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess) {                                                                         \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e_);                                   \
      return KP_ERR_CUDA;                                                                            \
    }                                                                                                \
  } while (0)

struct Arena {  // device allocations of one upload, bump-allocated from chunks that survive across uploads
  struct Chunk {
    char* base;
    size_t cap, used;
  };
  std::vector<Chunk> chunks;
  size_t bytes = 0;  // requested by the current upload
  template <class T>
  cudaError_t alloc(T** out, size_t n) {
    size_t need = (std::max<size_t>(n, 1) * sizeof(T) + 255) & ~(size_t)255;
    bytes += need;
    for (auto& c : chunks)
      if (c.cap - c.used >= need) {
        *out = (T*)(c.base + c.used);
        c.used += need;
        return cudaSuccess;
      }
    size_t cap = std::max<size_t>(need, (size_t)32 << 20);
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, cap);
    if (e != cudaSuccess) return e;
    chunks.push_back(Chunk{(char*)p, cap, need});
    *out = (T*)p;
    return cudaSuccess;
  }
  // start a new upload: keep the memory; if the last upload needed several chunks, replace them by one that fits
  void reset() {
    if (chunks.size() > 1) {
      size_t total = bytes + bytes / 4;
      destroy();
      void* p = nullptr;
      if (cudaMalloc(&p, total) == cudaSuccess) chunks.push_back(Chunk{(char*)p, total, 0});
    }
    for (auto& c : chunks) c.used = 0;
    bytes = 0;
  }
  void destroy() {
    for (auto& c : chunks) cudaFree(c.base);
    chunks.clear();
  }
};

// One uploaded problem == one Scheduler instance (scheduler.go:116-184): its tables in HBM and what the host needs to
// assemble the result.  A handle owns one for kp_solve / kp_consolidate and several for kp_solve_batch.
struct Instance {
  KpDev dev;
  HostTables host;
  bool resident = false;
  // copies of problem scalars needed to assemble results
  int64_t P = 0;
  int n_keys = 0, n_resources = 0, n_its = 0, hostname_key = -1, n_nodes = 0;
  std::vector<int> key_nvalues;
  std::vector<int64_t> tmpl_remaining0;
  // pod sort inputs (device)
  int32_t* d_pod_class = nullptr;
  int64_t* d_pod_creation = nullptr;
  uint64_t *d_uid_hi = nullptr, *d_uid_lo = nullptr;
  int64_t* d_class_rank = nullptr;
  int32_t *d_nsig_rs = nullptr, *d_nsig_tolset = nullptr;
  int64_t* d_rv_req = nullptr;
  int strict_undefined = 0;
  // state the solve mutates: pristine device copies, restored device-to-device before every solve (no host memory,
  // no allocation and no synchronisation sits between the first and the last kernel of a solve)
  struct Reset {
    void* dst;
    const void* src;
    size_t bytes;
  };
  std::vector<Reset> resets;
  const int32_t* d_host_cnt_nodes = nullptr;
  const uint32_t* d_host_pop_nodes = nullptr;
  // NewQueue radix sort buffers
  void *sort_keys_a = nullptr, *sort_keys_b = nullptr, *sort_tmp = nullptr;
  int32_t* sort_perm_b = nullptr;
  size_t sort_tmp_bytes = 0;
  bool lean = false;  // no topology group / bound / minValues / reservation: the lean instantiation of the solver serves it
  bool cohort = false;  // the queue holds long runs of identical pods: the cohort instantiation serves it (kp_wsolve.cuh cohort_try)
  // Results.TruncateInstanceTypes inside the solve (kp_problem.max_instance_types > 0): price lists + per-warp sort scratch
  int max_its = 0;
  PriceTabs price_tabs{};
  double* trunc_key = nullptr;
  int32_t* trunc_val = nullptr;
  unsigned long long* trunc_bits = nullptr;
  uint8_t* d_dropped = nullptr;
  // shared-memory plan of the solve CTA (plan_solve)
  int CS = 0, CQ = 0, CR = 0, tk_groups = 0;  // tk_groups: groups on the topology key whose state is on chip
  size_t smem = 0;
  // global counter table of a sharded job (kp_comm_set_counter_layout): dom_cnt index of each slot this instance owns
  int32_t* d_slot_src = nullptr;
  int64_t n_slots = 0, slot_off = 0;
};

// NCCL is bound at run time (dlopen), so the library loads -- and every single-GPU entry point works -- on a box
// without it; only kp_comm_init needs it.  Under torch the already-loaded libnccl.so.2 is the one that resolves.
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ struct KpNcclId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
struct KpNcclId {
  char internal[128];
};
static NcclApi g_nccl;
static bool nccl_load(std::string& err) {
  if (g_nccl.lib) return true;
  void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) {
    err = std::string("NCCL is not available: ") + dlerror();
    return false;
  }
  g_nccl.GetUniqueId = (int (*)(void*))dlsym(lib, "ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(void**, int, KpNcclId, int))dlsym(lib, "ncclCommInitRank");
  g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(lib, "ncclAllReduce");
  g_nccl.CommDestroy = (int (*)(void*))dlsym(lib, "ncclCommDestroy");
  g_nccl.GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.CommDestroy) {
    err = "libnccl lacks an expected symbol";
    return false;
  }
  g_nccl.lib = lib;
  return true;
}

struct kp_handle {
  int device = 0;
  int n_sm = 132;  // SMs of the device (kp_create); 132 on an H100 SXM
  cudaStream_t stream = nullptr;
  std::string err;
  Arena arena;
  // the instances of the last upload and the entry point that made it: kp_upload (also kp_solve, kp_feasibility and
  // kp_consolidate) uploads one, kp_upload_batch / kp_solve_batch any number
  enum Uploader { NONE, SINGLE, BATCH } uploaded = NONE;
  std::vector<std::unique_ptr<Instance>> insts;
  KpDev* d_devs = nullptr;  // [devs_cap] device copies of the instances' pointer blocks (run_solve)
  int4* d_plan = nullptr;   // [devs_cap] {CS, CQ, CR, tk_groups}
  int devs_cap = 0;
  // sharded job: NCCL communicator + the global topology-domain counter table (device resident, all-reduced per solve)
  void* comm = nullptr;
  int comm_rank = 0, comm_world = 1;
  int32_t* d_gcnt = nullptr;
  int64_t gcnt_slots = 0;
  float allreduce_ms = 0;
  cudaEvent_t ev3 = nullptr;
  kp_stats stats{};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

template <class T>
static cudaError_t up(kp_handle* h, const T** dst, const std::vector<T>& v) {
  T* p;
  cudaError_t e = h->arena.alloc(&p, v.size());
  if (e != cudaSuccess) return e;
  if (!v.empty()) e = cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, h->stream);
  h->stats.bytes_h2d += v.size() * sizeof(T);
  *dst = p;
  return e;
}
// a table the solve mutates: the upload goes to a pristine copy, the working copy is restored from it per solve
template <class T>
static cudaError_t up_mut(kp_handle* h, Instance& in, T** dst, const std::vector<T>& v) {
  const T* init;
  cudaError_t e = up(h, &init, v);
  if (e != cudaSuccess) return e;
  T* work;
  e = h->arena.alloc(&work, v.size());
  if (e != cudaSuccess) return e;
  if (!v.empty()) in.resets.push_back(Instance::Reset{work, init, v.size() * sizeof(T)});
  *dst = work;
  return cudaSuccess;
}
template <class T>
static cudaError_t up_raw(kp_handle* h, T** dst, const T* src, size_t n) {
  T* p;
  cudaError_t e = h->arena.alloc(&p, n);
  if (e != cudaSuccess) return e;
  if (n) e = cudaMemcpyAsync(p, src, n * sizeof(T), cudaMemcpyHostToDevice, h->stream);
  h->stats.bytes_h2d += n * sizeof(T);
  *dst = p;
  return e;
}
template <class T>
static cudaError_t zeros(kp_handle* h, T** dst, size_t n) {
  T* p;
  cudaError_t e = h->arena.alloc(&p, n);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(p, 0, std::max<size_t>(n, 1) * sizeof(T), h->stream);
  *dst = p;
  return e;
}

__global__ void k_sort_keys(const int32_t* pod_class, const int64_t* class_rank, const int32_t* perm, int64_t n,
                            int64_t* out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = class_rank[pod_class[perm[i]]];
}
template <class T>
__global__ void k_gather(const T* src, const int32_t* perm, int64_t n, T* out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[perm[i]];
}
__global__ void k_fill_i32(int32_t* p, int64_t n, int32_t v) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// slot i of an instance's share of the global counter table <- its dom_cnt entry
__global__ void k_scatter_counts(const int32_t* dom_cnt, const int32_t* slot_src, int64_t n, int32_t* out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = dom_cnt[slot_src[i]];
}

__global__ void k_slot_kats(const int64_t* val_int, uint64_t isint, uint64_t univ, const kp_slot_case* cs, int n, kp_slot_out* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const KeyInfo ki{val_int, isint, univ};
  const kp_slot_case c = cs[i];
  const Slot a{c.flags_a, c.mask_a, c.gte_a, c.lte_a}, b{c.flags_b, c.mask_b, c.gte_b, c.lte_b};
  kp_slot_out o;
  memset(&o, 0, sizeof(o));
  if (slot_present(a) && slot_present(b)) {
    const Slot r = slot_intersection(ki, a, b);
    o.mask = r.m;
    o.gte = r.gte;
    o.lte = r.lte;
    o.flags = r.f;
    o.op = slot_op(r);
    o.has_intersection = slot_has_intersection(ki, a, b);
  }
  o.has_value = c.value >= 0 ? slot_has(ki, a, c.value) : 0;
  o.compatible = slot_compatible(ki, a, b, c.well_known != 0, c.allow_undefined != 0);
  out[i] = o;
}

static int kp_consolidate_impl(kp_handle* h, const kp_problem* p, const kp_consol_input* in, int64_t deadline_ms,
                               kp_consol_result* out);
extern "C" {

int kp_debug_slot_algebra(kp_handle* h, const int64_t* value_int, uint64_t value_is_int, uint64_t universe,
                          const kp_slot_case* cases, int32_t n, kp_slot_out* out) {
  if (n < 0 || !value_int || (n > 0 && (!cases || !out))) return h->err = "kp_debug_slot_algebra: bad arguments", KP_ERR_INVALID;
  cudaSetDevice(h->device);
  int64_t* dv = nullptr;
  kp_slot_case* dc = nullptr;
  kp_slot_out* dout = nullptr;
  CK(cudaMalloc(&dv, 64 * 8));
  CK(cudaMalloc(&dc, sizeof(kp_slot_case) * std::max(n, 1)));
  CK(cudaMalloc(&dout, sizeof(kp_slot_out) * std::max(n, 1)));
  CK(cudaMemcpy(dv, value_int, 64 * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dc, cases, sizeof(kp_slot_case) * n, cudaMemcpyHostToDevice));
  if (n > 0) k_slot_kats<<<(n + 127) / 128, 128, 0, h->stream>>>(dv, value_is_int, universe, dc, n, dout);
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  CK(cudaMemcpy(out, dout, sizeof(kp_slot_out) * n, cudaMemcpyDeviceToHost));
  cudaFree(dv);
  cudaFree(dc);
  cudaFree(dout);
  return KP_OK;
}
}

extern "C" {

#define KP_TRUNC_BLOCKS 132  // k_truncate_claims: one block per H100 SM, 4 warps per block, one claim per warp at a time
int kp_version(void) { return KP_ABI_VERSION; }

// sort.Slice order of a key array (host; no device needed): see kp_gosort_host.hpp
int kp_go_sort_f64(const double* keys, int32_t n, int32_t* perm_out) {
  if (n < 0 || (n > 0 && (!keys || !perm_out))) return KP_ERR_INVALID;
  host_go_sort(keys, n, perm_out);
  return KP_OK;
}
int kp_go_sort_i64(const int64_t* keys, int32_t n, int32_t* perm_out) {
  if (n < 0 || (n > 0 && (!keys || !perm_out))) return KP_ERR_INVALID;
  host_go_sort(keys, n, perm_out);
  return KP_OK;
}

int kp_create(int device, kp_handle** out) {
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return KP_ERR_CUDA;  // no CPU fallback
  kp_handle* h = new kp_handle();
  if (device < 0) cudaGetDevice(&device);
  h->device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreate(&h->stream) != cudaSuccess) {
    delete h;
    return KP_ERR_CUDA;
  }
  cudaEventCreate(&h->ev0);
  cudaEventCreate(&h->ev1);
  cudaEventCreate(&h->ev3);
  cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device);
  cudaDeviceSetLimit(cudaLimitStackSize, 16384);  // pdqsort emulation recurses (log n deep)
  *out = h;
  return KP_OK;
}

void kp_destroy(kp_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  h->arena.destroy();
  cudaFree(h->d_devs);
  cudaFree(h->d_plan);
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  if (h->ev3) cudaEventDestroy(h->ev3);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

const char* kp_last_error(kp_handle* h) { return h ? h->err.c_str() : "no handle"; }

int kp_get_stats(kp_handle* h, kp_stats* out) {
  *out = h->stats;
  return KP_OK;
}

static int upload_tables(kp_handle* h, Instance& in, const kp_problem* p, int cmax_hint) {
  HostTables& t = in.host;
  KpDev& d = in.dev;
  memset(&d, 0, sizeof(d));
  d.K = t.K;
  d.R = t.R;
  d.T = t.T;
  d.ITW = t.ITW;
  d.N = t.N;
  d.X = t.X;
  d.G = t.G;
  d.GH = t.GH;
  d.E = t.E;
  d.D = t.D;
  d.n_reqsets = t.n_reqsets;
  d.n_taintsets = t.n_taintsets;
  d.n_tolsets = t.n_tolsets;
  d.has_bounds = t.has_bounds;
  d.hostname_key = t.hostname_key;
  d.nodes_res = t.nodes_res;
  d.n_rv = t.n_rv;
  d.stable_order = p->claim_order_mode == 1;
  CK(up(h, &d.key_wellknown, t.key_wellknown));
  CK(up(h, &d.key_univ, t.key_univ));
  CK(up(h, &d.val_int, t.val_int));
  CK(up(h, &d.val_isint, t.val_isint));
  CK(up(h, &d.rs_flags, t.rs_flags));
  CK(up(h, &d.rs_mask, t.rs_mask));
  CK(up(h, &d.rs_gte, t.rs_gte));
  CK(up(h, &d.rs_lte, t.rs_lte));
  CK(up(h, &d.tol_ok, t.tol_ok));
  CK(up(h, &d.itv_off, t.itv_off));
  CK(up(h, &d.itv, t.itv));
  CK(up(h, &d.it_nokey, t.it_nokey));
  CK(up(h, &d.it_dne, t.it_dne));
  CK(up(h, &d.it_nonempty, t.it_nonempty));
  CK(up(h, &d.it_valid, t.it_valid));
  CK(up(h, &d.ge_off, t.ge_off));
  CK(up(h, &d.ge_vals, t.ge_vals));
  CK(up(h, &d.ge_bits, t.ge_bits));
  d.n_ge = (int)t.ge_vals.size();
  d.n_itv = std::max(t.itv_off[d.K], 1);
  CK(up(h, &d.off_slots, t.off_slots));
  CK(up(h, &d.off_keys, t.off_keys));
  CK(up(h, &d.offset_bits, t.offset_bits));
  CK(up(h, &d.it_capacity, t.it_capacity));
  CK(up(h, &d.tmpl_rs, t.tmpl_rs));
  CK(up(h, &d.tmpl_taintset, t.tmpl_taintset));
  CK(up(h, &d.tmpl_its_raw, t.tmpl_its_raw));
  CK(zeros(h, &d.tmpl_its, t.tmpl_its_raw.size()));
  CK(up(h, &d.tmpl_daemon, t.tmpl_daemon));
  CK(up_mut(h, in, &d.tmpl_remaining, t.tmpl_remaining));
  CK(up(h, &d.tmpl_limit_present, t.tmpl_limit_present));
  CK(up(h, &d.host_rules, t.host_rules));
  CK(up(h, &d.cls_req, t.cls_req));
  CK(up(h, &d.cls_rs, t.cls_rs));
  CK(up(h, &d.cls_tolset, t.cls_tolset));
  CK(up(h, &d.cls_relax, t.cls_relax));
  d.mv_strict = t.min_values_strict ? 1 : 0;
  CK(up(h, &d.tmpl_mv_off, t.tmpl_mv_off));
  CK(up(h, &d.tmpl_mv_key, t.tmpl_mv_key));
  CK(up(h, &d.tmpl_mv_need, t.tmpl_mv_need));
  CK(up(h, &d.mv_val_off, t.mv_val_off));
  CK(up(h, &d.mv_masks, t.mv_masks));
  CK(up(h, &d.cls_match, t.cls_match));
  CK(up(h, &d.cls_rec, t.cls_rec));
  {  // class rows (one indirection less on the per-pod path): the class plan of kp_prep.cpp in the device's encoding
    if (t.N > 64) return h->err = "more than 64 NodePools", KP_ERR_CAPACITY;
    const ClassPlan& plan = t.plan;
    const bool domain_fp = !getenv("KP_NO_DOMAIN_FP");
    const size_t XK = (size_t)std::max(t.X, 1) * t.K;
    std::vector<int64_t> pg(XK, 0), pl(XK, 0), sg(XK, 0), sl(XK, 0);
    std::vector<ClsLane> rows((size_t)std::max(t.X, 1) * 32);
    memset(rows.data(), 0, rows.size() * sizeof(ClsLane));
    for (int x = 0; x < t.X; x++) {
      // tkinfo: the accepted-signature id if it has a bit in amask, and the shortcuts; a chain class has neither
      const int nm = t.cls_match_off[x + 1] - t.cls_match_off[x], nr = t.cls_rec_off[x + 1] - t.cls_rec_off[x];
      const int asig = plan.asig[x];
      int tki = 0xff;
      if (!plan.chain[x]) {
        tki = asig < 64 ? asig | TKI_ABIT : 0xff;
        if (plan.fast[x] && asig < 64) tki |= TKI_FAST;
        if (plan.fp[x] && nm <= KP_PG && nr <= KP_PG && domain_fp) tki |= TKI_FP | (plan.has_tk[x] ? TKI_TK : 0);
        if (nm + nr > 0) tki |= TKI_TOPO;
      }
      const int32_t hdr[KP_HDR] = {t.cls_tolset[x], t.cls_rv[x], t.cls_match_off[x], t.cls_match_off[x + 1], t.cls_rec_off[x],
                                   t.cls_rec_off[x + 1], plan.fsig[x], plan.nsig[x], plan.hchk_off[x], plan.hchk_off[x + 1]};
      const size_t a = (size_t)t.cls_rs[x] * t.K, b = (size_t)t.cls_strict_rs[x] * t.K;
      for (int l = 0; l < 32; l++) {
        ClsLane& c = rows[(size_t)x * 32 + l];
        if (l < t.K) {
          c.pod_m = t.rs_mask[a + l];
          c.strict_m = t.rs_mask[b + l];
          c.pod_f = t.rs_flags[a + l];
          c.strict_f = t.rs_flags[b + l];
          pg[(size_t)x * t.K + l] = t.rs_gte[a + l];
          pl[(size_t)x * t.K + l] = t.rs_lte[a + l];
          sg[(size_t)x * t.K + l] = t.rs_gte[b + l];
          sl[(size_t)x * t.K + l] = t.rs_lte[b + l];
        }
        if (l < t.R) c.req = t.cls_req[(size_t)x * t.R + l];
        if (l < KP_HDR) c.hdr = hdr[l];
        if (l == KP_HDR + 2) c.hdr = (int32_t)(plan.tok[x] & 0xffffffffull);
        if (l == KP_HDR + 3) c.hdr = (int32_t)(plan.tok[x] >> 32);
        if (l == KP_HDR + 4) c.hdr = t.cls_relax[x];
        if (l == KP_HDR + 5) c.hdr = tki;
        if (l == KP_HDR + 10) c.hdr = t.cls_vol_next[x];
        if (l >= KP_HDR + 6 && l <= KP_HDR + 9 && p->n_hostports > 0 && p->class_hostports) {
          const uint64_t ports = p->class_hostports[x];
          uint64_t conf = 0;
          for (uint64_t m = ports; m;) {
            const int i = __builtin_ctzll(m);
            m &= m - 1;
            conf |= p->hostport_conflicts[i];
          }
          const uint64_t v = l < KP_HDR + 8 ? ports : conf;
          c.hdr = (int32_t)(((l - KP_HDR) & 1) ? (v >> 32) : (v & 0xffffffffull));
        }
      }
    }
    std::vector<int4> hchk;
    for (const HostCheck& c : plan.hchk) hchk.push_back(int4{c.row, c.type | (c.self << 8), c.max_skew, c.g});
    if (hchk.empty()) hchk.push_back(int4{0, 0, 0, 0});
    std::vector<int32_t> nsig_rs = plan.nsig_rs, nsig_tolset = plan.nsig_tolset;
    if (nsig_rs.empty()) {
      nsig_rs.push_back(0);
      nsig_tolset.push_back(-1);
    }
    d.tk_key = plan.tk_key;
    d.n_fsig = plan.n_fsig;
    d.n_nsig = (int)plan.nsig_rs.size();
    d.EW = (t.E + 31) / 32;
    in.strict_undefined = plan.strict_undefined ? 1 : 0;
    std::vector<int64_t> rv_req((size_t)std::max(t.n_rv, 1) * t.R, 0);
    for (int x = 0; x < t.X; x++)
      for (int r = 0; r < t.R; r++) rv_req[(size_t)t.cls_rv[x] * t.R + r] = t.cls_req[(size_t)x * t.R + r];
    {
      const int32_t *a_, *b_;
      const int64_t* c_;
      CK(up(h, &a_, nsig_rs));
      CK(up(h, &b_, nsig_tolset));
      CK(up(h, &c_, rv_req));
      in.d_nsig_rs = const_cast<int32_t*>(a_);
      in.d_nsig_tolset = const_cast<int32_t*>(b_);
      in.d_rv_req = const_cast<int64_t*>(c_);
    }
    CK(up(h, &d.cls_hchk, hchk));
    std::vector<uint32_t> nact(std::max(d.EW, 1), 0);
    for (int n = 0; n < t.E; n++)
      if (t.node_flags[n] & KP_NODE_SCHEDULABLE) nact[n >> 5] |= 1u << (n & 31);
    CK(up_mut(h, in, &d.nactive, nact));
    d.ESW = (d.EW + 31) / 32;
    CK(zeros(h, &d.nfit_sum, (size_t)std::max(t.n_rv, 1) * std::max(d.ESW, 1)));
    CK(zeros(h, &d.nstat_sum, (size_t)std::max(d.n_nsig, 1) * std::max(d.ESW, 1)));
    CK(zeros(h, &d.nfit, (size_t)std::max(t.n_rv, 1) * std::max(d.EW, 1)));
    CK(zeros(h, &d.nstat, (size_t)std::max(d.n_nsig, 1) * std::max(d.EW, 1)));
    CK(up(h, &d.cls_lane, rows));
    CK(up(h, &d.cp_g, pg));
    CK(up(h, &d.cp_l, pl));
    CK(up(h, &d.cs_g, sg));
    CK(up(h, &d.cs_l, sl));
  }
  CK(up(h, &d.groups, t.groups));
  CK(up(h, &d.filter_rs, t.filter_rs));
  CK(up_mut(h, in, &d.dom_cnt, t.dom_cnt));
  CK(up_mut(h, in, &d.dom_reg, t.dom_reg));
  CK(up_mut(h, in, &d.dom_pop, t.dom_pop));
  d.tk_slot = nullptr;  // (on chip, set by k_wsolve_batch only)
  d.tk_reg = d.tk_pop = nullptr;
  d.tk_cnt = nullptr;
  d.tk_nv = t.plan.tk_key >= 0 ? 64 - __builtin_clzll(t.key_univ[t.plan.tk_key] | 1ull) : 0;  // value ids lie below
  d.n_lazy = 0;
  for (int32_t b : t.g_born) d.n_lazy += b == 0;
  CK(up_mut(h, in, &d.g_born, t.g_born));
  CK(up_mut(h, in, &d.g_birth, t.g_birth));
  CK(up(h, &d.cls_lazy_off, t.cls_lazy_off));
  CK(up(h, &d.cls_lazy, t.cls_lazy));
  CK(up_mut(h, in, &d.g_anypop, t.g_anypop));
  CK(up(h, &d.node_taintset, t.node_taintset));
  CK(up(h, &d.node_flags, t.node_flags));
  CK(up_mut(h, in, &d.node_rem, t.node_rem));
  CK(up_mut(h, in, &d.node_rem_present, t.node_rem_present));
  CK(up_mut(h, in, &d.node_sflags, t.node_sflags));
  CK(up_mut(h, in, &d.node_smask, t.node_smask));
  CK(up_mut(h, in, &d.node_sgte, t.node_sgte));
  CK(up_mut(h, in, &d.node_slte, t.node_slte));
  CK(zeros(h, &d.node_npods, (size_t)std::max(t.E, 1)));
  // claims
  d.Cmax = cmax_hint;
  size_t C = (size_t)d.Cmax;
  CK(zeros(h, &d.c_tmpl, C));
  CK(zeros(h, &d.c_npods, C));
  CK(zeros(h, &d.c_req, C * t.R));
  CK(zeros(h, &d.c_sflags, C * t.K));
  CK(zeros(h, &d.c_smask, C * t.K));
  CK(zeros(h, &d.c_sgte, C * t.K));
  CK(zeros(h, &d.c_slte, C * t.K));
  CK(zeros(h, &d.c_its, C * t.ITW));
  CK(zeros(h, &d.c_j, C * t.R));
  CK(zeros(h, &d.order, C));
  CK(zeros(h, &d.cnt_at, C));
  CK(zeros(h, &d.pmask, C));
  CK(zeros(h, &d.amask, C));
  CK(zeros(h, &d.c_dom, C));
  // host ports
  d.n_hostports = p->n_hostports > 0 ? p->n_hostports : 0;
  if (d.n_hostports > 64) return h->err = "more than 64 distinct host ports", KP_ERR_CAPACITY;
  if (d.n_hostports > 0 && !p->hostport_conflicts) return h->err = "hostport_conflicts is null", KP_ERR_INVALID;
  {
    std::vector<unsigned long long> np(std::max(t.E, 1), 0ull), tp(std::max(t.N, 1), 0ull);
    for (int n = 0; n < t.E; n++)
      if (d.n_hostports && p->node_hostports) np[n] = p->node_hostports[n];
    for (int n = 0; n < t.N; n++)
      if (d.n_hostports && p->tmpl_hostports) tp[n] = p->tmpl_hostports[n];
    CK(up_mut(h, in, &d.node_ports, np));
    CK(up(h, &d.tmpl_ports, tp));
    CK(zeros(h, &d.c_ports, C));
  }
  // reserved capacity
  d.n_rsv = t.n_rsv;
  d.rsv_strict = t.rsv_strict ? 1 : 0;
  d.rsv_sets = 0;
  {
    std::vector<int32_t> sr(std::max(t.D, 1), -1);
    for (int dd = 0; dd < t.D && dd < (int)t.set_rsv.size(); dd++) {
      sr[dd] = t.set_rsv[dd];
      if (sr[dd] >= 0) d.rsv_sets |= 1u << dd;
    }
    CK(up(h, &d.set_rsv, sr));
    std::vector<int32_t> cap0 = t.rsv_cap0;
    if (cap0.empty()) cap0.push_back(0);
    CK(up_mut(h, in, &d.rsv_cap, cap0));
    CK(zeros(h, &d.c_rsv, C));
    d.rsv_ct_key = p->reservation_capacity_type_key;
    d.rsv_reserved_val = p->reservation_reserved_value;
    d.rsv_id_key = p->reservation_id_key;
    memset(d.rsv_val_of, 0, sizeof(d.rsv_val_of));
    if (t.n_rsv > 0) {
      if (d.rsv_ct_key < 0 || d.rsv_ct_key >= t.K || d.rsv_id_key < 0 || d.rsv_id_key >= t.K || !p->reservation_value ||
          d.rsv_reserved_val < 0 || d.rsv_reserved_val >= 64)
        return h->err = "reserved offerings need reservation_capacity_type_key / reservation_id_key / reservation_value", KP_ERR_INVALID;
      for (int i = 0; i < t.n_rsv; i++) {
        if (p->reservation_value[i] < 0 || p->reservation_value[i] >= 64) return h->err = "reservation_value out of range", KP_ERR_INVALID;
        d.rsv_val_of[i] = 1ull << p->reservation_value[i];
      }
    }
  }
  d.tmpl_all = t.N >= 64 ? ~0ull : ((1ull << t.N) - 1);
  d.H = t.E + d.Cmax;
  d.GHS = std::max(t.GH, 1);
  CK(zeros(h, &d.host_cnt, (size_t)d.GHS * d.H));
  {  // initial counts of the existing nodes, host-major like the table itself: rows [0, E)
    std::vector<int32_t> tr((size_t)std::max(t.E, 1) * d.GHS, 0);
    for (int r = 0; r < t.GH; r++)
      for (int n = 0; n < t.E; n++) tr[(size_t)n * d.GHS + r] = t.host_cnt_nodes[(size_t)r * t.E + n];
    CK(up(h, &in.d_host_cnt_nodes, tr));
  }
  d.HW = (d.H + 31) / 32;
  CK(zeros(h, &d.host_pop, (size_t)std::max(t.GH, 1) * d.HW));
  {  // presence bits of the existing nodes: words [0, ceil(E/32)) of every row
    const int ew = (t.E + 31) / 32;
    std::vector<uint32_t> bits((size_t)std::max(t.GH, 1) * std::max(ew, 1), 0);
    for (int r = 0; r < t.GH; r++)
      for (int n = 0; n < t.E; n++)
        if (t.host_cnt_nodes[(size_t)r * t.E + n] > 0) bits[(size_t)r * ew + (n >> 5)] |= 1u << (n & 31);
    CK(up(h, &in.d_host_pop_nodes, bits));
  }
  CK(zeros(h, &d.n_claims, 1));
  CK(zeros(h, &d.counters, KP_NCOUNTERS));
  CK(zeros(h, &d.status, 1));
  return KP_OK;
}

// stack of state the solve mutates, so kp_solve_resident can be re-run on the same upload
static int reset_dynamic(kp_handle* h, Instance& in) {
  HostTables& t = in.host;
  KpDev& d = in.dev;
  for (auto& r : in.resets) CK(cudaMemcpyAsync(r.dst, r.src, r.bytes, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemsetAsync(d.node_npods, 0, (size_t)std::max(t.E, 1) * 4, h->stream));
  size_t C = (size_t)d.Cmax;
  CK(cudaMemsetAsync(d.c_npods, 0, C * 4, h->stream));
  CK(cudaMemsetAsync(d.pmask, 0, C * sizeof(ulonglong2), h->stream));
  CK(cudaMemsetAsync(d.amask, 0, C * 8, h->stream));
  CK(cudaMemsetAsync(d.c_rsv, 0, C * 8, h->stream));
  if (in.d_dropped) CK(cudaMemsetAsync(in.d_dropped, 0, C, h->stream));
  CK(cudaMemsetAsync(d.host_cnt, 0, (size_t)d.GHS * d.H * 4, h->stream));
  if (t.E && t.GH)  // initial hostname-group counts of the existing nodes: the first E host rows
    CK(cudaMemcpyAsync(d.host_cnt, in.d_host_cnt_nodes, (size_t)t.E * d.GHS * 4, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemsetAsync(d.host_pop, 0, (size_t)std::max(t.GH, 1) * d.HW * 4, h->stream));
  if (t.E && t.GH) {
    const size_t ew = (size_t)(t.E + 31) / 32;
    CK(cudaMemcpy2DAsync(d.host_pop, (size_t)d.HW * 4, in.d_host_pop_nodes, ew * 4, ew * 4, t.GH,
                         cudaMemcpyDeviceToDevice, h->stream));
  }
  CK(cudaMemsetAsync(d.n_claims, 0, 4, h->stream));
  CK(cudaMemsetAsync(d.counters, 0, 128, h->stream));
  CK(cudaMemsetAsync(d.status, 0, 4, h->stream));
  CK(cudaMemsetAsync(d.last_len, 0, (size_t)std::max<int64_t>(in.P, 1) * 4, h->stream));
  return KP_OK;
}

// shared-memory bytes of the read-only tables a kernel stages next to `fixed` bytes of its own (0 = leave them in L2)
static int plan_tables(const KpDev& d, size_t fixed, size_t budget) {
  const size_t tb = kp_tab_bytes(d);
  return (fixed + tb <= budget && tb <= 110 * 1024) ? (int)tb : 0;
}

// Host-side plan of the solver CTA; it depends on the upload and the KP_* knobs only.  Shared memory (SolveSmem) holds
// the pointer block, the staged tables and, when they fit, the hot claim rows of the first CQ claims, the cold ones of
// the first CR <= CQ, and the claim order, template ids and failure bitmaps of the first CS claims.
static void plan_solve(Instance& in) {
  KpDev& d = in.dev;
  const size_t budget = 224 * 1024;
  d.tab_bytes = plan_tables(d, SolveSmem(d, 0, 0, 0, 0, 0).tab, budget);
  auto layout = [&](int CS, int CQ, int CR) { return SolveSmem(d, d.tab_bytes, CS, CQ, CR, in.tk_groups); };
  const bool dom_fp = std::any_of(in.host.plan.fp.begin(), in.host.plan.fp.end(), [](uint8_t f) { return f != 0; });
  // The topology-key group state (every domain-fast-path pod reads it in domain_mask and writes it in topo_record_fast)
  // goes first when it takes at most 64 KB: C3's 1 000 zone groups with 4 zones take 44 KB with the slot map.
  in.tk_groups = 0;
  if (dom_fp && !in.cohort && d.tk_key >= 0 && d.tk_nv > 0 && d.tk_nv <= 64) {
    int ntk = 0;
    for (const KpGroup& G : in.host.groups) ntk += G.key == d.tk_key;
    const SolveSmem L(d, d.tab_bytes, 0, 0, 0, ntk);
    if (ntk > 0 && L.s_req - L.tk_slot <= 64 * 1024) in.tk_groups = ntk;
  }
  // claim rows: hot = requests + threshold row, cold = requirement slots + instance-type words.  The rows get what whole
  // rows of up to 512 claims take within half the budget; the small arrays keep the rest.
  int CR = std::min(d.Cmax, 512);
  while (CR > 0 && layout(0, CR, CR).pmask > budget / 2) CR -= 32;
  CR = std::max(CR, 0);
  const SolveSmem whole = layout(0, CR, CR);
  const size_t rows = whole.pmask - whole.s_req;
  int CQ = CR;
  // With classes on the domain fast path almost every commit is fp_fit + a store of the hot row: claims are visited
  // round-robin, so the hot rows of as many claims as possible (C3: all of them) beat whole rows of a few hundred.
  // Cold rows take what is left.
  if (dom_fp) {
    CQ = std::min((d.Cmax + 31) / 32 * 32, (int)(rows / ((size_t)d.R * 12 + 1)) / 32 * 32);
    while (CQ > 0 && layout(0, CQ, 0).pmask - whole.s_req > rows) CQ -= 32;
    CR = 0;
    while (CR + 32 <= CQ && layout(0, CQ, CR + 32).pmask - whole.s_req <= rows) CR += 32;
  }
  // ... and claim order / failure masks of the first CS claims
  int CS = 0;
  if (layout(64, CQ, CR).total <= budget) {  // the largest multiple of 32 that fits, capped at Cmax
    int lo = 64, hi = ((d.Cmax + 31) / 32) * 32;
    while (lo < hi) {
      int mid = ((lo + hi + 32) / 64) * 32;
      if (mid <= lo) mid = lo + 32;
      if (layout(mid, CQ, CR).total <= budget)
        lo = mid;
      else
        hi = mid - 32;
    }
    CS = lo;
  }
  // KP_SMEM_CAP="CS,CQ,CR,TK" (test knob): upper bounds on the plan, an empty field leaves that part as planned.  They only
  // lower it, so every capped layout is one the kernel is already handed: CS stays a multiple of 32, CR <= CQ, and a TK
  // below the number of groups on the topology key leaves their state in global memory.
  if (const char* cap = getenv("KP_SMEM_CAP")) {
    long v[4];
    bool set[4] = {false, false, false, false};
    for (int f = 0; f < 4 && cap; f++) {
      char* end;
      v[f] = std::max(0l, strtol(cap, &end, 10));
      set[f] = end != cap;
      cap = strchr(cap, ',');
      if (cap) cap++;
    }
    if (set[0]) CS = (int)std::min<long>(CS, v[0] / 32 * 32);
    if (set[1]) CQ = (int)std::min<long>(CQ, v[1]);
    if (set[2]) CR = (int)std::min<long>(CR, v[2]);
    if (set[3] && v[3] < in.tk_groups) in.tk_groups = 0;
  }
  CR = std::min(CR, CQ);
  in.lean = in.host.G == 0 && !in.host.has_bounds && !in.host.min_values_strict && in.host.n_rsv == 0 && d.n_hostports == 0 &&
            !in.host.has_vol_alts && !getenv("KP_NO_LEAN");
  if (in.host.has_vol_alts) in.cohort = false;  // (the volume-alternative instantiation exists without cohorts only)
  in.CS = CS;
  in.CQ = CQ;
  in.CR = CR;
  in.smem = layout(CS, CQ, CR).total;
  if (getenv("KP_DEBUG"))
    fprintf(stderr, "[kp] solver plan: tables %zu B, topology-key groups on chip %d, hot rows %d, cold rows %d, small arrays %d, %zu B shared\n",
            (size_t)d.tab_bytes, in.tk_groups, CQ, CR, CS, in.smem);
}

// Starts a fresh upload: the instances of either entry point are dropped and the arena is reused for the new ones.
static void begin_upload(kp_handle* h, kp_handle::Uploader by) {
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  h->insts.clear();
  h->uploaded = by;
  h->d_gcnt = nullptr;  // lived in the arena
  h->gcnt_slots = 0;
  h->arena.reset();
  h->stats = kp_stats{};
}

// Uploads p as one more instance of the handle, room for `cmax` NodeClaims.  The stats sum over the instances.
static int add_instance(kp_handle* h, const kp_problem* p, int64_t cmax) {
  h->insts.push_back(std::make_unique<Instance>());
  Instance& in = *h->insts.back();
  auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> active(p->n_nodes, 0);
  for (int i = 0; i < p->n_nodes; i++) active[i] = (p->node_flags[i] & KP_NODE_SCHEDULABLE) != 0;
  std::vector<int32_t> pending(p->pod_class, p->pod_class + p->n_pods);
  int rc = kp_prepare(p, active, {}, pending, in.host, h->err, true);
  if (rc != KP_OK) return rc;
  auto t1 = std::chrono::steady_clock::now();
  h->stats.prep_ms += std::chrono::duration<double, std::milli>(t1 - t0).count();
  in.P = p->n_pods;
  in.n_keys = p->n_keys;
  in.n_resources = p->n_resources;
  in.n_its = p->n_its;
  in.n_nodes = p->n_nodes;
  in.hostname_key = in.host.hostname_key;
  in.key_nvalues.resize(p->n_keys);
  for (int k = 0; k < p->n_keys; k++) in.key_nvalues[k] = p->key_value_off[k + 1] - p->key_value_off[k];
  if (p->n_pods >= (1ll << 31) - 2) return h->err = "more than 2^31 pods", KP_ERR_CAPACITY;
  rc = upload_tables(h, in, p, (int)cmax);
  if (rc != KP_OK) return rc;
  KpDev& d = in.dev;
  d.P = p->n_pods;
  size_t P = (size_t)p->n_pods;
  CK(up_raw(h, &in.d_pod_class, p->pod_class, P));
  d.pod_class = in.d_pod_class;
  if (p->pod_creation) {
    CK(up_raw(h, &in.d_pod_creation, p->pod_creation, P));
  } else {
    CK(zeros(h, &in.d_pod_creation, P));
  }
  CK(up_raw(h, &in.d_uid_hi, p->pod_uid_hi, P));
  CK(up_raw(h, &in.d_uid_lo, p->pod_uid_lo, P));
  const std::vector<int64_t>& rank = in.host.plan.rank;  // byCPUAndMemoryDescending (queue.go:72-108)
  CK(up_raw(h, &in.d_class_rank, rank.data(), rank.size()));
  {
    // Pods of classes that are alone in their (cpu, memory) rank stand together in the queue (byCPUAndMemoryDescending, then
    // creation time and UID, which interleave the classes of one rank): when they are at least a quarter of the queue the
    // solve runs the cohort instantiation.  KP_COHORT=1 / KP_NO_COHORT=1 force the choice.
    const int X = in.host.X;
    std::vector<int64_t> pods_of(std::max(X, 1), 0), classes_at(std::max(X, 1), 0);
    for (size_t i = 0; i < P; i++) pods_of[p->pod_class[i]]++;
    for (int x = 0; x < X; x++)
      if (pods_of[x] > 0) classes_at[rank[x]]++;
    int64_t in_runs = 0;
    for (int x = 0; x < X; x++)
      if (pods_of[x] > 1 && classes_at[rank[x]] == 1) in_runs += pods_of[x];
    in.cohort = (in_runs * 4 >= (int64_t)P && P > 0 && !getenv("KP_NO_COHORT")) || getenv("KP_COHORT");
    d.cohort = in.cohort ? 1 : 0;
  }
  in.max_its = p->max_instance_types > 0 ? p->max_instance_types : 0;
  if (in.max_its > 0) {
    const int T = p->n_its;
    const PriceLists ml = order_by_price(p, in.host);
    CK(up(h, &in.price_tabs.ml_off, ml.off));
    CK(up(h, &in.price_tabs.ml_set, ml.set));
    CK(up(h, &in.price_tabs.ml_price, ml.price));
    const size_t NW = (size_t)KP_TRUNC_BLOCKS * 4;
    CK(h->arena.alloc(&in.trunc_key, NW * std::max(T, 1)));
    CK(h->arena.alloc(&in.trunc_val, NW * std::max(T, 1)));
    CK(h->arena.alloc(&in.trunc_bits, NW * std::max((T + 63) / 64, 1)));
    CK(zeros(h, &in.d_dropped, (size_t)std::max<int64_t>(d.Cmax, 1)));
  }
  {  // NewQueue sort: key / permutation ping-pong buffers and cub's scratch, sized once per upload
    int64_t* ka;
    int64_t* kb;
    CK(h->arena.alloc(&ka, P));
    CK(h->arena.alloc(&kb, P));
    CK(h->arena.alloc(&in.sort_perm_b, P));
    in.sort_keys_a = ka;
    in.sort_keys_b = kb;
    size_t n1 = 0, n2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, n1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr,
                                    (int32_t*)nullptr, (int)std::max<size_t>(P, 1));
    cub::DeviceRadixSort::SortPairs(nullptr, n2, (const int64_t*)nullptr, (int64_t*)nullptr, (const int32_t*)nullptr,
                                    (int32_t*)nullptr, (int)std::max<size_t>(P, 1));
    in.sort_tmp_bytes = std::max(n1, n2);
    char* tmp;
    CK(h->arena.alloc(&tmp, in.sort_tmp_bytes));
    in.sort_tmp = tmp;
  }
  CK(zeros(h, &d.queue, P + 1));
  CK(zeros(h, &d.qcls, P + 1));
  CK(zeros(h, &d.last_len, P));
  CK(zeros(h, &d.pod_target, P));
  CK(zeros(h, &d.pod_error, P));
  CK(cudaStreamSynchronize(h->stream));
  auto t2 = std::chrono::steady_clock::now();
  h->stats.upload_ms += std::chrono::duration<double, std::milli>(t2 - t1).count();
  plan_solve(in);
  in.resident = true;
  return KP_OK;
}

static int upload(kp_handle* h, const kp_problem* const* problems, int n, const int64_t* cmax, kp_handle::Uploader by) {
  begin_upload(h, by);
  for (int b = 0; b < n; b++) {
    int rc = add_instance(h, problems[b], cmax[b]);
    if (rc != KP_OK) return rc;
  }
  return KP_OK;
}

// claim capacity: every pod could need its own NodeClaim; start with a generous bound and grow on demand
static int64_t cmax_guess(const kp_problem* p) {
  return std::max<int64_t>(1, std::min<int64_t>(p->n_pods, std::max<int64_t>(4096, p->n_pods / 8)));
}

int kp_upload(kp_handle* h, const kp_problem* p) {
  const int64_t cmax = cmax_guess(p);
  return upload(h, &p, 1, &cmax, kp_handle::SINGLE);
}

// NewQueue: sort pods cpu desc, mem desc, creation asc, uid asc (queue.go:37-43) into d.queue / d.qcls.
// Four LSD passes of a stable radix sort (cub), each on a gathered 64-bit key.
__global__ void k_iota(int32_t* p, int64_t n) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = (int32_t)i;
}

static int sort_queue(kp_handle* h, Instance& in) {
  KpDev& d = in.dev;
  const int64_t P = in.P;
  if (P <= 0) return KP_OK;
  const int nb = (int)((P + 255) / 256), n = (int)P;
  int32_t* perm_a = d.queue;  // passes ping-pong a -> b -> a -> b -> a: the result lands in d.queue
  int32_t* perm_b = in.sort_perm_b;
  uint64_t *ua = (uint64_t*)in.sort_keys_a, *ub = (uint64_t*)in.sort_keys_b;
  int64_t *sa = (int64_t*)in.sort_keys_a, *sb = (int64_t*)in.sort_keys_b;
  size_t tb = in.sort_tmp_bytes;
  k_iota<<<nb, 256, 0, h->stream>>>(perm_a, P);
  k_gather<<<nb, 256, 0, h->stream>>>(in.d_uid_lo, perm_a, P, ua);
  CK(cub::DeviceRadixSort::SortPairs(in.sort_tmp, tb, ua, ub, perm_a, perm_b, n, 0, 64, h->stream));
  k_gather<<<nb, 256, 0, h->stream>>>(in.d_uid_hi, perm_b, P, ua);
  CK(cub::DeviceRadixSort::SortPairs(in.sort_tmp, tb, ua, ub, perm_b, perm_a, n, 0, 64, h->stream));
  k_gather<<<nb, 256, 0, h->stream>>>(in.d_pod_creation, perm_a, P, sa);
  CK(cub::DeviceRadixSort::SortPairs(in.sort_tmp, tb, sa, sb, perm_a, perm_b, n, 0, 64, h->stream));
  k_sort_keys<<<nb, 256, 0, h->stream>>>(d.pod_class, in.d_class_rank, perm_b, P, sa);
  CK(cub::DeviceRadixSort::SortPairs(in.sort_tmp, tb, sa, sb, perm_b, perm_a, n, 0, 64, h->stream));
  k_gather<<<nb, 256, 0, h->stream>>>(d.pod_class, d.queue, P, d.qcls);
  h->stats.kernel_launches += 6;
  return KP_OK;
}

static int launch_node_cand(kp_handle* h, Instance& in) {
  KpDev& d = in.dev;
  if (d.E <= 0) return KP_OK;
  dim3 grid((d.E + 255) / 256, d.n_nsig + d.n_rv);
  k_node_cand<<<grid, 256, 0, h->stream>>>(d, in.d_nsig_rs, in.d_nsig_tolset, in.d_rv_req, in.strict_undefined);
  const int nsum = (d.n_rv + d.n_nsig) * d.ESW;
  k_node_sum<<<(nsum + 255) / 256, 256, 0, h->stream>>>(d);
  h->stats.kernel_launches += 2;
  return KP_OK;
}

// Everything of a solve in front of the solver kernel (after reset_dynamic): NewScheduler prefilter, NewQueue and the
// existing-node candidate bitmaps.  Asynchronous on the handle's stream.
static int prep_solve(kp_handle* h, Instance& in) {
  KpDev& d = in.dev;
  // NewScheduler prefilter of template instance types (scheduler.go:147)
  if (d.N > 0) {
    k_feasibility<<<(d.N * 32 + 255) / 256, 256, 0, h->stream>>>(d, nullptr, 1);
    h->stats.kernel_launches++;
  }
  int rc = sort_queue(h, in);
  if (rc != KP_OK) return rc;
  if (in.P > 0) {
    k_fill_i32<<<(int)((in.P + 255) / 256), 256, 0, h->stream>>>(d.pod_target, in.P, KP_TARGET_UNSCHEDULED);
    h->stats.kernel_launches++;
  }
  return launch_node_cand(h, in);
}

// The one collective of a NodePool-sharded job (SURVEY.md section 8(e)): every instance of this handle writes the
// counters of its topology groups into its slice of the global table, then one ncclAllReduce(sum, int32) over NVLink on
// the library's stream -- device resident from the solver kernel to the reduced table, inside the solve's event window.
static int reduce_counters(kp_handle* h) {
  if (!h->d_gcnt) return KP_OK;
  CK(cudaEventRecord(h->ev3, h->stream));
  CK(cudaMemsetAsync(h->d_gcnt, 0, (size_t)h->gcnt_slots * 4, h->stream));
  for (auto& in : h->insts)
    if (in->n_slots > 0) {
      k_scatter_counts<<<(int)((in->n_slots + 255) / 256), 256, 0, h->stream>>>(in->dev.dom_cnt, in->d_slot_src, in->n_slots,
                                                                                 h->d_gcnt + in->slot_off);
      h->stats.kernel_launches++;
    }
  if (h->comm) {
    int rc = g_nccl.AllReduce(h->d_gcnt, h->d_gcnt, (size_t)h->gcnt_slots, /*ncclInt32*/ 2, /*ncclSum*/ 0, h->comm, h->stream);
    if (rc != 0) return h->err = std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"), KP_ERR_CUDA;
  }
  return KP_OK;
}

// The solver instantiation of a launch: LEAN when every instance is lean, COHORT when any instance wants it, the
// volume-alternative one when any instance has a chain
static const void* solver_kernel(const std::vector<std::unique_ptr<Instance>>& insts) {
  bool lean = true, cohort = false, vol = false;
  for (auto& in : insts) {
    lean = lean && in->lean;
    cohort = cohort || in->cohort;
    vol = vol || in->host.has_vol_alts;
  }
  if (vol) return (const void*)k_wsolve_batch<false, false, true>;
  return lean ? (cohort ? (const void*)k_wsolve_batch<true, true> : (const void*)k_wsolve_batch<true, false>)
              : (cohort ? (const void*)k_wsolve_batch<false, true> : (const void*)k_wsolve_batch<false, false>);
}

// The consolidation instantiation of a topology-free pass: the volume-alternative one when any class of the cluster has a
// chain (it is never lean), else LEAN as the host decided
static const void* consol_kernel(bool lean, bool vol) {
  if (vol) return (const void*)k_consolidate<false, true>;
  return lean ? (const void*)k_consolidate<true> : (const void*)k_consolidate<false>;
}

// name of a solver or consolidation instantiation, for KP_DEBUG
static const char* kernel_name(const void* fn) {
  if (fn == (const void*)k_wsolve_batch<true, false>) return "k_wsolve_batch<true, false>";
  if (fn == (const void*)k_wsolve_batch<true, true>) return "k_wsolve_batch<true, true>";
  if (fn == (const void*)k_wsolve_batch<false, false>) return "k_wsolve_batch<false, false>";
  if (fn == (const void*)k_wsolve_batch<false, true>) return "k_wsolve_batch<false, true>";
  if (fn == (const void*)k_wsolve_batch<false, false, true>) return "k_wsolve_batch<false, false, true>";
  if (fn == (const void*)k_consolidate<true>) return "k_consolidate<true>";
  if (fn == (const void*)k_consolidate<false>) return "k_consolidate<false>";
  if (fn == (const void*)k_consolidate<false, true>) return "k_consolidate<false, true>";
  return "?";
}

// Scheduler.Solve of every uploaded instance, a single solve being a batch of one.  In front of the timed window: the
// dynamic state is restored and the pointer blocks and {CS, CQ, CR} plans are written to the device.  In it: the prep
// kernels per instance, ONE solver launch (one CTA per instance), truncation and the counter all-reduce.
// statuses[b]: KP_OK / KP_DEADLINE / KP_ERR_CAPACITY of instance b.
static int run_solve(kp_handle* h, int64_t deadline_ms, std::vector<int32_t>& statuses) {
  const int n = (int)h->insts.size();
  statuses.assign(n, KP_OK);
  if (n == 0) return KP_OK;
  cudaSetDevice(h->device);
  if (n > h->devs_cap) {  // device copies of the pointer blocks and plans, grown on demand
    cudaFree(h->d_devs);
    cudaFree(h->d_plan);
    h->d_devs = nullptr;
    h->d_plan = nullptr;
    h->devs_cap = 0;
    CK(cudaMalloc(&h->d_devs, sizeof(KpDev) * n));
    CK(cudaMalloc(&h->d_plan, sizeof(int4) * n));
    h->devs_cap = n;
  }
  std::vector<KpDev> devs(n);
  std::vector<int4> plan(n);
  size_t smem = 0;
  for (int b = 0; b < n; b++) {
    Instance& in = *h->insts[b];
    if (!in.resident) return h->err = "the last upload did not complete", KP_ERR_INVALID;
    in.dev.deadline_ns = deadline_ms > 0 ? deadline_ms * 1000000ll : 0;
    int rc = reset_dynamic(h, in);
    if (rc != KP_OK) return rc;
    devs[b] = in.dev;
    plan[b] = make_int4(in.CS, in.CQ, in.CR, in.tk_groups);
    smem = std::max(smem, in.smem);
  }
  CK(cudaMemcpyAsync(h->d_devs, devs.data(), sizeof(KpDev) * n, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->d_plan, plan.data(), sizeof(int4) * n, cudaMemcpyHostToDevice, h->stream));
  CK(cudaEventRecord(h->ev0, h->stream));
  h->stats.kernel_launches = 0;
  h->stats.cohort_pods = 0;
  for (auto& in : h->insts) {
    int rc = prep_solve(h, *in);
    if (rc != KP_OK) return rc;
  }
  const void* fn = solver_kernel(h->insts);
  CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  {
    void* args[] = {(void*)&h->d_devs, (void*)&h->d_plan};
    CK(cudaLaunchKernel(fn, dim3(n), dim3(64), args, smem, h->stream));
  }
  h->stats.kernel_launches++;
  for (auto& in : h->insts)
    if (in->max_its > 0) {  // Results.TruncateInstanceTypes (scheduler.go:361-379)
      k_truncate_claims<<<KP_TRUNC_BLOCKS, 128, 0, h->stream>>>(in->dev, in->price_tabs, in->max_its, in->trunc_key, in->trunc_val,
                                                                 in->trunc_bits, in->d_dropped);
      if (in->P > 0)
        k_mark_dropped<<<(int)((in->P + 255) / 256), 256, 0, h->stream>>>(in->dev.pod_target, in->dev.pod_error, in->d_dropped, in->P);
      h->stats.kernel_launches += 2;
    }
  int rc = reduce_counters(h);
  if (rc != KP_OK) return rc;
  CK(cudaEventRecord(h->ev1, h->stream));
  CK(cudaStreamSynchronize(h->stream));  // devs / plan are host vectors: the copies above must have completed
  CK(cudaGetLastError());
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  h->stats.solve_ms = ms;
  if (h->d_gcnt) cudaEventElapsedTime(&h->allreduce_ms, h->ev3, h->ev1);
  if (getenv("KP_DEBUG")) fprintf(stderr, "[kp] %d instance(s), kernel %s: step %.3f ms\n", n, kernel_name(fn), ms);
  for (int b = 0; b < n; b++) CK(cudaMemcpy(&statuses[b], h->insts[b]->dev.status, 4, cudaMemcpyDeviceToHost));
  return KP_OK;
}

// The ABI's per-key requirement layout (kp_result.claim_req_*, kp_consol_result.repl_req_*): flags, gte and lte per key,
// the mask of key k at word woff[k] of a row.  FinalizeScheduling drops the hostname requirement: it gets no mask words
// and is never materialised as a slot here.
struct ReqLayout {
  int K, hostname_key;
  std::vector<int> woff;  // [K + 1]
  explicit ReqLayout(const Instance& in) : K(in.n_keys), hostname_key(in.hostname_key), woff(in.n_keys + 1, 0) {
    for (int k = 0; k < K; k++) woff[k + 1] = woff[k] + (k == hostname_key ? 0 : (in.key_nvalues[k] + 63) / 64);
  }
  int words() const { return woff[K]; }
  // the K device requirement slots of one claim -> row r of the ABI arrays (sg / sl null: the problem has no bounds)
  void store(size_t r, const uint8_t* sf, const uint64_t* sm, const int64_t* sg, const int64_t* sl, uint8_t* flags,
             int64_t* gte, int64_t* lte, uint64_t* mask) const {
    for (int k = 0; k < K; k++) {
      const uint8_t f = sf[k];
      if (!(f & SF_PRESENT) || k == hostname_key) continue;
      flags[r * K + k] = KP_SLOT_PRESENT | ((f & SF_COMPLEMENT) ? KP_REQ_COMPLEMENT : 0) | ((f & SF_HAS_GTE) ? KP_REQ_HAS_GTE : 0) |
                         ((f & SF_HAS_LTE) ? KP_REQ_HAS_LTE : 0);
      if ((f & SF_HAS_GTE) && sg) gte[r * K + k] = sg[k];
      if ((f & SF_HAS_LTE) && sl) lte[r * K + k] = sl[k];
      if (woff[k + 1] > woff[k]) mask[r * words() + woff[k]] = sm[k];
    }
  }
};

// Result of one instance after run_solve.  Adds to the handle's download stats.
static int download(kp_handle* h, Instance& in, kp_result* out) {
  KpDev& d = in.dev;
  auto t0 = std::chrono::steady_clock::now();
  memset(out, 0, sizeof(*out));
  int32_t nclaims = 0;
  int64_t counters[16];
  CK(cudaMemcpy(&nclaims, d.n_claims, 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(counters, d.counters, 128, cudaMemcpyDeviceToHost));
  h->stats.cohort_pods += counters[5];
  if (getenv("KP_DEBUG"))
    fprintf(stderr, "[kp] slow_sorts=%lld evals=%lld commits=%lld fast_commits=%lld cohort_pods=%lld\n", (long long)counters[4],
            (long long)counters[6], (long long)counters[3], (long long)counters[9], (long long)counters[5]);
  int64_t P = in.P;
  int K = in.n_keys, R = in.n_resources, ITW = (in.n_its + 63) / 64;
  size_t C = (size_t)nclaims, c1 = C ? C : 1;
  out->n_pods = P;
  out->pod_target = (int32_t*)malloc(sizeof(int32_t) * (P ? P : 1));
  out->pod_error = (uint8_t*)malloc(P ? P : 1);
  CK(cudaMemcpy(out->pod_target, d.pod_target, P * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out->pod_error, d.pod_error, P, cudaMemcpyDeviceToHost));
  out->n_claims = nclaims;
  out->claim_template = (int32_t*)calloc(c1, 4);
  out->claim_npods = (int32_t*)calloc(c1, 4);
  out->claim_rank = (int32_t*)calloc(c1, 4);
  out->claim_reservations = (uint64_t*)calloc(c1, 8);
  CK(cudaMemcpy(out->claim_reservations, d.c_rsv, C * 8, cudaMemcpyDeviceToHost));
  out->claim_dropped = (uint8_t*)calloc(c1, 1);
  if (in.d_dropped) CK(cudaMemcpy(out->claim_dropped, in.d_dropped, C, cudaMemcpyDeviceToHost));
  out->claim_requests = (int64_t*)calloc(c1 * R, 8);
  out->it_words = ITW;
  out->claim_its = (uint64_t*)calloc(c1 * (ITW ? ITW : 1), 8);
  CK(cudaMemcpy(out->claim_template, d.c_tmpl, C * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out->claim_npods, d.c_npods, C * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out->claim_requests, d.c_req, C * R * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out->claim_its, d.c_its, C * ITW * 8, cudaMemcpyDeviceToHost));
  std::vector<int32_t> order(c1);
  CK(cudaMemcpy(order.data(), d.order, C * 4, cudaMemcpyDeviceToHost));
  for (size_t pos = 0; pos < C; pos++) out->claim_rank[order[pos]] = (int32_t)pos;
  std::vector<uint8_t> sf(c1 * K);
  std::vector<uint64_t> sm(c1 * K);
  std::vector<int64_t> sg(c1 * K), sl(c1 * K);
  CK(cudaMemcpy(sf.data(), d.c_sflags, C * K, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(sm.data(), d.c_smask, C * K * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(sg.data(), d.c_sgte, C * K * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(sl.data(), d.c_slte, C * K * 8, cudaMemcpyDeviceToHost));
  const ReqLayout L(in);
  const int MW = L.words();
  out->n_keys = K;
  out->mask_words = MW;
  out->claim_req_flags = (uint8_t*)calloc(c1 * (K ? K : 1), 1);
  out->claim_req_gte = (int64_t*)calloc(c1 * (K ? K : 1), 8);
  out->claim_req_lte = (int64_t*)calloc(c1 * (K ? K : 1), 8);
  out->claim_req_mask = (uint64_t*)calloc(c1 * (MW ? MW : 1), 8);
  for (size_t c = 0; c < C; c++)
    L.store(c, sf.data() + c * K, sm.data() + c * K, sg.data() + c * K, sl.data() + c * K, out->claim_req_flags,
            out->claim_req_gte, out->claim_req_lte, out->claim_req_mask);
  // topology counters, non-hostname groups (regular then inverse == creation order of the reference's two maps)
  HostTables& t = in.host;
  std::vector<int32_t> cnt((size_t)std::max(t.G, 1) * 64);
  CK(cudaMemcpy(cnt.data(), d.dom_cnt, cnt.size() * 4, cudaMemcpyDeviceToHost));
  // order of the reference's maps: groups of NewTopology in creation order, then the groups relaxed pods created, in
  // birth order (the ones never born do not exist), then the inverse groups
  std::vector<int32_t> birth(std::max(t.G, 1));
  CK(cudaMemcpy(birth.data(), d.g_birth, birth.size() * 4, cudaMemcpyDeviceToHost));
  std::vector<int> gorder;
  for (int g = 0; g < t.n_regular; g++)
    if (t.g_born[g]) gorder.push_back(g);
  {
    std::vector<std::pair<int, int>> born;
    for (int g = 0; g < t.n_regular; g++)
      if (!t.g_born[g] && birth[g] >= 0) born.push_back({birth[g], g});
    std::sort(born.begin(), born.end());
    for (auto& b : born) gorder.push_back(b.second);
  }
  for (int g = t.n_regular; g < t.G; g++) gorder.push_back(g);
  std::vector<int32_t> off{0}, flat;
  for (int g : gorder) {
    int key = t.groups[g].key;
    if (key != t.hostname_key) {
      int nv = in.key_nvalues[key];
      for (int v = 0; v < nv; v++) flat.push_back(cnt[(size_t)g * 64 + v]);
    }
    off.push_back((int32_t)flat.size());
  }
  out->n_groups = (int32_t)gorder.size();
  out->n_domain_slots = (int32_t)flat.size();
  out->group_domain_off = (int32_t*)malloc(off.size() * 4);
  memcpy(out->group_domain_off, off.data(), off.size() * 4);
  out->domain_counts = (int32_t*)malloc((flat.size() ? flat.size() : 1) * 4);
  if (!flat.empty()) memcpy(out->domain_counts, flat.data(), flat.size() * 4);
  out->n_existing_evals = counters[0];
  out->n_inflight_evals = counters[1];
  out->n_template_evals = counters[2];
  out->n_commits = counters[3];
  out->solve_ms = h->stats.solve_ms;
  h->stats.bytes_d2h += P * 5 + C * (8 + (size_t)R * 8 + (size_t)ITW * 8 + (size_t)K * 25) + cnt.size() * 4;
  auto t1 = std::chrono::steady_clock::now();
  h->stats.download_ms += std::chrono::duration<double, std::milli>(t1 - t0).count();
  return KP_OK;
}

// outs[b] <- instance b after run_solve; KP_DEADLINE when some instance ran out of time (partial results are valid,
// scheduler.go:411-414)
static int download_all(kp_handle* h, const std::vector<int32_t>& statuses, kp_result* outs) {
  h->stats.download_ms = 0;
  h->stats.bytes_d2h = 0;
  int worst = KP_OK;
  for (size_t b = 0; b < h->insts.size(); b++) {
    int rc = download(h, *h->insts[b], &outs[b]);
    if (rc != KP_OK) {
      for (size_t i = 0; i < b; i++) kp_result_free(&outs[i]);
      return rc;
    }
    if (statuses[b] == KP_DEADLINE) worst = KP_DEADLINE;
  }
  return worst;
}

static int solve_uploaded(kp_handle* h, int64_t deadline_ms, kp_result* outs) {
  std::vector<int32_t> st;
  int rc = run_solve(h, deadline_ms, st);
  if (rc != KP_OK) return rc;
  for (int32_t s : st)
    if (s != KP_OK && s != KP_DEADLINE) return h->err = "claim capacity exceeded", s;
  return download_all(h, st, outs);
}

// kp_solve / kp_solve_batch: upload, solve, and while some instance needs more NodeClaims than provisioned, grow its
// claim capacity and redo
static int solve_growing(kp_handle* h, const kp_problem* const* problems, int n, kp_handle::Uploader by, int64_t deadline_ms,
                         kp_result* outs) {
  std::vector<int64_t> cmax(n);
  for (int b = 0; b < n; b++) cmax[b] = cmax_guess(problems[b]);
  for (;;) {
    int rc = upload(h, problems, n, cmax.data(), by);
    if (rc != KP_OK) return rc;
    std::vector<int32_t> st;
    rc = run_solve(h, deadline_ms, st);
    if (rc != KP_OK) return rc;
    bool grow = false;
    for (int b = 0; b < n; b++) {
      if (st[b] == KP_ERR_CAPACITY && cmax[b] < problems[b]->n_pods) {
        cmax[b] = std::min<int64_t>(problems[b]->n_pods, cmax[b] * 4);
        grow = true;
      } else if (st[b] != KP_OK && st[b] != KP_DEADLINE) {
        return h->err = "claim capacity exceeded", st[b];
      }
    }
    if (!grow) return download_all(h, st, outs);
  }
}

int kp_solve_resident(kp_handle* h, int64_t deadline_ms, kp_result* out) {
  if (h->uploaded != kp_handle::SINGLE) return h->err = "kp_upload has not been called", KP_ERR_INVALID;
  return solve_uploaded(h, deadline_ms, out);
}

int kp_solve(kp_handle* h, const kp_problem* p, int64_t deadline_ms, kp_result* out) {
  return solve_growing(h, &p, 1, kp_handle::SINGLE, deadline_ms, out);
}

// ---- multi-GPU: the global topology-domain counter table of a NodePool-sharded job --------------------------------
int kp_comm_unique_id(uint8_t* id128) {
  std::string err;
  if (!nccl_load(err)) return KP_ERR_CUDA;
  KpNcclId id;
  if (g_nccl.GetUniqueId(&id) != 0) return KP_ERR_CUDA;
  memcpy(id128, &id, sizeof(id));
  return KP_OK;
}

int kp_comm_init(kp_handle* h, const uint8_t* id128, int32_t rank, int32_t world) {
  if (!nccl_load(h->err)) return KP_ERR_CUDA;
  if (h->comm) {
    g_nccl.CommDestroy(h->comm);
    h->comm = nullptr;
  }
  cudaSetDevice(h->device);
  KpNcclId id;
  memcpy(&id, id128, sizeof(id));
  int rc = g_nccl.CommInitRank(&h->comm, world, id, rank);
  if (rc != 0) return h->err = std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"), KP_ERR_CUDA;
  h->comm_rank = rank;
  h->comm_world = world;
  return KP_OK;
}

// Slots an uploaded instance contributes: its non-hostname groups in table order (regular groups in creation order, then
// the inverse groups), one slot per value of the group's key -- the layout of kp_result.domain_counts when no group is
// born mid-solve.  instance < 0: the kp_upload instance, else index into the kp_upload_batch list.
static Instance* pick_instance(kp_handle* h, int32_t instance) {
  const size_t i = instance < 0 ? 0 : (size_t)instance;
  if (h->uploaded != (instance < 0 ? kp_handle::SINGLE : kp_handle::BATCH) || i >= h->insts.size()) return nullptr;
  return h->insts[i]->resident ? h->insts[i].get() : nullptr;
}
int64_t kp_comm_counter_slots(kp_handle* h, int32_t instance) {
  Instance* in = pick_instance(h, instance);
  if (!in) return -1;
  int64_t n = 0;
  for (int g = 0; g < in->host.G; g++)
    if (in->host.groups[g].key != in->host.hostname_key) n += in->key_nvalues[in->host.groups[g].key];
  return n;
}

// total_slots: size of the global table (sum over all ranks' instances); slot_offset[i]: where instance i of THIS handle
// starts (n_instances == 0 with the kp_upload instance: slot_offset[0]).  From now on every kp_solve_resident /
// kp_solve_batch_resident ends with scatter + all-reduce (when kp_comm_init was called) inside its solve_ms.
int kp_comm_set_counter_layout(kp_handle* h, int64_t total_slots, const int64_t* slot_offset, int32_t n_instances) {
  cudaSetDevice(h->device);
  if (n_instances <= 0 ? !pick_instance(h, -1) : h->uploaded != kp_handle::BATCH || n_instances != (int)h->insts.size())
    return h->err = "kp_comm_set_counter_layout: the instances do not match the upload", KP_ERR_INVALID;
  if (total_slots < 0) return h->err = "kp_comm_set_counter_layout: negative size", KP_ERR_INVALID;
  CK(h->arena.alloc(&h->d_gcnt, (size_t)std::max<int64_t>(total_slots, 1)));
  h->gcnt_slots = total_slots;
  for (size_t i = 0; i < h->insts.size(); i++) {
    Instance* in = h->insts[i].get();
    std::vector<int32_t> src;
    for (int g = 0; g < in->host.G; g++) {
      const int key = in->host.groups[g].key;
      if (key == in->host.hostname_key) continue;
      for (int v = 0; v < in->key_nvalues[key]; v++) src.push_back(g * 64 + v);
    }
    in->n_slots = (int64_t)src.size();
    in->slot_off = slot_offset[i];
    if (in->slot_off < 0 || in->slot_off + in->n_slots > total_slots)
      return h->err = "kp_comm_set_counter_layout: slice outside the table", KP_ERR_INVALID;
    CK(h->arena.alloc(&in->d_slot_src, std::max<size_t>(src.size(), 1)));
    if (!src.empty()) CK(cudaMemcpyAsync(in->d_slot_src, src.data(), src.size() * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return KP_OK;
}

int kp_comm_global_counts(kp_handle* h, int32_t* out, int64_t n) {
  if (!h->d_gcnt || n != h->gcnt_slots) return h->err = "kp_comm_global_counts: no table of that size", KP_ERR_INVALID;
  cudaSetDevice(h->device);
  CK(cudaMemcpy(out, h->d_gcnt, (size_t)n * 4, cudaMemcpyDeviceToHost));
  return KP_OK;
}

double kp_comm_last_allreduce_ms(kp_handle* h) { return h->allreduce_ms; }

#ifdef KP_PHASE_PROF
// Profiling build only: the solver warp's cycles per phase of the last solve of an instance (see KP_PROF_LAP), out[p] for
// p < KP_NPHASE, then the cycles of the whole pod loop, then the in-flight scan's steps, the positions it walked up to
// its results and the cycles of its first 32-wide steps.  Returns the number of values written.
int kp_phase_profile(kp_handle* h, int32_t instance, int64_t* out, int32_t n) {
  Instance* in = pick_instance(h, instance);
  if (!in || n < KP_NPROF) return h->err = "kp_phase_profile: no such instance or buffer too small", -1;
  cudaSetDevice(h->device);
  CK(cudaMemcpy(out, in->dev.counters + KP_PROF_AT, KP_NPROF * 8, cudaMemcpyDeviceToHost));
  return KP_NPROF;
}
#endif

void kp_comm_destroy(kp_handle* h) {
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  h->comm = nullptr;
}

// ---- kp_solve_batch: n independent Scheduler instances, one launch (one CTA per instance) ------------------------
int kp_upload_batch(kp_handle* h, const kp_problem* const* problems, int32_t n) {
  if (n < 0 || (n > 0 && !problems)) return h->err = "kp_upload_batch: bad arguments", KP_ERR_INVALID;
  std::vector<int64_t> cmax(n);
  for (int b = 0; b < n; b++) cmax[b] = cmax_guess(problems[b]);
  return upload(h, problems, n, cmax.data(), kp_handle::BATCH);
}

int kp_solve_batch_resident(kp_handle* h, int64_t deadline_ms, kp_result* outs) {
  if (h->uploaded != kp_handle::BATCH) return KP_OK;  // nothing from kp_upload_batch: an empty batch
  return solve_uploaded(h, deadline_ms, outs);
}

int kp_solve_batch(kp_handle* h, const kp_problem* const* problems, int32_t n, int64_t deadline_ms, kp_result* outs) {
  if (n < 0 || (n > 0 && (!problems || !outs))) return h->err = "kp_solve_batch: bad arguments", KP_ERR_INVALID;
  return solve_growing(h, problems, n, kp_handle::BATCH, deadline_ms, outs);
}

void kp_result_free(kp_result* r) {
  free(r->pod_target);
  free(r->pod_error);
  free(r->claim_template);
  free(r->claim_npods);
  free(r->claim_rank);
  free(r->claim_requests);
  free(r->claim_its);
  free(r->claim_req_flags);
  free(r->claim_req_gte);
  free(r->claim_req_lte);
  free(r->claim_req_mask);
  free(r->group_domain_off);
  free(r->domain_counts);
  free(r->claim_reservations);
  free(r->claim_dropped);
  memset(r, 0, sizeof(*r));
}

int kp_feasibility(kp_handle* h, const kp_problem* p, uint64_t* out_bits, int32_t* out_it_words) {
  const int64_t one = 1;
  int rc = upload(h, &p, 1, &one, kp_handle::SINGLE);
  if (rc != KP_OK) return rc;
  KpDev& d = h->insts[0]->dev;
  *out_it_words = d.ITW;
  size_t n = (size_t)d.X * d.N * d.ITW;
  uint64_t* dout;
  CK(cudaMalloc(&dout, std::max<size_t>(n, 1) * 8));
  if (d.N > 0) k_feasibility<<<(d.N * 32 + 255) / 256, 256, 0, h->stream>>>(d, nullptr, 1);
  CK(cudaEventRecord(h->ev0, h->stream));
  if (d.N > 0 && d.X > 0) {
    int blocks = h->n_sm * 8;
    k_feasibility<<<blocks, 256, 0, h->stream>>>(d, dout, 0);
  }
  CK(cudaEventRecord(h->ev1, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  h->stats.solve_ms = ms;
  CK(cudaMemcpy(out_bits, dout, n * 8, cudaMemcpyDeviceToHost));
  cudaFree(dout);
  return KP_OK;
}

int kp_consolidate(kp_handle* h, const kp_problem* cluster, const kp_consol_input* in, int64_t deadline_ms,
                   kp_consol_result* out) {
  memset(out, 0, sizeof(*out));
  int rc = kp_consolidate_impl(h, cluster, in, deadline_ms, out);
  if (rc != KP_OK && rc != KP_DEADLINE) kp_consol_result_free(out);  // nothing half-built leaves the library
  return rc;
}

void kp_consol_result_free(kp_consol_result* r) {
  free(r->decision);
  free(r->replacement_its);
  free(r->n_new_claims);
  free(r->n_unscheduled);
  free(r->repl_template);
  free(r->repl_requests);
  free(r->repl_req_flags);
  free(r->repl_req_gte);
  free(r->repl_req_lte);
  free(r->repl_req_mask);
  free(r->repl_order_off);
  free(r->repl_order);
  memset(r, 0, sizeof(*r));
}
}

__global__ void k_scatter_rank(const int32_t* perm, int64_t n, int32_t* rank) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) rank[perm[i]] = (int32_t)i;
}

// Rows [0, n) of the KpConsol outputs -> subsets at[0, n) of `out` (at null: row b is subset b, and the fixed-size
// fields are copied in place); with the price-order export, the orders go to order_rows
static int read_consol(kp_handle* h, const KpConsol& q, int n, const int32_t* at, const ReqLayout& L, int R, int ITW,
                       std::vector<std::vector<int32_t>>& order_rows, kp_consol_result* out) {
  const size_t K = (size_t)L.K, n1 = (size_t)std::max(n, 1), cap = (size_t)q.order_cap;
  auto sub = [&](size_t b) { return at ? (size_t)at[b] : b; };
  auto rows = [&](auto* dst, const auto* src, size_t width) {  // `width` elements per row
    const size_t row = width * sizeof(*dst);
    if (!at) return cudaMemcpy(dst, src, n * row, cudaMemcpyDeviceToHost);
    std::vector<std::remove_pointer_t<decltype(dst)>> tmp(n1 * width);
    const cudaError_t e = cudaMemcpy(tmp.data(), src, n * row, cudaMemcpyDeviceToHost);
    for (size_t b = 0; b < (size_t)n; b++) memcpy(dst + sub(b) * width, tmp.data() + b * width, row);
    return e;
  };
  CK(rows(out->decision, q.decision, 1));
  CK(rows(out->replacement_its, q.replacement_its, ITW));
  CK(rows(out->n_new_claims, q.n_new_claims, 1));
  CK(rows(out->n_unscheduled, q.n_unscheduled, 1));
  CK(rows(out->repl_template, q.repl_tmpl, 1));
  CK(rows(out->repl_requests, q.repl_req, R));
  std::vector<uint8_t> sfl(n1 * K);
  std::vector<uint64_t> smk(n1 * K);
  std::vector<int32_t> on(n1), ord(q.repl_order ? n1 * cap : 0);
  std::vector<int64_t> sg(q.repl_sgte ? n1 * K : 0), sl(sg.size());
  CK(cudaMemcpy(sfl.data(), q.repl_sflags, (size_t)n * K, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(smk.data(), q.repl_smask, (size_t)n * K * 8, cudaMemcpyDeviceToHost));
  if (q.repl_sgte) {
    CK(cudaMemcpy(sg.data(), q.repl_sgte, (size_t)n * K * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(sl.data(), q.repl_slte, (size_t)n * K * 8, cudaMemcpyDeviceToHost));
  }
  if (q.repl_order) {
    CK(cudaMemcpy(ord.data(), q.repl_order, (size_t)n * cap * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(on.data(), q.repl_order_n, (size_t)n * 4, cudaMemcpyDeviceToHost));
  }
  for (size_t b = 0; b < (size_t)n; b++) {
    const size_t s = sub(b);
    if (out->decision[s] != KP_DECISION_REPLACE)
      out->repl_template[s] = -1;
    else
      L.store(s, sfl.data() + b * K, smk.data() + b * K, q.repl_sgte ? sg.data() + b * K : nullptr,
              q.repl_sgte ? sl.data() + b * K : nullptr, out->repl_req_flags, out->repl_req_gte, out->repl_req_lte,
              out->repl_req_mask);
    if (q.repl_order) order_rows[s].assign(ord.begin() + b * cap, ord.begin() + b * cap + on[b]);
  }
  return KP_OK;
}

// kp_consolidate: every subset is one SimulateScheduling + computeConsolidation (helpers.go:51-142,
// consolidation.go:136-229); they are independent, so each runs as its own solver instance on its own warp.
static int kp_consolidate_impl(kp_handle* h, const kp_problem* p, const kp_consol_input* in, int64_t deadline_ms,
                               kp_consol_result* out) {
  const auto t_call = std::chrono::steady_clock::now();
  const int S = in->n_subsets;
  const int n_extra = in->n_extra_pods > 0 ? in->n_extra_pods : 0;
  if (p->n_nodes > 0 && !in->node_pod_off) return h->err = "kp_consolidate: node_pod_off is null", KP_ERR_INVALID;
  const int64_t extra_row0 = p->n_nodes > 0 ? in->node_pod_off[p->n_nodes] : 0;
  if (n_extra > 0 && (!in->extra_pod_kind || extra_row0 + n_extra != p->n_pods))
    return h->err = "kp_consolidate: the extra pods must be the last n_extra_pods rows of the pod table, with kinds", KP_ERR_INVALID;
  for (int i = 0; i < n_extra; i++)
    if (in->extra_pod_kind[i] != KP_EXTRA_PENDING && in->extra_pod_kind[i] != KP_EXTRA_DELETING_NODE)
      return h->err = "kp_consolidate: unknown extra pod kind", KP_ERR_INVALID;
  const int64_t one = 1;
  int rc = upload(h, &p, 1, &one, kp_handle::SINGLE);  // the cluster's pod table doubles as the "pods" of the problem (rows by node)
  if (rc != KP_OK) return rc;
  Instance& cl = *h->insts[0];
  HostTables& t = cl.host;
  KpDev& d = cl.dev;
  if (t.has_min_values && !t.min_values_strict) {
    // BestEffort lowers minValues per NodeClaim during the simulation (nodeclaim.go:186-191); carrying those per-claim values
    // through RemoveInstanceTypeOptionsByPriceAndMinValues is not built.  Strict (the default policy) is served.
    h->err = "consolidation with minValues under the BestEffort policy is not supported yet";
    return KP_ERR_UNSUPPORTED;
  }
  const int K = t.K, R = t.R, ITW = t.ITW, E = t.E, T = t.T;
  const bool general = t.G > 0;  // the evicted pods carry topology constraints: one full solve per candidate set
  const ReqLayout L(cl);
  // ---- result arrays (owned by `out` from here on: kp_consolidate frees them on any error return)
  const int MW = L.words();
  {
    const size_t s1 = S ? S : 1;
    out->n_subsets = S;
    out->it_words = ITW;
    out->n_keys = K;
    out->mask_words = MW;
    out->n_resources = R;
    out->decision = (uint8_t*)malloc(s1);
    memset(out->decision, KP_DECISION_UNKNOWN, s1);
    out->replacement_its = (uint64_t*)calloc(s1 * (ITW ? ITW : 1), sizeof(uint64_t));
    out->n_new_claims = (int32_t*)calloc(s1, sizeof(int32_t));
    out->n_unscheduled = (int32_t*)calloc(s1, sizeof(int32_t));
    out->repl_template = (int32_t*)malloc(s1 * 4);
    for (size_t i = 0; i < s1; i++) out->repl_template[i] = -1;
    out->repl_requests = (int64_t*)calloc(s1 * (R ? R : 1), 8);
    out->repl_req_flags = (uint8_t*)calloc(s1 * (K ? K : 1), 1);
    out->repl_req_gte = (int64_t*)calloc(s1 * (K ? K : 1), 8);
    out->repl_req_lte = (int64_t*)calloc(s1 * (K ? K : 1), 8);
    out->repl_req_mask = (uint64_t*)calloc(s1 * (MW ? MW : 1), 8);
  }
  const int order_cap = std::min(std::max(T, 1), 600);
  std::vector<std::vector<int32_t>> order_rows(in->export_price_order ? S : 0);
  auto finish_order = [&]() {
    if (!in->export_price_order) return;
    out->repl_order_off = (int32_t*)calloc((size_t)S + 1, 4);
    size_t tot = 0;
    for (int s_ = 0; s_ < S; s_++) {
      tot += order_rows[s_].size();
      out->repl_order_off[s_ + 1] = (int32_t)tot;
    }
    out->repl_order = (int32_t*)calloc(tot ? tot : 1, 4);
    for (int s_ = 0; s_ < S; s_++)
      if (!order_rows[s_].empty()) memcpy(out->repl_order + out->repl_order_off[s_], order_rows[s_].data(), order_rows[s_].size() * 4);
  };
  auto ms_left = [&]() -> int64_t {  // < 0: no deadline
    if (deadline_ms <= 0) return -1;
    const double used = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_call).count();
    return std::max<int64_t>(0, deadline_ms - (int64_t)used);
  };
  auto t_begin = std::chrono::steady_clock::now();
  // ---- host-side constants of the decision step
  const ConsolPrices cp = consol_prices(p, t, in);
  const PriceLists ml = order_by_price(p, t);
  // price tables and decision constants of the device side (both paths)
  auto upload_prices = [&](KpConsol& q) -> int {
    q.ct_key = in->capacity_type_key;
    q.ct_spot = in->ct_spot;
    q.ct_od = in->ct_on_demand;
    q.export_order = in->export_price_order ? 1 : 0;
    q.order_cap = order_cap;
    q.ct_order_valid = cp.ct_valid;
    q.spot_to_spot_enabled = in->spot_to_spot_enabled;
    q.T = T;
    CK(up(h, &q.node_price, cp.node_price));
    uint8_t* u8;
    CK(up_raw(h, &u8, in->node_is_spot, (size_t)E));
    q.node_is_spot = u8;
    int32_t* nit = nullptr;
    CK(up_raw(h, &nit, in->node_it, (size_t)E));
    q.node_it = nit;
    q.filter_same_type = in->filter_same_instance_type;
    CK(up(h, &q.ml_off, ml.off));
    CK(up(h, &q.ml_set, ml.set));
    CK(up(h, &q.ml_price, ml.price));
    CK(up(h, &q.wl_off, cp.worst.off));
    CK(up(h, &q.wl_set, cp.worst.set));
    CK(up(h, &q.wl_price, cp.worst.price));
    return KP_OK;
  };
  // per-row outputs of `n` candidate sets
  auto alloc_rows = [&](KpConsol& q, size_t n) -> int {
    CK(zeros(h, &q.decision, n));
    CK(zeros(h, &q.replacement_its, n * std::max(ITW, 1)));
    CK(zeros(h, &q.n_new_claims, n));
    CK(zeros(h, &q.n_unscheduled, n));
    CK(zeros(h, &q.repl_tmpl, n));
    CK(zeros(h, &q.repl_req, n * std::max(R, 1)));
    CK(zeros(h, &q.repl_sflags, n * std::max(K, 1)));
    CK(zeros(h, &q.repl_smask, n * std::max(K, 1)));
    if (t.has_bounds) {
      CK(zeros(h, &q.repl_sgte, n * std::max(K, 1)));
      CK(zeros(h, &q.repl_slte, n * std::max(K, 1)));
    }
    if (in->export_price_order) {
      CK(zeros(h, &q.repl_order, n * order_cap));
      CK(zeros(h, &q.repl_order_n, n));
    }
    return KP_OK;
  };
  // `slots` x the per-slot count of each scratch array the pass needs (KP_CONSOL_SCRATCH, KP_SORT_SCRATCH)
#define KP_ALLOC_SCRATCH(f, type, count, present) \
  if (present) CK(zeros(h, &q.ws.f, slots * (size_t)(count)));
  for (int s = 0; s < S; s++)
    for (int i = in->subset_off[s]; i < in->subset_off[s + 1]; i++)
      if (in->subset_nodes[i] < 0 || in->subset_nodes[i] >= E) return h->err = "subset node out of range", KP_ERR_INVALID;
  if (general) {
    // ---- general path: a candidate set is SimulateScheduling over its own stateNodes / bound pods / pending pods
    // (helpers.go:51-142) -> a derived kp_problem (fresh NewTopology).  All sets of a chunk are uploaded side by side and
    // solved by ONE k_wsolve_batch launch (one CTA per set), then k_decide_batch applies computeConsolidation.  Each
    // chunk's upload replaces the handle's instances and reuses the arena: from then on only the cluster's host tables
    // are read.
    const std::unique_ptr<Instance> cluster = std::move(h->insts[0]);
    h->insts.clear();
    h->uploaded = kp_handle::NONE;
    double total_ms = 0;
    bool timed_out = false;
    const int CHUNK = 2 * h->n_sm;  // two waves of CTAs; bounds the HBM the side-by-side tables take
    std::vector<uint8_t> is_cand(std::max(E, 1), 0), flags(std::max(E, 1), 0);
    for (int c0 = 0; c0 < S && !timed_out; c0 += CHUNK) {
      const int c1 = std::min(S, c0 + CHUNK);
      if (deadline_ms > 0 && ms_left() == 0) {
        timed_out = true;
        break;
      }
      begin_upload(h, kp_handle::NONE);  // the sets of a chunk are no upload kp_solve_resident / kp_solve_batch_resident serve
      std::vector<int> set_of;  // instance -> subset
      std::vector<int32_t> soff{0}, snodes_all;
      for (int s = c0; s < c1; s++) {
        const int so = in->subset_off[s], sn = in->subset_off[s + 1] - so;
        std::fill(is_cand.begin(), is_cand.end(), 0);
        for (int i = 0; i < sn; i++) is_cand[in->subset_nodes[so + i]] = 1;
        for (int n = 0; n < E; n++)
          flags[n] = is_cand[n] ? (uint8_t)(p->node_flags[n] & ~KP_NODE_SCHEDULABLE) : p->node_flags[n];
        std::vector<int32_t> pod_class, run_class(p->run_class, p->run_class + p->n_running),
            run_node(p->run_node, p->run_node + p->n_running);
        std::vector<int64_t> creation;
        std::vector<uint64_t> uid_hi, uid_lo;
        std::vector<uint8_t> kinds;
        auto take = [&](int64_t j, uint8_t kind) {
          pod_class.push_back(p->pod_class[j]);
          creation.push_back(p->pod_creation ? p->pod_creation[j] : 0);
          uid_hi.push_back(p->pod_uid_hi[j]);
          uid_lo.push_back(p->pod_uid_lo[j]);
          kinds.push_back(kind);
        };
        for (int n = 0; n < E; n++)
          for (int j = in->node_pod_off[n]; j < in->node_pod_off[n + 1]; j++) {
            if (is_cand[n]) {
              take(j, 0);
            } else {  // still running where it is: counted by the topology
              run_class.push_back(p->pod_class[j]);
              run_node.push_back(n);
            }
          }
        for (int i = 0; i < n_extra; i++) take(extra_row0 + i, in->extra_pod_kind[i]);
        if (pod_class.empty()) {  // nothing to reschedule: every pod is "placed", no NodeClaim
          out->decision[s] = KP_DECISION_DELETE;
          continue;
        }
        kp_problem sp = *p;
        sp.node_flags = flags.data();
        sp.n_pods = (int64_t)pod_class.size();
        sp.pod_class = pod_class.data();
        sp.pod_creation = creation.data();
        sp.pod_uid_hi = uid_hi.data();
        sp.pod_uid_lo = uid_lo.data();
        sp.n_running = (int64_t)run_class.size();
        sp.run_class = run_class.data();
        sp.run_node = run_node.data();
        rc = add_instance(h, &sp, sp.n_pods);
        if (rc != KP_OK) return rc;
        if (n_extra > 0) {
          uint8_t* dk;
          CK(up_raw(h, &dk, kinds.data(), kinds.size()));
          h->insts.back()->dev.pod_kind = dk;
          CK(cudaStreamSynchronize(h->stream));  // `kinds` dies with this iteration
        }
        set_of.push_back(s);
        for (int i = 0; i < sn; i++) snodes_all.push_back(in->subset_nodes[so + i]);
        soff.push_back((int32_t)snodes_all.size());
      }
      const int nb = (int)set_of.size();
      if (nb == 0) continue;
      KpConsol q;
      memset(&q, 0, sizeof(q));
      rc = upload_prices(q);
      if (rc != KP_OK) return rc;
      int32_t *d_soff, *d_snodes;
      CK(up_raw(h, &d_soff, soff.data(), soff.size()));
      CK(up_raw(h, &d_snodes, snodes_all.data(), std::max<size_t>(snodes_all.size(), 1)));
      const size_t slots = (size_t)nb;  // k_decide_batch: block b uses sort slot b
      KP_SORT_SCRATCH(KP_ALLOC_SCRATCH, d, q)
      rc = alloc_rows(q, (size_t)nb);
      if (rc != KP_OK) return rc;
      std::vector<int32_t> st;
      rc = run_solve(h, ms_left() < 0 ? 0 : std::max<int64_t>(ms_left(), 1), st);
      if (rc != KP_OK) return rc;
      total_ms += h->stats.solve_ms;
      bool chunk_timed_out = false;
      for (int32_t v : st) {
        if (v == KP_DEADLINE)
          chunk_timed_out = true;
        else if (v != KP_OK)
          return h->err = "consolidation simulation failed", v;
      }
      if (chunk_timed_out) {  // partial simulations decide nothing (the reference drops the whole pass on ctx.Err())
        timed_out = true;
        break;
      }
      k_decide_batch<<<nb, 32, 0, h->stream>>>(h->d_devs, q, d_soff, d_snodes);
      CK(cudaStreamSynchronize(h->stream));
      CK(cudaGetLastError());
      rc = read_consol(h, q, nb, set_of.data(), L, R, ITW, order_rows, out);
      if (rc != KP_OK) return rc;
    }
    h->insts.clear();
    finish_order();
    out->solve_ms = total_ms;
    h->stats.solve_ms = total_ms;
    return timed_out ? KP_DEADLINE : KP_OK;
  }
  int capq = 1;
  for (int s = 0; s < S; s++) {
    int n = 0;
    for (int i = in->subset_off[s]; i < in->subset_off[s + 1]; i++) {
      const int node = in->subset_nodes[i];
      n += in->node_pod_off[node + 1] - in->node_pod_off[node];
    }
    capq = std::max(capq, n);
  }
  capq += n_extra;
  // ---- device inputs
  KpConsol q;
  memset(&q, 0, sizeof(q));
  q.n_subsets = S;
  q.capq = capq;
  int n_sub_nodes = S ? in->subset_off[S] : 0;
  int32_t* tmp32;
  CK(up_raw(h, &tmp32, in->subset_off, (size_t)S + 1));
  q.subset_off = tmp32;
  CK(up_raw(h, &tmp32, in->subset_nodes, (size_t)n_sub_nodes));
  q.subset_nodes = tmp32;
  CK(up_raw(h, &tmp32, in->node_pod_off, (size_t)E + 1));
  q.node_pod_off = tmp32;
  q.pod_class = cl.d_pod_class;
  q.n_extra = n_extra;
  q.extra_row0 = (int)extra_row0;
  if (n_extra > 0) {
    uint8_t* dk;
    CK(up_raw(h, &dk, in->extra_pod_kind, (size_t)n_extra));
    q.extra_kind = dk;
  }
  q.deadline_ns = deadline_ms > 0 ? std::max<int64_t>(ms_left(), 1) * 1000000ll : 0;
  CK(zeros(h, &q.t_start, 1));
  CK(zeros(h, &tmp32, (size_t)std::max<int64_t>(cl.P, 1)));
  int32_t* d_rank = tmp32;
  q.pod_rank = d_rank;
  {
    std::vector<int32_t> ntm(std::max(E, 1), -1);
    std::vector<int64_t> ncap((size_t)std::max(E, 1) * R, 0);
    for (int n = 0; n < E; n++) {
      ntm[n] = p->node_template ? p->node_template[n] : -1;
      if (p->node_capacity)
        for (int r = 0; r < R; r++) ncap[(size_t)n * R + r] = p->node_capacity[(size_t)n * R + r];
    }
    CK(up(h, &q.node_tmpl, ntm));
    CK(up(h, &q.node_capacity, ncap));
    CK(up(h, &q.tmpl_remaining0, t.tmpl_remaining));
    rc = upload_prices(q);
    if (rc != KP_OK) return rc;
  }
  // ---- launch geometry: as many resident warps as the GPU holds, each with a private scratch slot
  const size_t budget = 200 * 1024;
  const size_t fixed = KP_ALIGN16(sizeof(ConsolShared));
  KpDev dq = d;  // the cluster's pointer block with k_consolidate's table plan (the upload keeps the solver's)
  dq.tab_bytes = plan_tables(dq, fixed, budget);
  const size_t smem = fixed + dq.tab_bytes + 64;
  // the solver's `in.lean` predicate (G == 0 here)
  const bool lean = !t.has_bounds && !t.min_values_strict && t.n_rsv == 0 && d.n_hostports == 0 && !t.has_vol_alts &&
                    !getenv("KP_NO_LEAN");
  const void* fn = consol_kernel(lean, t.has_vol_alts);
  if (getenv("KP_DEBUG"))
    fprintf(stderr, "[kp] consolidate plan: tables %zu B staged of %zu B, %zu B shared, kernel %s\n", (size_t)dq.tab_bytes,
            kp_tab_bytes(dq), smem, kernel_name(fn));
  CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, CONSOL_WARPS * 32, smem);
  per_sm = std::max(per_sm, 1);
  int grid = std::min(h->n_sm * per_sm, std::max(1, (S + CONSOL_WARPS - 1) / CONSOL_WARPS));
  const size_t slots = (size_t)grid * CONSOL_WARPS;
  KP_CONSOL_SCRATCH(KP_ALLOC_SCRATCH, d, q)
  const size_t S1 = (size_t)std::max(S, 1);
  rc = alloc_rows(q, S1);
  if (rc != KP_OK) return rc;
  CK(cudaMemsetAsync(q.decision, KP_DECISION_UNKNOWN, S1, h->stream));  // a subset the deadline cut off stays unknown
  CK(zeros(h, &q.next, 1));
  CK(zeros(h, &q.status, 1));
  rc = reset_dynamic(h, cl);
  if (rc != KP_OK) return rc;
  auto t_up = std::chrono::steady_clock::now();
  h->stats.upload_ms += std::chrono::duration<double, std::milli>(t_up - t_begin).count();
  // ---- kernels
  CK(cudaEventRecord(h->ev0, h->stream));
  h->stats.kernel_launches = 0;
  h->stats.cohort_pods = 0;
  if (d.N > 0) {
    k_feasibility<<<(d.N * 32 + 255) / 256, 256, 0, h->stream>>>(d, nullptr, 1);
    h->stats.kernel_launches++;
  }
  rc = sort_queue(h, cl);  // byCPUAndMemoryDescending over every pod row; a subset's queue is its rows in rank order
  if (rc != KP_OK) return rc;
  if (cl.P > 0) {
    k_scatter_rank<<<(int)((cl.P + 255) / 256), 256, 0, h->stream>>>(d.queue, cl.P, d_rank);
    h->stats.kernel_launches++;
  }
  rc = launch_node_cand(h, cl);
  if (rc != KP_OK) return rc;
  if (S > 0) {
    void* args[] = {(void*)&dq, (void*)&q};
    CK(cudaLaunchKernel(fn, dim3(grid), dim3(CONSOL_WARPS * 32), args, smem, h->stream));
    h->stats.kernel_launches++;
  }
  CK(cudaEventRecord(h->ev1, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaGetLastError());
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  h->stats.solve_ms = ms;
  int32_t status = 0;
  CK(cudaMemcpy(&status, q.status, 4, cudaMemcpyDeviceToHost));
  if (status != KP_OK) return h->err = "consolidation instance failed (capacity or invalid state)", status;
  // ---- results
  auto t0 = std::chrono::steady_clock::now();
  rc = read_consol(h, q, S, nullptr, L, R, ITW, order_rows, out);
  if (rc != KP_OK) return rc;
  finish_order();
  out->solve_ms = ms;
  h->stats.bytes_d2h = (size_t)S * (13 + (size_t)ITW * 8 + (size_t)R * 8 + (size_t)K * 9);
  h->stats.download_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  bool unknown = false;
  for (int s_ = 0; s_ < S; s_++) unknown = unknown || out->decision[s_] == KP_DECISION_UNKNOWN;
  if (unknown) {
    if (deadline_ms > 0) return KP_DEADLINE;  // the subsets that finished are valid
    return h->err = "internal: a candidate set was not evaluated", KP_ERR_INVALID;
  }
  return KP_OK;
}
#undef KP_ALLOC_SCRATCH
