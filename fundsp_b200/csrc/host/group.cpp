// fundsp_b200 multi-GPU mix-down — see group.h.
#include "group.h"

#include <dlfcn.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace fdsp {
namespace host {

namespace {

// the handful of NCCL declarations used (nccl.h is not needed to build; values are part of NCCL's stable ABI)
typedef void* ncclComm_t;
struct NcclId { char internal[128]; };
constexpr int kNcclFloat32 = 7, kNcclSum = 0;
struct Nccl {
  void* lib = nullptr; bool ok = false; std::string why;
  int (*GetUniqueId)(NcclId*);
  int (*CommInitRank)(ncclComm_t*, int, NcclId, int);
  int (*CommDestroy)(ncclComm_t);
  int (*GroupStart)();
  int (*GroupEnd)();
  int (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t);
  int (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t);
  int (*Reduce)(const void*, void*, size_t, int, int, int, ncclComm_t, cudaStream_t);
  const char* (*GetErrorString)(int);
};
template <class F> bool sym(void* lib, const char* name, F& f) { f = reinterpret_cast<F>(dlsym(lib, name)); return f != nullptr; }
Nccl& nccl() {
  static Nccl n;
  static std::once_flag once;
  std::call_once(once, [] {
#ifdef FDSP_HOST_EMUL
    n.why = "the mock device has no NCCL";
#else
    const char* env = getenv("FDSP_NCCL_LIB");
    for (const char* name : {env ? env : "libnccl.so.2", "libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2"})
      if ((n.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL))) break;
    if (!n.lib) { n.why = "libnccl.so.2 not found (set FDSP_NCCL_LIB)"; return; }
    n.ok = sym(n.lib, "ncclGetUniqueId", n.GetUniqueId) && sym(n.lib, "ncclCommInitRank", n.CommInitRank) && sym(n.lib, "ncclCommDestroy", n.CommDestroy) &&
           sym(n.lib, "ncclGroupStart", n.GroupStart) && sym(n.lib, "ncclGroupEnd", n.GroupEnd) && sym(n.lib, "ncclSend", n.Send) && sym(n.lib, "ncclRecv", n.Recv) &&
           sym(n.lib, "ncclReduce", n.Reduce) && sym(n.lib, "ncclGetErrorString", n.GetErrorString);
    if (!n.ok) n.why = "libnccl lacks the expected symbols";
#endif
  });
  return n;
}
std::string nerr(const char* what, int rc) { return std::string(what) + ": " + (nccl().GetErrorString ? nccl().GetErrorString(rc) : "NCCL error"); }
#define NC(call) do { int rc_ = (call); if (rc_ != 0) return nerr(#call, rc_); } while (0)
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return std::string(#call) + ": " + cudaGetErrorString(e_); } while (0)

#ifndef FDSP_HOST_EMUL
// root: mix[c][t] = ((p_0 + p_1) + p_2) + ... in rank order; the root's own partial is read from `mix` itself
__global__ void rank_fold_kernel(float* mix, uint32_t mix_stride, const float* gathered, uint32_t nranks, uint32_t root, uint32_t channels, uint32_t n) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= channels * n) return;
  const uint32_t c = e / n, t = e - c * n;
  float* own = mix + (size_t)c * mix_stride + t;
  const size_t plane = (size_t)channels * n;
  float s = root == 0 ? *own : gathered[(size_t)c * n + t];
  for (uint32_t r = 1; r < nranks; r++) s += (r == root) ? *own : gathered[r * plane + (size_t)c * n + t];
  *own = s;
}
#endif

}  // namespace

Group::~Group() {
  cudaSetDevice(device);
  if (d_gather) cudaFree(d_gather);
  if (comm && nccl().ok) nccl().CommDestroy((ncclComm_t)comm);
}

std::string group_unique_id(void* id128) {
  Nccl& N = nccl();
  if (!N.ok) return N.why;
  if (!id128) return "null id buffer";
  NcclId id;
  NC(N.GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return "";
}

std::string group_create(int nranks, int rank, const void* id128, int device, Group** out) {
  if (!out) return "null out pointer";
  if (nranks < 1 || rank < 0 || rank >= nranks) return "group: rank out of range";
  std::unique_ptr<Group> g(new Group());
  g->nranks = nranks; g->rank = rank; g->device = device;
  const char* mode = getenv("FDSP_GROUP_REDUCE");
  g->nccl_reduce = mode && strcmp(mode, "nccl") == 0;
  if (nranks > 1) {
    Nccl& N = nccl();
    if (!N.ok) return N.why;
    if (!id128) return "group: null unique id";
    CU(cudaSetDevice(device));
    NcclId id; memcpy(&id, id128, sizeof(id));
    ncclComm_t c = nullptr;
    NC(N.CommInitRank(&c, nranks, id, rank));
    g->comm = c;
  }
  *out = g.release();
  return "";
}

std::string group_reduce_device(Bank& b, Group& g, uint64_t n, float* mix_dev, uint64_t mix_stride, int root) {
  if (b.sh_writes()) return "#U reduce: a bank whose monitor / timer writes a Shared cannot be part of a multi-GPU group (each rank would store its own value)";
  if (g.nranks == 1 || n == 0) return "";
  if (root < 0 || root >= g.nranks) return "reduce: root out of range";
  if (!mix_dev) return "reduce: null mix buffer";
  if (g.device != b.device) return "reduce: the group and the bank live on different devices";
#ifdef FDSP_HOST_EMUL
  return "the mock device has no NCCL";
#else
  Nccl& N = nccl();
  CU(cudaSetDevice(b.device));
  const uint32_t ch = (uint32_t)b.nout;
  if (n > 0xffffffffull / std::max(1u, ch)) return "reduce: too many samples for one call";
  // an NCCL group that was started is always ended, also when a call inside it fails (an open group would swallow every later NCCL call)
  struct GroupScope {
    Nccl& N; bool open = false;
    explicit GroupScope(Nccl& n) : N(n) {}
    int start() { const int rc = N.GroupStart(); open = rc == 0; return rc; }
    int end() { open = false; return N.GroupEnd(); }
    ~GroupScope() { if (open) N.GroupEnd(); }
  };
  if (g.nccl_reduce) {
    GroupScope gs(N);
    NC(gs.start());
    for (uint32_t c = 0; c < ch; c++) NC(N.Reduce(mix_dev + c * mix_stride, mix_dev + c * mix_stride, n, kNcclFloat32, kNcclSum, root, (ncclComm_t)g.comm, b.stream));
    NC(gs.end());
    return "";
  }
  const size_t plane = (size_t)ch * n;
  if (g.rank == root && g.gather_cap < plane * g.nranks) {
    if (g.d_gather) { CU(cudaStreamSynchronize(b.stream)); cudaFree(g.d_gather); g.d_gather = nullptr; }
    CU(cudaMalloc((void**)&g.d_gather, plane * g.nranks * sizeof(float)));
    g.gather_cap = plane * g.nranks;
  }
  GroupScope gs(N);
  NC(gs.start());
  if (g.rank == root) {
    // one receive per channel row: NCCL pairs sends and receives in order, and their counts must agree (the sender's rows may be strided)
    for (int r = 0; r < g.nranks; r++) if (r != root)
      for (uint32_t c = 0; c < ch; c++) NC(N.Recv(g.d_gather + (size_t)r * plane + (size_t)c * n, n, kNcclFloat32, r, (ncclComm_t)g.comm, b.stream));
  } else {
    // rows of a strided mix buffer go one by one (the receiver's plane is dense [channel][n])
    for (uint32_t c = 0; c < ch; c++) NC(N.Send(mix_dev + c * mix_stride, n, kNcclFloat32, root, (ncclComm_t)g.comm, b.stream));
  }
  NC(gs.end());
  if (g.rank == root) {
    const uint32_t total = ch * (uint32_t)n;
    rank_fold_kernel<<<(total + 255) / 256, 256, 0, b.stream>>>(mix_dev, (uint32_t)mix_stride, g.d_gather, (uint32_t)g.nranks, (uint32_t)root, ch, (uint32_t)n);
    CU(cudaGetLastError());
    b.launches++;
  }
  return "";
#endif
}

std::string group_render_host(Bank& b, Group& g, uint64_t n, const float* in, float* out_mix, int root) {
  if (!(b.out_mode & 2u)) return "render_reduced: the bank was not created with FDSP_OUT_MIX";
  if (g.rank == root && !out_mix) return "render_reduced: the root needs an output buffer";
  CU(cudaSetDevice(b.device));
  if (n == 0) return "";
  if (b.sh_writes()) return "#U render_reduced: a bank whose monitor / timer writes a Shared cannot be part of a multi-GPU group (each rank would store its own value)";
  { std::string se = b.sh_pull(); if (!se.empty()) return se; }   // every rank reads the cells into its own voices' words
  const uint32_t chunk = (uint32_t)std::min<uint64_t>(16384, (n + 63) / 64 * 64);
  std::string e = b.ensure_staging(chunk);
  if (!e.empty()) return e;
  for (uint64_t t0 = 0; t0 < n; t0 += chunk) {
    const uint32_t len = (uint32_t)std::min<uint64_t>(chunk, n - t0);
    if (b.nin > 0) {
      if (!in) return "bank has inputs but no input buffer was given";
      CU(cudaMemcpy2DAsync(b.d_in, (size_t)chunk * 4, in + t0, (size_t)n * 4, (size_t)len * 4, b.nin, cudaMemcpyHostToDevice, b.stream));
    }
    if (!(e = b.render_device(len, b.d_in, chunk, nullptr, chunk, b.d_mix, chunk)).empty()) return e;
    if (!(e = group_reduce_device(b, g, len, b.d_mix, chunk, root)).empty()) return e;
    if (g.rank == root) CU(cudaMemcpy2DAsync(out_mix + t0, (size_t)n * 4, b.d_mix, (size_t)chunk * 4, (size_t)len * 4, b.nout, cudaMemcpyDeviceToHost, b.stream));
  }
  CU(cudaStreamSynchronize(b.stream));
  return "";
}

}  // namespace host
}  // namespace fdsp
