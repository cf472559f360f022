// fundsp_b200 multi-GPU mix-down below the C ABI (SURVEY.md §8e): voices shard across ranks — one bank per GPU, one process per
// GPU — and the ONE exchange step of the path, the sum of the per-GPU partial mixes, runs here, on the bank's own stream, so a
// host in any language (the Rust shim of INTEGRATION.md has no torch.distributed) gets the reduced mix from one call.
//
// Transport: NCCL (dlopen'ed: libnccl.so.2 — the copy already loaded into the process when torch is, else the system one).
// Default reduction = GATHER + ORDERED FOLD: every rank sends its [channels][n] partial to the root (ncclSend / ncclRecv in one
// group over NVLink), and the root adds them in RANK ORDER ((p0 + p1) + p2) + ... with one small kernel. The association is fixed
// by construction — it does not depend on NCCL's ring / tree choice, message size or topology — which is what parity against the
// CPU reference's index-order sum needs (ranks own contiguous voice ranges). FDSP_GROUP_REDUCE=nccl switches to a plain
// ncclReduce(sum) (same bytes on the wire for the root, NCCL's own association).
#pragma once
#include <string>

#include "bank.h"

namespace fdsp {
namespace host {

struct Group {
  int nranks = 1, rank = 0, device = 0;
  void* comm = nullptr;            // ncclComm_t
  Array<float> d_gather;           // root: [nranks][channels][chunk]
  bool nccl_reduce = false;
  ~Group();
};

std::string group_unique_id(void* id128);                                   // ncclGetUniqueId -> 128 bytes
std::string group_create(int nranks, int rank, const void* id128, int device, Group** out);
// Sum the banks' mixes: `mix_dev` [channels][mix_stride] holds this rank's partial for `n` samples and, on the root, the sum
// afterwards. Enqueued on bank.stream (no host synchronisation).
std::string group_reduce_device(Bank& b, Group& g, uint64_t n, float* mix_dev, uint64_t mix_stride, int root);
// render `n` samples of this rank's bank and reduce; `out_mix` [channels][n] (host) is written on the root only
std::string group_render_host(Bank& b, Group& g, uint64_t n, const float* in, float* out_mix, int root);

}  // namespace host
}  // namespace fdsp
