// kgv_comm.cu — multi-GPU exchange of per-shard verdicts (K7; include/kgv.h "multi-GPU").
//
// Signature batches shard across GPUs as contiguous ranges of (signature, key) pairs (SURVEY.md §8e); the only exchange
// step of the whole path is "every rank ends up with every shard's verdicts".  Two transports behind one interface:
//
//   NCCL    ncclAllGather on the context's stream.  libnccl.so.2 is resolved at run time (dlopen) so that the library
//           loads - and every single-GPU entry point works - on hosts without NCCL; inside a process that already uses
//           NCCL (torch) the loader hands back that same library.
//   peer    the payload is tiny (a verdict bitmap is 128 KiB per million signatures), so a collective's rendezvous costs
//           more than its transfer (measured in round 1: 6 ms per step inside ncclAllGather at 8 ranks vs 0.07 ms at 4).
//           Here the kernel that PRODUCES a shard's verdicts (bitmap packing, or the verify kernels' status bytes) writes
//           them straight into every peer's receive buffer over NVLink (peer mappings: CUDA IPC across processes, direct
//           peer access inside one process), fences, and raises a per-source epoch flag in the peer's memory; consumers
//           wait on their LOCAL flags.  No host rendezvous, no extra kernel between producer and transfer; two receive
//           buffers alternate by epoch parity so a fast rank can be one epoch ahead.
#include "kgv_internal.h"

#include <dlfcn.h>

#include <cstdio>
#include <cstring>
#include <vector>

// ---------------------------------------------------------------------------------------------
// NCCL through dlopen (the five entry points used; signatures as in nccl.h 2.x)
// ---------------------------------------------------------------------------------------------
namespace {
struct nccl_uid { char internal[128]; };
typedef void* nccl_comm_t;
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(nccl_uid*) = nullptr;
  int (*CommInitRank)(nccl_comm_t*, int, nccl_uid, int) = nullptr;
  int (*CommDestroy)(nccl_comm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string why;
};
NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.lib) break;
    }
    if (!api.lib) { api.why = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : ""); return; }
    api.GetUniqueId = (int (*)(nccl_uid*))dlsym(api.lib, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(nccl_comm_t*, int, nccl_uid, int))dlsym(api.lib, "ncclCommInitRank");
    api.CommDestroy = (int (*)(nccl_comm_t))dlsym(api.lib, "ncclCommDestroy");
    api.AllGather = (int (*)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t))dlsym(api.lib, "ncclAllGather");
    api.GetErrorString = (const char* (*)(int))dlsym(api.lib, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather) { api.why = "libnccl lacks an expected symbol"; api.lib = nullptr; }
  });
  return api;
}
}  // namespace

#define KGV_P2P_MAX_RANKS 16

struct kgv_comm {
  kgv_ctx* ctx = nullptr;
  int n_ranks = 1, rank = 0;
  nccl_comm_t nccl = nullptr;
  // peer transport
  uint8_t* local = nullptr;            // [2][n_ranks][slice_cap] receive buffers, then [2][KGV_P2P_MAX_RANKS] u64 flags, then one u32 block counter
  size_t slice_cap = 0;
  uint8_t* peer[KGV_P2P_MAX_RANKS] = {};  // peer[r] = rank r's `local` mapped here (peer[rank] = local)
  bool peer_ipc[KGV_P2P_MAX_RANKS] = {};
  bool peers_open = false;
  uint64_t epoch = 0;                  // last published epoch
};

static size_t p2p_flags_off(const kgv_comm* c) { return (2 * (size_t)c->n_ranks * c->slice_cap + 255) & ~(size_t)255; }
static size_t p2p_total(const kgv_comm* c) { return p2p_flags_off(c) + 2 * KGV_P2P_MAX_RANKS * 8 + 256; }

struct P2PView {
  uint8_t* peer[KGV_P2P_MAX_RANKS];
  int n_ranks, rank;
  size_t slice_cap, flags_off;
};
static P2PView view_of(const kgv_comm* c) {
  P2PView v;
  for (int i = 0; i < KGV_P2P_MAX_RANKS; i++) v.peer[i] = c->peer[i];
  v.n_ranks = c->n_ranks; v.rank = c->rank; v.slice_cap = c->slice_cap; v.flags_off = p2p_flags_off(c);
  return v;
}

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// Fused producer + transfer: packs this rank's verdicts into its validity bitmap (bit i = status[i] == valid) and stores every
// 32-bit word of it into slot [epoch & 1][rank] of EVERY rank's receive buffer (its own included); the last block to finish
// raises the epoch flag of this source on every rank.
__global__ void __launch_bounds__(256) k_publish_bitmap(P2PView v, const uint8_t* __restrict__ status, size_t n, unsigned long long epoch, unsigned int* __restrict__ done_blocks) {
  const size_t n_words = (n + 31) / 32;
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w < n_words) {
    uint32_t bits = 0;
    const size_t base = 32 * w;
    if (base + 32 <= n && ((uintptr_t)(status + base) & 15) == 0) {
      const uint4* q = (const uint4*)(status + base);
#pragma unroll
      for (int k = 0; k < 2; k++) {
        uint4 x = q[k];
        uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
          for (int b = 0; b < 4; b++) bits |= (((xs[j] >> (8 * b)) & 0xFFu) == 1u ? 1u : 0u) << (16 * k + 4 * j + b);
      }
    } else {
      for (int j = 0; j < 32; j++) if (base + j < n && status[base + j] == 1) bits |= 1u << j;
    }
    const size_t slot = ((size_t)(epoch & 1) * v.n_ranks + v.rank) * v.slice_cap + 4 * w;
    for (int r = 0; r < v.n_ranks; r++) *(uint32_t*)(v.peer[r] + slot) = bits;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned prev = atomicAdd(done_blocks, 1u);
    if (prev == gridDim.x - 1) {
      *done_blocks = 0;
      __threadfence_system();
      for (int r = 0; r < v.n_ranks; r++)
        st_release_sys_u64((unsigned long long*)(v.peer[r] + v.flags_off) + (epoch & 1) * KGV_P2P_MAX_RANKS + v.rank, epoch);
    }
  }
}
// same for raw bytes (the status slices of a sharded script pre-check): copies src[0..nbytes) to offset dst_off of slot [epoch&1][rank]
__global__ void __launch_bounds__(256) k_publish_bytes(P2PView v, const uint8_t* __restrict__ src, size_t nbytes, unsigned long long epoch, unsigned int* __restrict__ done_blocks) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t slot = ((size_t)(epoch & 1) * v.n_ranks + v.rank) * v.slice_cap;
  if (i < nbytes) {
    const uint8_t x = src[i];
    for (int r = 0; r < v.n_ranks; r++) v.peer[r][slot + i] = x;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned prev = atomicAdd(done_blocks, 1u);
    if (prev == gridDim.x - 1) {
      *done_blocks = 0;
      __threadfence_system();
      for (int r = 0; r < v.n_ranks; r++)
        st_release_sys_u64((unsigned long long*)(v.peer[r] + v.flags_off) + (epoch & 1) * KGV_P2P_MAX_RANKS + v.rank, epoch);
    }
  }
}
// wait until every source has delivered `epoch` (flags live in local memory: the spin never crosses NVLink)
__global__ void k_wait_epoch(const unsigned long long* __restrict__ flags, int n_ranks, unsigned long long epoch) {
  const int r = threadIdx.x;
  if (r < n_ranks) {
    const unsigned long long* f = flags + (epoch & 1) * KGV_P2P_MAX_RANKS + r;
    while (ld_acquire_sys_u64(f) < epoch) __nanosleep(200);
  }
}
// gather the n_ranks slots of one epoch into a contiguous array (slot r -> out + r * nbytes)
__global__ void k_collect(const uint8_t* __restrict__ local, int n_ranks, size_t slice_cap, unsigned long long epoch, size_t nbytes, uint8_t* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)n_ranks * nbytes;
  if (i >= total) return;
  const size_t r = i / nbytes, o = i % nbytes;
  out[i] = __ldcg(local + ((size_t)(epoch & 1) * n_ranks + r) * slice_cap + o);
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" int kgv_comm_unique_id(uint8_t id[KGV_COMM_ID_BYTES]) {
  if (!id) return KGV_ERR_ARG;
  NcclApi& a = nccl();
  if (!a.lib) return KGV_ERR_NCCL;
  nccl_uid u;
  if (a.GetUniqueId(&u) != 0) return KGV_ERR_NCCL;
  memcpy(id, u.internal, 128);
  return KGV_OK;
}

extern "C" int kgv_comm_create(kgv_ctx* ctx, int n_ranks, int rank, const uint8_t* id, size_t slice_capacity_bytes, kgv_comm** out) {
  if (!ctx || !out || n_ranks < 1 || n_ranks > KGV_P2P_MAX_RANKS || rank < 0 || rank >= n_ranks) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  *out = nullptr;
  CK(cudaSetDevice(ctx->device));
  kgv_comm* c = new kgv_comm();
  c->ctx = ctx; c->n_ranks = n_ranks; c->rank = rank;
  if (id) {  // NCCL transport requested
    NcclApi& a = nccl();
    if (!a.lib) { ctx->err = "NCCL unavailable: " + a.why; delete c; return KGV_ERR_NCCL; }
    nccl_uid u;
    memcpy(u.internal, id, 128);
    int rc = a.CommInitRank(&c->nccl, n_ranks, u, rank);
    if (rc != 0) { ctx->err = std::string("ncclCommInitRank failed: ") + (a.GetErrorString ? a.GetErrorString(rc) : "?"); delete c; return KGV_ERR_NCCL; }
  }
  c->slice_cap = (slice_capacity_bytes + 255) & ~(size_t)255;
  if (c->slice_cap) {
    cudaError_t e = cudaMalloc((void**)&c->local, p2p_total(c));
    if (e != cudaSuccess) { ctx->err = std::string("cudaMalloc failed for the peer receive buffers: ") + cudaGetErrorString(e); (void)cudaGetLastError(); delete c; return KGV_ERR_NOMEM; }
    CK(cudaMemsetAsync(c->local, 0, p2p_total(c), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    c->peer[rank] = c->local;
  }
  *out = c;
  return KGV_OK;
}

extern "C" void kgv_comm_destroy(kgv_comm* c) {
  if (!c) return;
  kgv_ctx* ctx = c->ctx;
  if (ctx) { cudaSetDevice(ctx->device); cudaStreamSynchronize(ctx->stream); }
  for (int r = 0; r < c->n_ranks; r++)
    if (r != c->rank && c->peer[r] && c->peer_ipc[r]) cudaIpcCloseMemHandle(c->peer[r]);
  if (c->local) cudaFree(c->local);
  if (c->nccl) nccl().CommDestroy(c->nccl);
  delete c;
}

extern "C" int kgv_comm_export(kgv_comm* c, uint8_t handle[KGV_COMM_HANDLE_BYTES]) {
  if (!c || !handle || !c->local) return KGV_ERR_ARG;
  kgv_ctx* ctx = c->ctx;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  static_assert(sizeof(cudaIpcMemHandle_t) <= KGV_COMM_HANDLE_BYTES, "handle size");
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, c->local));
  memset(handle, 0, KGV_COMM_HANDLE_BYTES);
  memcpy(handle, &h, sizeof h);
  return KGV_OK;
}

extern "C" int kgv_comm_import(kgv_comm* c, const uint8_t* handles) {
  if (!c || !handles || !c->local) return KGV_ERR_ARG;
  kgv_ctx* ctx = c->ctx;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  for (int r = 0; r < c->n_ranks; r++) {
    if (r == c->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * KGV_COMM_HANDLE_BYTES, sizeof h);
    void* p = nullptr;
    CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer[r] = (uint8_t*)p;
    c->peer_ipc[r] = true;
  }
  c->peers_open = true;
  return KGV_OK;
}

// single-process form: the peers are communicators of other contexts of THIS process
extern "C" int kgv_comm_connect_local(kgv_comm* const* comms, int n) {
  if (!comms || n < 1 || n > KGV_P2P_MAX_RANKS) return KGV_ERR_ARG;
  for (int i = 0; i < n; i++) if (!comms[i] || comms[i]->n_ranks != n || comms[i]->rank != i || !comms[i]->local) return KGV_ERR_ARG;
  for (int i = 0; i < n; i++) {
    kgv_ctx* ctx = comms[i]->ctx;
    std::lock_guard<std::recursive_mutex> g(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    for (int j = 0; j < n; j++) {
      if (j == i) continue;
      if (comms[j]->ctx->device != ctx->device) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, ctx->device, comms[j]->ctx->device));
        if (!can) { ctx->err = "peer access between the devices is not possible"; return KGV_ERR_CUDA; }
        cudaError_t e = cudaDeviceEnablePeerAccess(comms[j]->ctx->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { ctx->err = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e); return KGV_ERR_CUDA; }
        (void)cudaGetLastError();
      }
      comms[i]->peer[j] = comms[j]->local;
    }
    comms[i]->peers_open = true;
  }
  return KGV_OK;
}

extern "C" int kgv_shard_allgather(kgv_ctx* ctx, kgv_comm* c, const uint8_t* local_shard, size_t nbytes_per_rank, uint8_t* all_shards) {
  if (!ctx || !c || c->ctx != ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!local_shard || !all_shards) { ctx->err = "null buffer"; return KGV_ERR_ARG; }
  if (!kgv_ptr_is_device(local_shard) || !kgv_ptr_is_device(all_shards)) { ctx->err = "kgv_shard_allgather: local_shard and all_shards must be device memory"; return KGV_ERR_ARG; }
  if (!c->nccl) { ctx->err = "communicator was created without the NCCL transport"; return KGV_ERR_NCCL; }
  CK(cudaSetDevice(ctx->device));
  int rc = nccl().AllGather(local_shard, all_shards, nbytes_per_rank, /*ncclUint8*/ 1, c->nccl, ctx->stream);
  if (rc != 0) { ctx->err = std::string("ncclAllGather failed: ") + (nccl().GetErrorString ? nccl().GetErrorString(rc) : "?"); return KGV_ERR_NCCL; }
  ctx->launches++;
  return KGV_OK;
}

static int p2p_ready(kgv_ctx* ctx, kgv_comm* c, size_t nbytes) {
  if (!c->local) { ctx->err = "communicator was created without peer receive buffers"; return KGV_ERR_ARG; }
  if (c->n_ranks > 1 && !c->peers_open) { ctx->err = "peer buffers not connected (kgv_comm_import / kgv_comm_connect_local)"; return KGV_ERR_ARG; }
  if (nbytes > c->slice_cap) { ctx->err = "shard larger than the communicator's slice capacity"; return KGV_ERR_ARG; }
  return KGV_OK;
}

extern "C" int kgv_shard_publish_bitmap(kgv_ctx* ctx, kgv_comm* c, const uint8_t* status, size_t n, uint64_t* epoch_out) {
  if (!ctx || !c || c->ctx != ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if ((n && !status) || !kgv_ptr_is_device(status)) { ctx->err = "kgv_shard_publish_bitmap: status must be device memory"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_shard_publish_bitmap", "epoch_out", epoch_out)) return rc;
  int rc = p2p_ready(ctx, c, 4 * ((n + 31) / 32));
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  const uint64_t e = ++c->epoch;
  const size_t n_words = (n + 31) / 32;
  unsigned blocks = (unsigned)((n_words + 255) / 256);
  if (blocks == 0) blocks = 1;
  unsigned int* ctr = (unsigned int*)(c->local + p2p_flags_off(c) + 2 * KGV_P2P_MAX_RANKS * 8);
  k_publish_bitmap<<<blocks, 256, 0, ctx->stream>>>(view_of(c), status, n, e, ctr);
  CK(cudaGetLastError());
  ctx->launches++;
  if (epoch_out) *epoch_out = e;
  return KGV_OK;
}

extern "C" int kgv_shard_publish_bytes(kgv_ctx* ctx, kgv_comm* c, const uint8_t* src, size_t nbytes, uint64_t* epoch_out) {
  if (!ctx || !c || c->ctx != ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if ((nbytes && !src) || (nbytes && !kgv_ptr_is_device(src))) { ctx->err = "kgv_shard_publish_bytes: src must be device memory"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_shard_publish_bytes", "epoch_out", epoch_out)) return rc;
  int rc = p2p_ready(ctx, c, nbytes);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  const uint64_t e = ++c->epoch;
  unsigned blocks = (unsigned)((nbytes + 255) / 256);
  if (blocks == 0) blocks = 1;
  unsigned int* ctr = (unsigned int*)(c->local + p2p_flags_off(c) + 2 * KGV_P2P_MAX_RANKS * 8);
  k_publish_bytes<<<blocks, 256, 0, ctx->stream>>>(view_of(c), src, nbytes, e, ctr);
  CK(cudaGetLastError());
  ctx->launches++;
  if (epoch_out) *epoch_out = e;
  return KGV_OK;
}

extern "C" int kgv_shard_wait(kgv_ctx* ctx, kgv_comm* c, uint64_t epoch, size_t nbytes_per_rank, uint8_t* all_shards) {
  if (!ctx || !c || c->ctx != ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  int rc = p2p_ready(ctx, c, nbytes_per_rank);
  if (rc) return rc;
  if (all_shards && !kgv_ptr_is_device(all_shards)) { ctx->err = "kgv_shard_wait: all_shards must be device memory"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  k_wait_epoch<<<1, 32, 0, ctx->stream>>>((const unsigned long long*)(c->local + p2p_flags_off(c)), c->n_ranks, epoch);
  CK(cudaGetLastError());
  ctx->launches++;
  if (all_shards && nbytes_per_rank) {
    const size_t total = (size_t)c->n_ranks * nbytes_per_rank;
    k_collect<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(c->local, c->n_ranks, c->slice_cap, epoch, nbytes_per_rank, all_shards);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  return KGV_OK;
}

extern "C" int kgv_set_sharding(kgv_ctx* ctx, kgv_comm* c) {
  if (!ctx || (c && c->ctx != ctx)) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  ctx->shard_comm = c;
  return KGV_OK;
}
int kgv_comm_ranks(const kgv_comm* c, int* rank) {
  if (rank) *rank = c->rank;
  return c->n_ranks;
}
int kgv_comm_exchange_slices(kgv_ctx* ctx, kgv_comm* c, uint8_t* buf, size_t per) {
  if (c->n_ranks == 1 || per == 0) return KGV_OK;
  if (c->local && c->peers_open && per <= c->slice_cap) {
    uint64_t e = 0;
    int rc = kgv_shard_publish_bytes(ctx, c, buf + (size_t)c->rank * per, per, &e);
    if (rc) return rc;
    return kgv_shard_wait(ctx, c, e, per, buf);
  }
  return kgv_shard_allgather(ctx, c, buf + (size_t)c->rank * per, per, buf);
}
