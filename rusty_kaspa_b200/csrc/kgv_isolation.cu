// kgv_isolation.cu — validate_tx_in_isolation, lock-time finality and the non-contextual masses for a batch (kgv_isolation.cuh), and
// the public call kgv_validate_txs_in_isolation.  kgv_validate_mempool_txs_in_parallel (kgv_validate.cu) runs the same launch first.
//
//   k_tx_isolation        one warp per tx : masses, then every rule in order; a tx with more than 32 inputs that reaches the
//                                           duplicate-input check is appended to a list instead of finishing
//   k_tx_isolation_large  one block per listed tx : sorts the (hash, input) pairs of its outpoints in shared memory (up to
//                                           ISO_SORT_MAX inputs), compares equal-hash neighbours exactly, then runs the remaining rules
#include "kgv_internal.h"
#include "kgv_isolation.cuh"

#include <cub/block/block_radix_sort.cuh>
#include <algorithm>
#include <cstdio>

using namespace kgv;

static_assert(sizeof(kgv_tx_rules) == 72, "kgv_tx_rules is 72 bytes");
static_assert(sizeof(kgv_tx_masses) == 16, "kgv_tx_masses is 16 bytes");


constexpr int ISO_WARPS = 4;            // transactions per block of k_tx_isolation
constexpr int ISO_LARGE_THREADS = 256;  // k_tx_isolation_large
constexpr int ISO_LARGE_ITEMS = 8;
constexpr uint32_t ISO_SORT_MAX = ISO_LARGE_THREADS * ISO_LARGE_ITEMS;  // 2048 >= mainnet's max_tx_inputs (1000)
constexpr uint32_t ISO_PAD = 0xFFFFFFFFu;

__global__ void __launch_bounds__(32 * ISO_WARPS)
k_tx_isolation(BatchView b, uint32_t n_txs, kgv_tx_rules r, IsoContext c, bool finality, kgv_tx_result* __restrict__ res,
               kgv_tx_masses* __restrict__ masses, uint64_t* __restrict__ nc_mass, uint32_t* __restrict__ large, uint32_t* __restrict__ n_large) {
  const uint32_t ti = blockIdx.x * ISO_WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (ti >= n_txs) return;  // uniform per warp
  const uint64_t daa = c.daa(ti), pmt = c.pmt(ti);
  const kgv_tx t = b.txs[ti];
  const bool cb = tx_is_coinbase(t);
  const kgv_tx_masses m = iso_masses(b, t, cb, r, lane);
  kgv_tx_result out = iso_head(b, t, cb, r, lane);
  if (out.status == KGV_TX_OK) {
    if (t.n_inputs > ISO_WARP_DUP_MAX) {
      if (lane == 0) large[atomicAdd(n_large, 1u)] = ti;  // k_tx_isolation_large finishes it
    } else if (iso_warp_duplicates(b, t, lane)) {
      out = iso_result(KGV_TX_DUPLICATE_INPUTS, 0);
    } else {
      out = iso_tail(b, t, cb, daa, pmt, finality, lane);
    }
  }
  if (lane == 0) {
    res[ti] = out;
    if (masses) masses[ti] = m;
    if (nc_mass) nc_mass[ti] = m.compute_mass > m.transient_mass ? m.compute_mass : m.transient_mass;
  }
}

// outpoints a and b (absolute input indices) are equal: all 36 bytes
__device__ __forceinline__ bool same_outpoint(const kgv_input* in, uint32_t a, uint32_t b) {
  uint32_t ka[9], kb[9];
  input_key(ka, in[a]);
  input_key(kb, in[b]);
  bool eq = true;
#pragma unroll
  for (int w = 0; w < 9; w++) eq = eq && ka[w] == kb[w];
  return eq;
}

// check_duplicate_transaction_inputs for the listed transactions (more than 32 inputs), then the rules after it.  Up to ISO_SORT_MAX
// inputs: a block radix sort of (key_hash, input) in shared memory, and every sorted neighbour run of equal hashes compared exactly.
// Above that (only with rules beyond mainnet's input limit) each input is compared with every earlier one: quadratic, exact.
__global__ void __launch_bounds__(ISO_LARGE_THREADS)
k_tx_isolation_large(BatchView b, kgv_tx_rules r, IsoContext c, bool finality, const uint32_t* __restrict__ large,
                     const uint32_t* __restrict__ n_large, kgv_tx_result* __restrict__ res) {
  using Sort = cub::BlockRadixSort<unsigned long long, ISO_LARGE_THREADS, ISO_LARGE_ITEMS, uint32_t>;
  __shared__ union {
    typename Sort::TempStorage sort;
    struct {
      unsigned long long h[ISO_SORT_MAX];
      uint32_t idx[ISO_SORT_MAX];
    } s;
  } sm;
  __shared__ int dup;
  const uint32_t n_list = *n_large;
  for (uint32_t li = blockIdx.x; li < n_list; li += gridDim.x) {
    const uint32_t ti = large[li];
    const kgv_tx t = b.txs[ti];
    const kgv_input* in = b.inputs + t.first_input;
    const uint32_t n = t.n_inputs;
    if (threadIdx.x == 0) dup = 0;
    __syncthreads();
    if (n <= ISO_SORT_MAX) {
      unsigned long long key[ISO_LARGE_ITEMS];
      uint32_t val[ISO_LARGE_ITEMS];
#pragma unroll
      for (int k = 0; k < ISO_LARGE_ITEMS; k++) {
        const uint32_t i = threadIdx.x * ISO_LARGE_ITEMS + k;
        key[k] = ~0ull;
        val[k] = ISO_PAD;
        if (i < n) {
          uint32_t w[9];
          input_key(w, in[i]);
          key[k] = key_hash(w);
          val[k] = i;
        }
      }
      Sort(sm.sort).Sort(key, val);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < ISO_LARGE_ITEMS; k++) {
        const uint32_t p = threadIdx.x * ISO_LARGE_ITEMS + k;
        sm.s.h[p] = key[k];
        sm.s.idx[p] = val[k];
      }
      __syncthreads();
      // each position compares itself with the earlier positions of its equal-hash run (padding may share the all-ones hash)
      for (uint32_t p = threadIdx.x + 1; p < ISO_SORT_MAX; p += ISO_LARGE_THREADS) {
        const unsigned long long hp = sm.s.h[p];
        const uint32_t ip = sm.s.idx[p];
        if (ip == ISO_PAD || sm.s.h[p - 1] != hp) continue;
        for (uint32_t q = p; q-- > 0 && sm.s.h[q] == hp;)
          if (sm.s.idx[q] != ISO_PAD && same_outpoint(in, ip, sm.s.idx[q])) { dup = 1; break; }
      }
    } else {
      for (uint32_t i = threadIdx.x; i < n && !dup; i += ISO_LARGE_THREADS)
        for (uint32_t j = 0; j < i; j++)
          if (same_outpoint(in, i, j)) { dup = 1; break; }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      const kgv_tx_result out = dup ? iso_result(KGV_TX_DUPLICATE_INPUTS, 0) : iso_tail(b, t, tx_is_coinbase(t), c.daa(ti), c.pmt(ti), finality, threadIdx.x);
      if (threadIdx.x == 0) res[ti] = out;
    }
    __syncthreads();  // sm and dup are reused by the next listed tx
  }
}

int kgv_isolation_run(kgv_ctx* ctx, const kgv_dev_batch& d, const kgv_tx_rules& rules, uint64_t daa, uint64_t pmt, bool finality, kgv_tx_result* dres,
                      kgv_tx_masses* dmasses, uint64_t* dnc, uint32_t* dlist, cudaStream_t st, const kgv_block_header_ctx* dheaders,
                      const uint32_t* dtx_block) {
  const size_t nt = d.n_txs;
  if (nt == 0) return KGV_OK;
  const IsoContext c{daa, pmt, dheaders, dtx_block};
  uint32_t* n_large = dlist + nt;
  CK(cudaMemsetAsync(n_large, 0, 4, st));
  const BatchView v{d.txs, d.inputs, d.outputs, nullptr, d.bytes};
  k_tx_isolation<<<(unsigned)((nt + ISO_WARPS - 1) / ISO_WARPS), 32 * ISO_WARPS, 0, st>>>(v, (uint32_t)nt, rules, c, finality, dres, dmasses, dnc,
                                                                                            dlist, n_large);
  CK(cudaGetLastError());
  // the list's length stays on the device: a fixed grid strides over it (blocks past its end return at once)
  const unsigned grid = (unsigned)std::min<size_t>(nt, 2 * 132);
  k_tx_isolation_large<<<grid, ISO_LARGE_THREADS, 0, st>>>(v, rules, c, finality, dlist, n_large, dres);
  CK(cudaGetLastError());
  ctx->launches += 2;
  return KGV_OK;
}

extern "C" int kgv_validate_txs_in_isolation(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_tx_rules* rules, uint64_t ctx_daa_score,
                                             uint64_t ctx_past_median_time, uint32_t flags, kgv_tx_result* results, kgv_tx_masses* masses) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || !rules || (batch->n_txs && !results)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (flags & ~KGV_ISOLATION_SKIP_FINALITY) { ctx->err = "kgv_validate_txs_in_isolation: unknown flags"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_validate_txs_in_isolation", "rules", rules)) return rc;
  if (batch->n_txs == 0) return KGV_OK;
  if (batch->n_txs > 0xFFFFFFFFull) { ctx->err = "kgv_validate_txs_in_isolation: more than 2^32 - 1 transactions"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_validate_txs_in_isolation", {results, batch->txs, masses})) return rc;
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  const size_t nt = d.n_txs;
  kgv_tx_result* dres;
  kgv_tx_masses* dm;
  io.out(results, nt * sizeof(kgv_tx_result), &dres);
  io.out(masses, nt * sizeof(kgv_tx_masses), &dm);
  if ((rc = io.stage())) return rc;
  if ((rc = kgv_reserve(ctx, &ctx->d_work, &ctx->d_work_cap, (nt + 1) * 4))) return rc;
  rc = kgv_isolation_run(ctx, d, *rules, ctx_daa_score, ctx_past_median_time, !(flags & KGV_ISOLATION_SKIP_FINALITY), dres, dm, nullptr,
                         (uint32_t*)ctx->d_work, ctx->stream);
  if (rc) return rc;
  return io.finish();
}
