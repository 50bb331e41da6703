// kgv_block_body.cu — validate_body_in_isolation and validate_body_in_context for a window of blocks (kgv_validate_block_bodies), and the
// set checks kgv_block_set_checks shares with it.
//
// Whole-batch passes first: tx hashes -> merkle roots, tx ids, and the isolation / finality kernels with each transaction's own block
// context (kgv_hash.cu, kgv_isolation.cu).  Then one thread block per body, striding over the bodies of the call:
//   k_body_tx_block  the block index of every tx
//   k_body_sets      duplicate ids, double spends, chained transactions: insert into hashed sets, then look every item up; linear work
//   k_body_rules     coinbase position, first failing tx, the mass rule as a saturating scan with a carried prefix, the coinbase payload,
//                    and the choice of the first failing rule in the reference's order
#include "kgv_internal.h"
#include "kgv_block_body.cuh"

#include <cub/block/block_scan.cuh>
#include <algorithm>
#include <cstdio>
#include <random>

using namespace kgv;

static_assert(sizeof(kgv_block_header_ctx) == 64, "kgv_block_header_ctx is 64 bytes");
static_assert(sizeof(kgv_body_rules) == 16, "kgv_body_rules is 16 bytes");
static_assert(sizeof(kgv_body_result) == 32, "kgv_body_result is 32 bytes");
static_assert(sizeof(kgv_block_masses) == 24, "kgv_block_masses is 24 bytes");


constexpr int BODY_SET_THREADS = 256;
constexpr uint32_t BODY_SET_SMEM_SLOTS = 8192;  // 32 KiB: a body of up to 4096 transactions + inputs keeps both of its sets in shared memory
constexpr int BODY_RULE_THREADS = 128;
constexpr unsigned BODY_MAX_GRID = 132 * 8;     // bodies in flight; the rest are reached by striding

__global__ void k_body_tx_block(const uint32_t* __restrict__ first, uint32_t n_blocks, uint32_t* __restrict__ tx_block) {
  for (uint32_t b = blockIdx.x; b < n_blocks; b += gridDim.x)
    for (uint32_t t = first[b] + threadIdx.x; t < first[b + 1]; t += blockDim.x) tx_block[t] = b;
}

// Set A: the tx ids of the body (2 slots per tx).  Set B: the outpoints its inputs spend (2 slots per input).  Both live in shared memory
// when they fit and in the body's own slice of gtab otherwise (slots [2 * t0, 2 * t1) of the first part, [2 * i0, 2 * i1) of the second;
// gtab arrives filled with BODY_NONE).  Where a set lives changes no result: every comparison is of the full 32 / 36 bytes.
__global__ void __launch_bounds__(BODY_SET_THREADS)
k_body_sets(const kgv_tx* __restrict__ txs, const kgv_input* __restrict__ inputs, const uint64_t* __restrict__ ids, const uint32_t* __restrict__ first,
            uint32_t n_blocks, uint32_t n_txs, uint64_t salt, kgv_block_check_acc* __restrict__ acc, uint32_t* __restrict__ gtab) {
  __shared__ uint32_t stab[BODY_SET_SMEM_SLOTS];
  __shared__ uint32_t s_acc[3];
  for (uint32_t b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    const uint32_t t0 = first[b], t1 = first[b + 1];
    if (t0 == t1) continue;  // uniform
    const uint32_t i0 = txs[t0].first_input, i1 = txs[t1 - 1].first_input + txs[t1 - 1].n_inputs;
    const uint64_t ca64 = 2ull * (t1 - t0), cb64 = 2ull * (i1 - i0);
    const bool in_smem = ca64 + cb64 <= BODY_SET_SMEM_SLOTS;
    const uint32_t ca = (uint32_t)ca64, cb = (uint32_t)cb64;  // fewer than 2^31 items: a larger batch cannot be staged
    uint32_t* set_a = in_smem ? stab : gtab + 2 * (size_t)t0;
    uint32_t* set_b = in_smem ? stab + ca : gtab + 2 * (size_t)n_txs + 2 * (size_t)i0;
    if (in_smem)
      for (uint32_t k = threadIdx.x; k < ca + cb; k += BODY_SET_THREADS) stab[k] = BODY_NONE;
    if (threadIdx.x < 3) s_acc[threadIdx.x] = BODY_NONE;
    __syncthreads();
    for (uint32_t t = t0 + threadIdx.x; t < t1; t += BODY_SET_THREADS) {
      const uint64_t* id = ids + 4 * (size_t)t;
      body_set_insert(set_a, ca, body_hash_id(id, salt), t, [&](uint32_t j) { return body_same_id(ids + 4 * (size_t)j, id); });
    }
    for (uint32_t i = i0 + threadIdx.x; i < i1; i += BODY_SET_THREADS) {
      body_set_insert(set_b, cb, body_hash_outpoint(inputs[i], salt), i, [&](uint32_t j) { return body_same_outpoint(inputs[j], inputs[i]); });
    }
    __syncthreads();
    // check_duplicate_transactions: the first tx whose id an earlier tx has
    for (uint32_t t = t0 + threadIdx.x; t < t1; t += BODY_SET_THREADS) {
      const uint64_t* id = ids + 4 * (size_t)t;
      if (body_set_find(set_a, ca, body_hash_id(id, salt), [&](uint32_t j) { return body_same_id(ids + 4 * (size_t)j, id); }) < t) atomicMin(&s_acc[0], t);
    }
    for (uint32_t i = i0 + threadIdx.x; i < i1; i += BODY_SET_THREADS) {
      // check_block_double_spends: the first input whose outpoint an earlier input spends
      if (body_set_find(set_b, cb, body_hash_outpoint(inputs[i], salt), [&](uint32_t j) { return body_same_outpoint(inputs[j], inputs[i]); }) < i) atomicMin(&s_acc[1], i);
      // check_no_chained_transactions: the first input spending an output some tx of this body creates
      const uint64_t* pid = reinterpret_cast<const uint64_t*>(inputs[i].prev_txid);
      const uint32_t j = body_set_find(set_a, ca, body_hash_id(pid, salt), [&](uint32_t x) { return body_same_id(ids + 4 * (size_t)x, pid); });
      if (j != BODY_NONE && inputs[i].prev_index < txs[j].n_outputs) atomicMin(&s_acc[2], i);
    }
    __syncthreads();
    if (threadIdx.x == 0) acc[b] = kgv_block_check_acc{s_acc[0], s_acc[1], s_acc[2]};
    __syncthreads();  // stab and s_acc are reused by the next body
  }
}

void kgv_body_sets_work::carve(kgv_carve& c, size_t n_txs, size_t n_inputs) {
  const size_t at = c.at;
  tab = c.take<uint32_t>(2 * (n_txs + n_inputs));
  bytes = c.at - at;
}

int kgv_body_sets_run(kgv_ctx* ctx, const kgv_dev_batch& d, size_t n_txs, const uint64_t* dids, const uint32_t* dfirst, uint32_t n_blocks,
                      kgv_block_check_acc* dacc, const kgv_body_sets_work& w, cudaStream_t st) {
  // the key of the sets' hashes (body_hash_id / body_hash_outpoint), drawn once per process; the verdicts do not depend on it
  static const uint64_t salt = [] { std::random_device r; return (uint64_t)r() << 32 | r(); }();
  if (n_blocks == 0 || n_txs == 0) return KGV_OK;
  CK(cudaMemsetAsync(w.tab, 0xFF, w.bytes, st));
  k_body_sets<<<std::min(n_blocks, BODY_MAX_GRID), BODY_SET_THREADS, 0, st>>>(d.txs, d.inputs, dids, dfirst, n_blocks, (uint32_t)n_txs, salt, dacc, w.tab);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

struct BodyArgs {
  const kgv_tx* txs;
  const uint8_t* bytes;
  const uint32_t* first;
  const kgv_block_header_ctx* headers;
  const uint64_t* roots;
  const kgv_tx_result* tx_res;
  const kgv_tx_masses* tx_masses;
  const kgv_block_check_acc* acc;
  uint32_t n_blocks;
  bool isolation_only;
  uint64_t max_block_mass, max_coinbase_payload_len, max_coinbase_spk_len;
};

__global__ void __launch_bounds__(BODY_RULE_THREADS) k_body_rules(BodyArgs a, kgv_body_result* __restrict__ results, kgv_block_masses* __restrict__ masses) {
  using Scan = cub::BlockScan<BodyMass, BODY_RULE_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ uint32_t s_first[4];  // lowest position of: a coinbase after the first tx, an isolation failure, a mass excess, a tx that is not final
  __shared__ BodyMass s_excess;    // the running totals at the mass offender
  for (uint32_t b = blockIdx.x; b < a.n_blocks; b += gridDim.x) {
    const uint32_t t0 = a.first[b], n = a.first[b + 1] - t0;
    if (threadIdx.x < 4) s_first[threadIdx.x] = BODY_NONE;
    __syncthreads();
    BodyMass carry{0, 0, 0}, my_excess{0, 0, 0};
    uint32_t my_first_excess = BODY_NONE;
    for (uint32_t base = 0; base < n; base += BODY_RULE_THREADS) {
      const uint32_t p = base + threadIdx.x;
      BodyMass v{0, 0, 0};
      if (p < n) {
        const kgv_tx& t = a.txs[t0 + p];
        const uint8_t st = a.tx_res[t0 + p].status;
        if (p > 0 && tx_is_coinbase(t)) atomicMin(&s_first[0], p - 1);  // transactions[1..].position(is_coinbase)
        if (st == KGV_TX_NOT_FINALIZED) atomicMin(&s_first[3], p);
        else if (st != KGV_TX_OK) atomicMin(&s_first[1], p);
        v = BodyMass{a.tx_masses[t0 + p].compute_mass, a.tx_masses[t0 + p].transient_mass, t.mass};
      }
      BodyMass incl, chunk;
      Scan(scan_tmp).InclusiveScan(v, incl, BodyMassAdd(), chunk);
      incl = BodyMassAdd()(carry, incl);
      // the totals only grow, so a thread's first excess is its lowest, and the lowest over the threads is the reference's offender
      if (p < n && my_first_excess == BODY_NONE && (incl.compute > a.max_block_mass || incl.transient > a.max_block_mass || incl.storage > a.max_block_mass)) {
        my_first_excess = p;
        my_excess = incl;
        atomicMin(&s_first[2], p);
      }
      carry = BodyMassAdd()(carry, chunk);
      __syncthreads();  // scan_tmp is reused by the next chunk
    }
    __syncthreads();
    if (my_first_excess != BODY_NONE && my_first_excess == s_first[2]) s_excess = my_excess;
    __syncthreads();
    if (threadIdx.x == 0) {
      kgv_body_result r;
      r.status = KGV_BODY_OK; r.index = r.tx_status = r.fail_input = 0; r.a = r.b = 0;
      const kgv_block_header_ctx& h = a.headers[b];
      const uint64_t* want = reinterpret_cast<const uint64_t*>(h.hash_merkle_root);
      const kgv_block_check_acc sets = a.acc[b];
      if (n == 0) {
        r.status = KGV_BODY_NO_TRANSACTIONS;
      } else if (!body_same_id(want, a.roots + 4 * (size_t)b)) {
        r.status = KGV_BODY_BAD_MERKLE_ROOT;
      } else if (!tx_is_coinbase(a.txs[t0])) {
        r.status = KGV_BODY_FIRST_TX_NOT_COINBASE;
      } else if (s_first[0] != BODY_NONE) {
        r.status = KGV_BODY_MULTIPLE_COINBASES; r.index = s_first[0];
      } else if (s_first[1] != BODY_NONE) {
        const kgv_tx_result tr = a.tx_res[t0 + s_first[1]];
        r.status = KGV_BODY_TX_IN_ISOLATION_FAILED; r.index = s_first[1]; r.tx_status = tr.status; r.fail_input = tr.fail_input;
      } else if (s_first[2] != BODY_NONE) {
        r.index = s_first[2]; r.b = a.max_block_mass;
        if (s_excess.compute > a.max_block_mass) { r.status = KGV_BODY_EXCEEDS_COMPUTE_MASS_LIMIT; r.a = s_excess.compute; }
        else if (s_excess.transient > a.max_block_mass) { r.status = KGV_BODY_EXCEEDS_TRANSIENT_MASS_LIMIT; r.a = s_excess.transient; }
        else { r.status = KGV_BODY_EXCEEDS_STORAGE_MASS_LIMIT; r.a = s_excess.storage; }
      } else if (sets.dup_tx != BODY_NONE) {
        r.status = KGV_BODY_DUPLICATE_TRANSACTIONS; r.index = sets.dup_tx;
      } else if (sets.double_spend != BODY_NONE) {
        r.status = KGV_BODY_DOUBLE_SPEND_IN_SAME_BLOCK; r.index = sets.double_spend;
      } else if (sets.chained != BODY_NONE) {
        r.status = KGV_BODY_CHAINED_TRANSACTION; r.index = sets.chained;
      } else if (!a.isolation_only) {
        const kgv_tx& cb = a.txs[t0];
        body_coinbase_payload(r, a.bytes + cb.payload_off, cb.payload_len, h, a.max_coinbase_payload_len, a.max_coinbase_spk_len);
        if (r.status == KGV_BODY_OK && s_first[3] != BODY_NONE) {
          r.status = KGV_BODY_TX_IN_CONTEXT_FAILED; r.index = s_first[3]; r.tx_status = KGV_TX_NOT_FINALIZED; r.fail_input = a.tx_res[t0 + s_first[3]].fail_input;
        }
      }
      results[b] = r;
      if (masses) masses[b] = r.status == KGV_BODY_OK ? kgv_block_masses{carry.compute, carry.transient, carry.storage} : kgv_block_masses{0, 0, 0};
    }
    __syncthreads();  // s_first is reset for the next body
  }
}

extern "C" int kgv_validate_block_bodies(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* block_first_tx, uint32_t n_blocks,
                                         const kgv_block_header_ctx* headers, const kgv_tx_rules* rules, const kgv_body_rules* body_rules, uint32_t flags,
                                         kgv_body_result* results, kgv_block_masses* masses, uint8_t* roots32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (flags & ~KGV_BODY_ISOLATION_ONLY) { ctx->err = "kgv_validate_block_bodies: unknown flags"; return KGV_ERR_ARG; }
  if (n_blocks == 0) return KGV_OK;
  if (!batch || !block_first_tx || !headers || !rules || !body_rules || !results) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"block_first_tx", block_first_tx}, {"rules", rules}, {"body_rules", body_rules}})
    if (int rc = kgv_host_only(ctx, "kgv_validate_block_bodies", what, p)) return rc;
  if (batch->n_txs > 0xFFFFFFFFull || batch->n_inputs > 0x7FFFFFFFull) { ctx->err = "kgv_validate_block_bodies: more than 2^32 - 1 transactions or 2^31 - 1 inputs"; return KGV_ERR_ARG; }
  if (block_first_tx[0] != 0 || block_first_tx[n_blocks] != batch->n_txs) { ctx->err = "block offsets must start at 0 and end at the number of transactions"; return KGV_ERR_ARG; }
  for (uint32_t b = 0; b < n_blocks; b++)
    if (block_first_tx[b + 1] < block_first_tx[b]) { ctx->err = "block offsets not monotone"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_validate_block_bodies", {results, batch->txs, headers, masses, roots32})) return rc;
  kgv_dev_batch d{};
  if (batch->n_txs) {
    int rc = kgv_batch_to_device(ctx, batch, &d, false);
    if (rc) return rc;
  }
  const size_t nt = d.n_txs, nb = n_blocks;
  // tx hashes (consumed by the merkle tree) and the roots: d_in; everything else: d_work (the merkle tree owns d_scratch)
  uint64_t *dhash, *droots;  // droots is copied out below: roots32 is a byte array of any alignment
  int rc = kgv_reserve_carved(ctx, &ctx->d_in, &ctx->d_in_cap, [&](kgv_carve& c) { dhash = c.take<uint64_t>(nt * 4, 32); droots = c.take<uint64_t>(nb * 4); });
  if (rc) return rc;
  uint32_t *dfirst, *dtxb, *dlist;
  kgv_tx_result* dtxr;
  kgv_tx_masses* dtxm;
  uint64_t* dids;
  kgv_block_check_acc* dacc;
  kgv_body_sets_work sets;
  rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap, [&](kgv_carve& c) {
    dfirst = c.take<uint32_t>(nb + 1); dtxb = c.take<uint32_t>(nt); dtxr = c.take<kgv_tx_result>(nt); dtxm = c.take<kgv_tx_masses>(nt);
    dlist = c.take<uint32_t>(nt + 1); dids = c.take<uint64_t>(nt * 4); dacc = c.take<kgv_block_check_acc>(nb); sets.carve(c, nt, d.n_inputs);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const kgv_block_header_ctx* dhdr;
  kgv_body_result* dres;
  kgv_block_masses* dbm;
  io.in(headers, nb * sizeof(kgv_block_header_ctx), &dhdr);
  io.out(results, nb * sizeof(kgv_body_result), &dres);
  io.out(masses, nb * sizeof(kgv_block_masses), &dbm);
  if ((rc = io.stage())) return rc;
  CK(cudaMemcpyAsync(dfirst, block_first_tx, (nb + 1) * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(dacc, 0xFF, nb * sizeof(kgv_block_check_acc), st));
  const unsigned grid = std::min(n_blocks, BODY_MAX_GRID);
  const bool isolation_only = (flags & KGV_BODY_ISOLATION_ONLY) != 0;
  if (nt) {
    k_body_tx_block<<<grid, 128, 0, st>>>(dfirst, n_blocks, dtxb);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  if ((rc = kgv_tx_digests_run(ctx, d, nt, dhash, true))) return rc;
  if ((rc = kgv_merkle_run(ctx, dhash, nt, block_first_tx, n_blocks, droots))) return rc;
  if ((rc = kgv_tx_digests_run(ctx, d, nt, dids, false))) return rc;
  if ((rc = kgv_isolation_run(ctx, d, *rules, 0, 0, !isolation_only, dtxr, dtxm, nullptr, dlist, st, dhdr, dtxb))) return rc;
  if ((rc = kgv_body_sets_run(ctx, d, nt, dids, dfirst, n_blocks, dacc, sets, st))) return rc;
  const BodyArgs a{d.txs, d.bytes, dfirst, dhdr, droots, dtxr, dtxm, dacc, n_blocks, isolation_only, body_rules->max_block_mass,
                   body_rules->max_coinbase_payload_len, rules->coinbase_payload_script_public_key_max_len};
  k_body_rules<<<grid, BODY_RULE_THREADS, 0, st>>>(a, dres, dbm);
  CK(cudaGetLastError());
  ctx->launches++;
  if (roots32 && (rc = io.copy_out(roots32, droots, nb * 32))) return rc;
  return io.finish();
}
