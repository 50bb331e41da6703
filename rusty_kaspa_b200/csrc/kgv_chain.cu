// kgv_chain.cu — kgv_replay_verify_chain: verify_expected_utxo_state (utxo_validation.rs:182-228) for every chain block of the last
// kgv_replay_window call, with the mergeset rewards and accepted ids calculate_utxo_state (:110-173) gathers.  Everything it reads is the
// window state kgv_replay_window leaves in d_replay (tx ids, accept mask, per-tx results, the staged batch); nothing goes back to the host
// between the stages:
//   k_chain_blocks    one warp per window block: its total fees (with the overflow the reference panics on), its coinbase payload parse, and
//                     the accepted-id flag of each of its transactions
//   scan + compact    the accepted ids of the whole window in window order; each group is a contiguous run of them (a VERIFY_ONLY block
//                     accepts nothing), whose device offsets feed the merkle builder of kgv_hash.cu
//   MuHash            the per-group multisets of kgv_replay_muhash, the prefix combine with init768 and one batched finalize (kgv_muhash.cu)
//   k_chain_verdict   one warp per chain block: the first panic among its merged blocks, checks 1 and 2, the expected coinbase (kgv_chain.cuh)
//                     against the actual one, and check 5's count
#include "kgv_internal.h"
#include "kgv_chain.cuh"
#include "kgv_muhash.cuh"

#include <cstdio>

using namespace kgv;

static_assert(sizeof(kgv_chain_header) == 112, "kgv_chain_header is 112 bytes");
static_assert(sizeof(kgv_chain_result) == 112, "kgv_chain_result is 112 bytes");


constexpr int CHAIN_BLOCK_WARPS = 4;

struct ChainArgs {
  BatchView v;                   // the window's staged batch (entries unused)
  const kgv_replay_block* blk;   // the window's blocks
  const kgv_tx_result* res;      // per-tx results of the window
  const uint8_t* accept;
  const uint64_t* ids;           // tx ids, 4 words each
  const uint32_t* gf;            // n_groups + 1 block offsets
  uint32_t n_groups, nt;
  const kgv_chain_header* hdr;
  const uint8_t* mflags;         // KGV_MERGED_* per block
  uint64_t max_payload_len, max_spk_len;
  uint64_t* fee;                 // per block: total_fees
  uint8_t* code;                 // per block: the calculate_utxo_state panic it causes (KGV_CHAIN_*), 0 if none
  uint32_t* flag;                // per tx: 1 = its id is in the group's accepted ids
  const uint32_t* scan;          // exclusive scan of flag
  const uint32_t* n_ids;         // its total
  uint64_t* comp;                // compacted accepted ids
  uint32_t* id_first;            // per group (n_groups + 1): first accepted id
  const uint64_t* inner;         // per group: calc_merkle_root(accepted ids), 4 words
  const uint32_t* commit;        // per group: the finalized multiset, 8 words
  kgv_chain_result* out;
};

__device__ __forceinline__ uint32_t payload_parse_code(const ChainArgs& a, const kgv_replay_block& bl, CoinbasePayload& c) {
  if (bl.n_txs == 0) return KGV_CHAIN_COINBASE_PAYLOAD_UNPARSABLE;  // no txs[0] to read
  const kgv_tx& cb = a.v.txs[bl.first_tx];
  uint64_t x, y;
  return coinbase_payload_parse(c, a.v.bytes + cb.payload_off, cb.payload_len, a.max_payload_len, a.max_spk_len, x, y) ? KGV_CHAIN_COINBASE_PAYLOAD_UNPARSABLE : 0u;
}

// one CTA per group, one warp per block of it
__global__ void __launch_bounds__(32 * CHAIN_BLOCK_WARPS) k_chain_blocks(ChainArgs a) {
  const uint32_t g = blockIdx.x, lane = threadIdx.x & 31;
  const uint32_t b0 = a.gf[g], b1 = a.gf[g + 1];
  for (uint32_t b = b0 + (threadIdx.x >> 5); b < b1; b += CHAIN_BLOCK_WARPS) {
    const kgv_replay_block bl = a.blk[b];
    const uint32_t t0 = bl.first_tx, t1 = bl.first_tx + bl.n_txs;
    const bool merged = !(bl.flags & KGV_REPLAY_VERIFY_ONLY);
    uint64_t sum = 0;
    bool ovf = false;
    for (uint32_t t = t0 + lane; t < t1; t += 32) {
      const bool acc = merged && a.accept[t];
      // ctx.accepted_tx_ids: the selected parent's coinbase, then the accepted non-coinbase transactions
      a.flag[t] = acc && (t > t0 || b == b0);
      if (acc && t > t0) {
        const uint64_t f = a.res[t].fee;
        ovf |= sum + f < sum;
        sum += f;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t s2 = __shfl_down_sync(0xFFFFFFFFu, sum, o);
      const bool o2 = __shfl_down_sync(0xFFFFFFFFu, (int)ovf, o) != 0;
      ovf |= o2 || sum + s2 < sum;
      sum += s2;
    }
    if (lane == 0) {
      uint8_t c = 0;
      if (merged) {  // calculate_utxo_state: block_fee += ... (:147), then deserialize_coinbase_payload(&txs[0].payload).unwrap() (:163)
        CoinbasePayload p;
        c = ovf ? KGV_CHAIN_REWARD_OVERFLOW : (uint8_t)payload_parse_code(a, bl, p);
      }
      a.fee[b] = merged ? sum : 0;
      a.code[b] = c;
    }
  }
}

__global__ void k_chain_compact(ChainArgs a) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.nt || !a.flag[t]) return;
  const uint32_t j = a.scan[t];
#pragma unroll
  for (int k = 0; k < 4; k++) a.comp[4 * (size_t)j + k] = a.ids[4 * (size_t)t + k];
}
__global__ void k_chain_id_first(ChainArgs a) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > a.n_groups) return;
  const uint32_t t = g < a.n_groups ? a.blk[a.gf[g]].first_tx : a.nt;
  a.id_first[g] = t < a.nt ? a.scan[t] : *a.n_ids;
}

// The expected coinbase of the chain block whose mergeset is blocks b0 .. b0 + n - 1 (all of them parsed and summed without a panic).  Kept
// out of line: its hasher is live across the payload reads, and the caller hashes the actual coinbase with a second one (DESIGN.md §6).
__device__ __noinline__ bool chain_expected_coinbase(uint64_t* out4, const kgv_tx* txs, const uint8_t* bytes, const kgv_replay_block* blk, const uint64_t* fee,
                                                     const uint8_t* mflags, uint32_t b0, uint32_t n, uint64_t blue_score, uint64_t expected_subsidy,
                                                     const uint8_t* miner_payload, uint32_t miner_payload_len, CoinbasePayload miner) {
  auto rw = [&](uint32_t j) {
    const uint32_t b = b0 + j;
    const kgv_tx& cb = txs[blk[b].first_tx];
    const uint8_t* p = bytes + cb.payload_off;
    MergedReward r;
    r.subsidy = le64(p + 8);
    r.fees = fee[b];
    r.spk_version = (uint32_t)p[16] | (uint32_t)p[17] << 8;
    r.script_len = p[18];
    r.script = p + COINBASE_MIN_PAYLOAD_LENGTH;
    r.flags = mflags[b];
    return r;
  };
  return expected_coinbase_hash(out4, n, rw, blue_score, expected_subsidy, miner_payload, miner_payload_len, miner);
}

__device__ __forceinline__ void store_words(uint8_t* dst, const uint32_t* w) {  // dst is 4-byte aligned
#pragma unroll
  for (int k = 0; k < 8; k++) reinterpret_cast<uint32_t*>(dst)[k] = w[k];
}
__device__ __forceinline__ bool same32(const uint8_t* hdr_bytes, const uint32_t* w) {  // hdr_bytes is 8-byte aligned
  bool eq = true;
#pragma unroll
  for (int k = 0; k < 8; k++) eq &= reinterpret_cast<const uint32_t*>(hdr_bytes)[k] == w[k];
  return eq;
}

// one warp per group
__global__ void __launch_bounds__(128) k_chain_verdict(ChainArgs a) {
  const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (g >= a.n_groups) return;
  const uint32_t b0 = a.gf[g], bt = a.gf[g + 1] - 1;  // merged blocks b0 .. bt - 1, the chain block's body bt
  // the first panic of calculate_utxo_state, in merge order
  uint32_t calc = 0;
  for (uint32_t base = b0; base < bt; base += 32) {
    const uint32_t b = base + lane;
    const uint32_t c = b < bt ? a.code[b] : 0u;
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, c != 0);
    if (m) { calc = __shfl_sync(0xFFFFFFFFu, c, __ffs(m) - 1); break; }
  }
  // check 5: the chain block's own transactions against its UTXO view (the VERIFY_ONLY block's verdicts)
  const kgv_replay_block tail = a.blk[bt];
  uint32_t n_invalid = 0;
  const uint32_t t_end = tail.first_tx + tail.n_txs;
  for (uint32_t base = tail.first_tx + 1; base < t_end; base += 32) {
    const uint32_t t = base + lane;
    const bool bad = t < t_end && a.res[t].status != KGV_TX_OK;
    n_invalid += __popc(__ballot_sync(0xFFFFFFFFu, bad));
  }
  if (lane != 0) return;
  const kgv_chain_header& h = a.hdr[g];
  kgv_chain_result& r = a.out[g];
  r.n_invalid_txs = n_invalid;
  r.n_txs = tail.n_txs ? tail.n_txs - 1 : 0;
  r.pad_ = 0;
  // 1: the commitment
  uint32_t w[8];
#pragma unroll
  for (int k = 0; k < 8; k++) w[k] = a.commit[8 * (size_t)g + k];
  store_words(r.utxo_commitment, w);
  const bool commit_ok = same32(h.utxo_commitment, w);
  // 2: merkle_hash(selected parent's accepted_id_merkle_root, calc_merkle_root(accepted ids))
  uint64_t d[4];
  {
    Blake2b m;
    b2b_init_keyed_words(m, 0x7242656C6B72654Dull, 0x6873614868636E61ull, 16);  // "MerkleBranchHash"
#pragma unroll
    for (int k = 0; k < 4; k++) b2b_u64(m, le64(h.selected_parent_accepted_id_merkle_root + 8 * k));
#pragma unroll
    for (int k = 0; k < 4; k++) b2b_u64(m, a.inner[4 * (size_t)g + k]);
    b2b_final(m, d);
  }
#pragma unroll
  for (int k = 0; k < 4; k++) { w[2 * k] = (uint32_t)d[k]; w[2 * k + 1] = (uint32_t)(d[k] >> 32); }
  store_words(r.accepted_id_merkle_root, w);
  const bool root_ok = same32(h.accepted_id_merkle_root, w);
  // 4: verify_coinbase_transaction - the chain block's miner data (unwrap), expected_coinbase_transaction (unwrap), the two hashes
  CoinbasePayload miner;
  const uint32_t miner_code = payload_parse_code(a, tail, miner);
  bool built = false, cb_ok = false;
#pragma unroll
  for (int k = 0; k < 8; k++) w[k] = 0;
  if (calc == 0 && miner_code == 0) {
    const kgv_tx& cb = a.v.txs[tail.first_tx];
    built = chain_expected_coinbase(d, a.v.txs, a.v.bytes, a.blk, a.fee, a.mflags, b0, bt - b0, h.blue_score, h.expected_subsidy, a.v.bytes + cb.payload_off,
                                    cb.payload_len, miner);
    if (built) {
#pragma unroll
      for (int k = 0; k < 4; k++) { w[2 * k] = (uint32_t)d[k]; w[2 * k + 1] = (uint32_t)(d[k] >> 32); }
      uint64_t e[4];
      tx_hash(e, a.v, tail.first_tx);
      cb_ok = e[0] == d[0] && e[1] == d[1] && e[2] == d[2] && e[3] == d[3];
    }
  }
  store_words(r.coinbase_hash, w);
  uint32_t st = calc;
  if (!st) st = !commit_ok ? KGV_CHAIN_BAD_UTXO_COMMITMENT
                : !root_ok ? KGV_CHAIN_BAD_ACCEPTED_ID_MERKLE_ROOT
                : miner_code ? miner_code
                : !built ? KGV_CHAIN_REWARD_OVERFLOW
                : !cb_ok ? KGV_CHAIN_BAD_COINBASE_TRANSACTION : KGV_CHAIN_OK;
  r.status = st;
}

extern "C" int kgv_replay_verify_chain(kgv_ctx* ctx, const uint32_t* group_first_block, size_t n_groups, const kgv_chain_header* headers,
                                       const uint8_t* merged_flags, const uint8_t* init768, const kgv_tx_rules* rules, const kgv_body_rules* body_rules,
                                       kgv_chain_result* results, uint64_t* block_fees, uint8_t* multisets768) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> lk(ctx->mu);
  if (n_groups == 0) { ctx->err = "kgv_replay_verify_chain: no groups (the groups must tile the window, which has at least one block)"; return KGV_ERR_ARG; }
  if (!group_first_block || !headers || !merged_flags || !init768 || !rules || !body_rules || !results) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (!ctx->last_replay.valid) {
    ctx->err = "kgv_replay_verify_chain refers to the last kgv_replay_window call, and none is current (another batch was staged or the table rehashed since)";
    return KGV_ERR_ARG;
  }
  const auto& L = ctx->last_replay;
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"group_first_block", group_first_block}, {"rules", rules}, {"body_rules", body_rules}})
    if (int rc = kgv_host_only(ctx, "kgv_replay_verify_chain", what, p)) return rc;
  if (group_first_block[0] != 0 || group_first_block[n_groups] != L.n_blocks) { ctx->err = "groups must tile the blocks of the window"; return KGV_ERR_ARG; }
  // group layout: the selected parent (ACCEPT_COINBASE), the rest of the mergeset, the chain block's body (VERIFY_ONLY) last and only there
  uint32_t max_ids = 0;
  for (size_t g = 0; g < n_groups; g++) {
    const uint32_t b0 = group_first_block[g], b1 = group_first_block[g + 1];
    if (b1 < b0 + 2) { ctx->err = "a group holds at least its selected parent and the chain block's body"; return KGV_ERR_ARG; }
    if (!(L.block_flags[b0] & KGV_REPLAY_ACCEPT_COINBASE)) { ctx->err = "the first block of a group must be its selected parent (KGV_REPLAY_ACCEPT_COINBASE)"; return KGV_ERR_ARG; }
    if (!(L.block_flags[b1 - 1] & KGV_REPLAY_VERIFY_ONLY)) { ctx->err = "the last block of a group must be the chain block's body (KGV_REPLAY_VERIFY_ONLY)"; return KGV_ERR_ARG; }
    uint64_t n = 0;
    for (uint32_t b = b0; b + 1 < b1; b++) {
      if (L.block_flags[b] & KGV_REPLAY_VERIFY_ONLY) { ctx->err = "only the last block of a group may be KGV_REPLAY_VERIFY_ONLY"; return KGV_ERR_ARG; }
      n += L.block_n_txs[b];
    }
    if (n > max_ids) max_ids = (uint32_t)n;
  }
  kgv_io io(ctx);
  bool dev;
  if (int rc = io.one_side("kgv_replay_verify_chain", {results, headers, merged_flags, init768, block_fees, multisets768}, &dev)) return rc;
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = kgv_last_replay_read(ctx, acc, "kgv_replay_verify_chain")) return rc;
  cudaStream_t st = ctx->stream;
  const cudaMemcpyKind in_kind = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  const size_t nt = L.nt, nb = L.n_blocks;
  // scratch (d_work is free between validation calls); inputs are copied in, outputs copied out, so the caller's arrays need no alignment
  ChainArgs a;
  uint32_t *gf, *init, *scan, *n_ids, *vals, *commit;
  uint64_t* inner;
  kgv_chain_header* hdr;
  uint8_t* mflags;
  kgv_merkle_work mk;
  kgv_replay_muhash_work mu;
  kgv_mu_prefix_work ptot;
  kgv_mu_finalize_work fin;
  int rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap, [&](kgv_carve& c) {
    gf = c.take<uint32_t>(n_groups + 1); hdr = c.take<kgv_chain_header>(n_groups); mflags = c.take<uint8_t>(nb); init = c.take<uint32_t>(192);
    a.fee = c.take<uint64_t>(nb); a.code = c.take<uint8_t>(nb); a.flag = c.take<uint32_t>(nt); scan = c.take<uint32_t>(nt); n_ids = c.take<uint32_t>(64);
    a.comp = c.take<uint64_t>(nt * 4, 32); a.id_first = c.take<uint32_t>(n_groups + 1); inner = c.take<uint64_t>(n_groups * 4);
    mk.carve(c, nt); mu.carve(c, nt, n_groups); vals = c.take<uint32_t>(n_groups * 192); ptot.carve(c, n_groups); fin.carve(c, n_groups);
    commit = c.take<uint32_t>(n_groups * 8); a.out = c.take<kgv_chain_result>(n_groups);
  });
  if (rc) return rc;
  CK(cudaMemcpyAsync(gf, group_first_block, (n_groups + 1) * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(hdr, headers, n_groups * sizeof(kgv_chain_header), in_kind, st));
  CK(cudaMemcpyAsync(mflags, merged_flags, nb, in_kind, st));
  CK(cudaMemcpyAsync(init, init768, 768, in_kind, st));
  a.v = BatchView{(const kgv_tx*)L.txs, (const kgv_input*)L.inputs, (const kgv_output*)L.outputs, nullptr, (const uint8_t*)L.bytes};
  a.blk = L.blk; a.res = L.res; a.accept = L.acc; a.ids = L.ids;
  a.gf = gf; a.n_groups = (uint32_t)n_groups; a.nt = (uint32_t)nt;
  a.hdr = hdr; a.mflags = mflags;
  a.max_payload_len = body_rules->max_coinbase_payload_len; a.max_spk_len = rules->coinbase_payload_script_public_key_max_len;
  a.scan = scan; a.n_ids = n_ids; a.inner = inner; a.commit = commit;
  // fees, payloads and accepted-id flags per block; the accepted ids, compacted; their merkle roots per group
  k_chain_blocks<<<(unsigned)n_groups, 32 * CHAIN_BLOCK_WARPS, 0, st>>>(a);
  CK(cudaGetLastError());
  rc = kgv_scan_u32(ctx, a.flag, scan, nullptr, nullptr, nt, n_ids, st);
  if (rc) return rc;
  k_chain_compact<<<nblk(nt, 256), 256, 0, st>>>(a);
  CK(cudaGetLastError());
  k_chain_id_first<<<nblk(n_groups + 1, 128), 128, 0, st>>>(a);
  CK(cudaGetLastError());
  ctx->launches += 3;
  rc = kgv_merkle_levels(ctx, a.comp, nt, a.id_first, (uint32_t)n_groups, max_ids, mk, inner, st);
  if (rc) return rc;
  // the running multiset after every group, finalized in one batch
  rc = kgv_replay_muhash_run(ctx, a.gf, n_groups, mu, vals, st);
  if (rc) return rc;
  rc = kgv_mu_prefix_combine_run(ctx, init, vals, n_groups, ptot, st);
  if (rc) return rc;
  rc = kgv_mu_finalize_run(ctx, vals, vals + 96, n_groups, 192, fin, nullptr, commit, st);
  if (rc) return rc;
  k_chain_verdict<<<nblk(n_groups * 32, 128), 128, 0, st>>>(a);
  CK(cudaGetLastError());
  ctx->launches++;
  if ((rc = io.copy_out(results, a.out, n_groups * sizeof(kgv_chain_result)))) return rc;
  if (block_fees && (rc = io.copy_out(block_fees, a.fee, nb * 8))) return rc;
  if (multisets768 && (rc = io.copy_out(multisets768, vals, n_groups * 768))) return rc;
  return io.finish();
}
