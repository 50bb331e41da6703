// kgv_scripts_dev.cu — check_scripts (tx_validation_in_utxo_context.rs:162-200) with the full script engine on the device
// (kgv_script_dev.cuh) for a list of transactions of a populated batch: the transactions the fast path declines
// (KGV_TX_NEEDS_HOST_VM) in the table-backed calls, and kgv_check_scripts.
//
// Every input of a listed transaction is a work item.  Rounds:
//   k_se_run      grid-stride over the pending work items, one ScriptSlot per thread (at most 64 MiB of slots in all): run the
//                 input from the start over its verdict log; an input that needs one more verdict writes its request
//   (scan)        requests per work item (0 / 1, Schnorr and ECDSA), exclusive prefix sums -> the items of the round in input order
//   k_se_emit     gather (pk, sig) of every request
//   k_se_msgs     signature hashes (the per-transaction sub-hashes are computed once per call, k_se_reused)
//   verify        the fast path's item verification step (SigCache included), kgv_verify_items
//   k_se_append   verdict k of a request -> slot k of its input's log
// until no input asks for more; one 8-byte read-back per round.  An input makes at most 255 checks (its sig_op_count), so a call
// takes at most 256 rounds.  k_se_finalize then gives each transaction the host loop's result: the first failing input in index order.
#include "kgv_internal.h"
#include "kgv_script_dev.cuh"

#include <algorithm>
#include <cstdio>
#include <vector>

using namespace kgv;


static const size_t kSlotBytes = 64ull << 20;  // ScriptSlots of one call, whatever the batch size

struct ScriptWork { uint32_t in_abs, tx, idx, list; };

// per listed tx: its input count (and a range check of the index); *total = the 64-bit sum (the scan's offsets are 32-bit: a list that repeats
// large transactions could pass 2^32 work items, which the host rejects)
__global__ void k_se_count(const kgv_tx* __restrict__ txs, size_t n_txs, const uint32_t* __restrict__ list, uint32_t n, uint32_t* __restrict__ cnt,
                           uint32_t* __restrict__ fail_at, unsigned int* __restrict__ bad, unsigned long long* __restrict__ total) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t ti = list[j];
  fail_at[j] = 0xFFFFFFFFu;
  if (ti >= n_txs) { cnt[j] = 0; atomicOr(bad, 1u); return; }
  cnt[j] = txs[ti].n_inputs;
  if (txs[ti].n_inputs) atomicAdd(total, (unsigned long long)txs[ti].n_inputs);
}
__global__ void k_se_expand(const kgv_tx* __restrict__ txs, const uint32_t* __restrict__ list, uint32_t n, const uint32_t* __restrict__ off,
                            ScriptWork* __restrict__ work, uint8_t* __restrict__ status, uint8_t* __restrict__ nlog) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const kgv_tx t = txs[list[j]];
  for (uint32_t k = 0; k < t.n_inputs; k++) {
    const uint32_t w = off[j] + k;
    work[w] = ScriptWork{t.first_input + k, list[j], k, j};
    status[w] = SE_PENDING;
    nlog[w] = 0;
  }
}
__global__ void __launch_bounds__(128) k_se_reused(BatchView b, const uint32_t* __restrict__ list, uint32_t n, SigHashReused* __restrict__ reused) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  SigHashReused r;
  sighash_reused(r, b, list[j]);
  reused[j] = r;
}
__global__ void __launch_bounds__(64) k_se_run(BatchView b, const ScriptWork* __restrict__ work, uint32_t n, uint8_t* __restrict__ status,
                                               const uint8_t* __restrict__ nlog, const uint8_t* __restrict__ logs, ScriptReq* __restrict__ req,
                                               ScriptSlot* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ fail_at,
                                               uint32_t* __restrict__ cnt_s, uint32_t* __restrict__ cnt_e, unsigned int* __restrict__ overflow) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_slots) return;
  ScriptSlot* slot = slots + g;
  for (uint32_t w = g; w < n; w += n_slots) {
    uint32_t cs = 0, ce = 0;
    if (status[w] == SE_PENDING) {
      const ScriptWork wk = work[w];
      if (fail_at[wk.list] < wk.idx) {
        status[w] = SE_SKIPPED;  // an earlier input of the transaction already failed: this one cannot change the result
      } else {
        const uint8_t r = script_run_input(b, wk.tx, wk.in_abs, slot, logs + (size_t)SE_LOG_BYTES * w, nlog[w], req + w);
        if (r == SE_NEEDS) {
          if (req[w].ecdsa) ce = 1;
          else cs = 1;
        } else {
          status[w] = r;
          if (r == SE_OVERFLOW) atomicOr(overflow, 1u);
          else if (r != KGV_SCRIPT_OK) atomicMin(&fail_at[wk.list], wk.idx);
        }
      }
    }
    cnt_s[w] = cs;
    cnt_e[w] = ce;
  }
}
__global__ void k_se_emit(const uint32_t* __restrict__ cnt_s, const uint32_t* __restrict__ cnt_e, const uint32_t* __restrict__ off_s,
                          const uint32_t* __restrict__ off_e, uint32_t n, const ScriptReq* __restrict__ req, uint8_t* __restrict__ pk_s,
                          uint8_t* __restrict__ sig_s, uint32_t* __restrict__ ref_s, uint8_t* __restrict__ pk_e, uint8_t* __restrict__ sig_e,
                          uint32_t* __restrict__ ref_e) {
  uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n || !(cnt_s[w] | cnt_e[w])) return;
  const ScriptReq& r = req[w];
  if (cnt_e[w]) {
    const uint32_t it = off_e[w];
    for (int x = 0; x < 33; x++) pk_e[33 * (size_t)it + x] = r.key[x];
    for (int x = 0; x < 64; x++) sig_e[64 * (size_t)it + x] = r.sig[x];
    ref_e[it] = w;
  } else {
    const uint32_t it = off_s[w];
    for (int x = 0; x < 32; x++) pk_s[32 * (size_t)it + x] = r.key[x];
    for (int x = 0; x < 64; x++) sig_s[64 * (size_t)it + x] = r.sig[x];
    ref_s[it] = w;
  }
}
__global__ void __launch_bounds__(128) k_se_msgs(BatchView b, const ScriptWork* __restrict__ work, const ScriptReq* __restrict__ req,
                                                 const SigHashReused* __restrict__ reused, const uint32_t* __restrict__ refs, uint32_t n_items, bool ecdsa,
                                                 uint32_t* __restrict__ msgs) {
  uint32_t it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= n_items) return;
  const uint32_t w = refs[it];
  const ScriptWork wk = work[w];
  const SigHashReused r = reused[wk.list];
  uint32_t h[8];
  sighash_final(h, b, wk.tx, wk.in_abs, req[w].hash_type, ecdsa, r);  // the engine only asks for allowed hash types
#pragma unroll
  for (int k = 0; k < 8; k++) msgs[8 * (size_t)it + k] = bswap32(h[k]);
}
__global__ void k_se_append(const uint32_t* __restrict__ refs, const uint8_t* __restrict__ st, uint32_t n_items, uint8_t* __restrict__ nlog,
                            uint8_t* __restrict__ logs) {
  uint32_t it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= n_items) return;
  const uint32_t w = refs[it], k = nlog[w];
  uint8_t* l = logs + (size_t)SE_LOG_BYTES * w + (k >> 2);
  *l = (uint8_t)((*l & ~(3u << (2 * (k & 3)))) | ((uint32_t)(st[it] & 3) << (2 * (k & 3))));
  nlog[w] = (uint8_t)(k + 1);
}
// per listed tx: the first failing input in index order (check_scripts_sequential, :170-178; map_script_err :198-200).  patch: write the
// verdict fields of res[list[j]] (the caller's per-tx results), else res[j] as a whole record
__global__ void k_se_finalize(BatchView b, const uint32_t* __restrict__ list, uint32_t n, const uint32_t* __restrict__ off, const uint8_t* __restrict__ status,
                              kgv_tx_result* __restrict__ res, bool patch) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t ti = list[j];
  const kgv_tx& t = b.txs[ti];
  kgv_tx_result r = patch ? res[ti] : kgv_tx_result{};
  r.status = KGV_TX_OK; r.script_err = KGV_SCRIPT_OK; r.fail_input = 0;
  for (uint32_t k = 0; k < t.n_inputs; k++) {
    const uint8_t e = status[off[j] + k];
    if (e == KGV_SCRIPT_OK) continue;
    r.fail_input = k;
    r.script_err = e;
    r.status = b.inputs[t.first_input + k].sigscript_len == 0 ? KGV_TX_SIGNATURE_EMPTY : KGV_TX_SIGNATURE_INVALID;
    break;
  }
  res[patch ? ti : j] = r;
}

// the transactions whose status is KGV_TX_NEEDS_HOST_VM, in index order
__global__ void k_se_select_flag(const kgv_tx_result* __restrict__ res, uint32_t n, uint32_t* __restrict__ flag) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = res[i].status == KGV_TX_NEEDS_HOST_VM ? 1u : 0u;
}
__global__ void k_se_select_scatter(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ off, uint32_t n, uint32_t* __restrict__ list) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) list[off[i]] = i;
}

// Decides the listed transactions with the device engine.  dlist: n_list device indices into v.txs; or null: the n_list transactions
// whose dres status is KGV_TX_NEEDS_HOST_VM.  v.entries: the populated entries.  patch: the results go to dres[tx] (status, script_err,
// fail_input; the fee stays), else to dres[j] for list entry j.  Scratch: ctx->d_out (per listed tx), ctx->d_scratch (work items, logs,
// requests, slots) and ctx->d_in (the items of a round).
int kgv_script_engine_run(kgv_ctx* ctx, const BatchView& v, size_t n_txs, const uint32_t* dlist, size_t n_list, kgv_tx_result* dres, bool patch,
                          uint32_t* rounds_out) {
  if (rounds_out) *rounds_out = 0;
  ctx->last_script_rounds = 0;
  if (n_list == 0) return KGV_OK;
  if (n_list > 0xFFFFFFFFull) { ctx->err = "kgv_check_scripts: too many transactions"; return KGV_ERR_ARG; }
  cudaStream_t st = ctx->stream;
  const uint32_t nl = (uint32_t)n_list;
  // phase 1, in ctx->d_out: per listed tx its input count, work offset, first failing input and sub-hashes; flags; without dlist the
  // selected list and its flags and offsets
  const bool select = !dlist;
  uint32_t *cnt, *off, *fail_at, *list, *sel, *selo;
  SigHashReused* reu;
  unsigned int* flags;  // [0] bad index, [1] overflow, [2..3] round totals, [4] work total, [6..7] its 64-bit sum, [8] the selection's total
  int rc = kgv_reserve_carved(ctx, &ctx->d_out, &ctx->d_out_cap, [&](kgv_carve& c) {
    cnt = c.take<uint32_t>(n_list); off = c.take<uint32_t>(n_list); fail_at = c.take<uint32_t>(n_list); reu = c.take<SigHashReused>(n_list);
    flags = c.take<unsigned int>(16);
    list = select ? c.take<uint32_t>(n_list) : nullptr; sel = select ? c.take<uint32_t>(n_txs) : nullptr; selo = select ? c.take<uint32_t>(n_txs) : nullptr;
  });
  if (rc) return rc;
  if (select) {
    k_se_select_flag<<<nblk(n_txs, 256), 256, 0, st>>>(dres, (uint32_t)n_txs, sel);
    CK(cudaGetLastError());
    rc = kgv_scan_u32(ctx, sel, selo, nullptr, nullptr, n_txs, (uint32_t*)(flags + 8), st);
    if (rc) return rc;
    k_se_select_scatter<<<nblk(n_txs, 256), 256, 0, st>>>(sel, selo, (uint32_t)n_txs, list);
    CK(cudaGetLastError());
    ctx->launches += 3;
    dlist = list;
  }
  CK(cudaMemsetAsync(flags, 0, 64, st));
  k_se_count<<<nblk(nl, 128), 128, 0, st>>>(v.txs, n_txs, dlist, nl, cnt, fail_at, flags, (unsigned long long*)(flags + 6));
  CK(cudaGetLastError());
  rc = kgv_scan_u32(ctx, cnt, off, nullptr, nullptr, n_list, (uint32_t*)(flags + 4), st);
  if (rc) return rc;
  ctx->launches += 1;
  unsigned int hf[8];
  CK(cudaMemcpyAsync(hf, flags, sizeof hf, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (hf[0]) { ctx->err = "kgv_check_scripts: a transaction index is out of range"; return KGV_ERR_ARG; }
  const uint64_t nw64 = (uint64_t)hf[6] | ((uint64_t)hf[7] << 32);
  if (nw64 > 0xFFFFFFFFull) { ctx->err = "kgv_check_scripts: the listed transactions have 2^32 or more inputs in all"; return KGV_ERR_ARG; }
  const size_t nw = (size_t)nw64;
  if (nw == 0) {
    k_se_finalize<<<nblk(nl, 128), 128, 0, st>>>(v, dlist, nl, off, nullptr, dres, patch);
    CK(cudaGetLastError());
    ctx->launches++;
    return KGV_OK;
  }
  // phase 2, in ctx->d_scratch: per-work-item state and the slots
  const uint32_t n_slots = (uint32_t)std::min(nw, kSlotBytes / sizeof(ScriptSlot));
  ScriptWork* work;
  uint8_t *status, *nlog, *logs;
  ScriptReq* req;
  uint32_t *cs, *ce, *os, *oe;
  ScriptSlot* slots;
  rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap, [&](kgv_carve& c) {
    work = c.take<ScriptWork>(nw); status = c.take<uint8_t>(nw); nlog = c.take<uint8_t>(nw); logs = c.take<uint8_t>(nw * SE_LOG_BYTES); req = c.take<ScriptReq>(nw);
    cs = c.take<uint32_t>(nw); ce = c.take<uint32_t>(nw); os = c.take<uint32_t>(nw); oe = c.take<uint32_t>(nw); slots = c.take<ScriptSlot>(n_slots);
  });
  if (rc) return rc;
  CK(cudaMemsetAsync(logs, 0, nw * SE_LOG_BYTES, st));
  k_se_expand<<<nblk(nl, 128), 128, 0, st>>>(v.txs, dlist, nl, off, work, status, nlog);
  CK(cudaGetLastError());
  k_se_reused<<<nblk(nl, 128), 128, 0, st>>>(v, dlist, nl, reu);
  CK(cudaGetLastError());
  ctx->launches += 2;
  // the engine's checks go through the SigCache like any other (not combined with sharding, as in the fast path)
  kgv_sigcache* sc = ctx->shard_comm ? nullptr : ctx->sigcache;
  uint32_t round = 0;
  for (;; round++) {
    k_se_run<<<nblk(n_slots, 64), 64, 0, st>>>(v, work, (uint32_t)nw, status, nlog, logs, req, slots, n_slots, fail_at, cs, ce, flags + 1);
    CK(cudaGetLastError());
    rc = kgv_scan_u32(ctx, cs, os, ce, oe, nw, (uint32_t*)(flags + 2), st);
    if (rc) return rc;
    ctx->launches += 2;
    unsigned int h[3];
    CK(cudaMemcpyAsync(h, flags + 1, sizeof h, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (h[0]) { ctx->err = "script engine: a per-input scratch bound was exceeded (internal error)"; return KGV_ERR_LIMIT; }
    const size_t ns = h[1], ne = h[2];
    if (ns + ne == 0) break;
    if (round >= 256) { ctx->err = "script engine: an input asked for more than 255 signature checks (internal error)"; return KGV_ERR_LIMIT; }
    struct Kind { size_t n; uint8_t *pk, *sig, *msg, *st, *dig; uint32_t *ref, *idx, *nm; } kind[2] = {{ns}, {ne}};
    rc = kgv_reserve_carved(ctx, &ctx->d_in, &ctx->d_in_cap, [&](kgv_carve& c) {
      for (int e = 0; e < 2; e++) {
        Kind& k = kind[e];
        k.pk = c.take<uint8_t>(k.n * (e ? 33 : 32)); k.sig = c.take<uint8_t>(k.n * 64); k.msg = c.take<uint8_t>(k.n * 32); k.ref = c.take<uint32_t>(k.n);
        k.st = c.take<uint8_t>(k.n, 64);
        k.dig = c.take<uint8_t>(sc ? k.n * 32 : 0); k.idx = c.take<uint32_t>(sc ? k.n : 0); k.nm = c.take<uint32_t>(16);
      }
    });
    if (rc) return rc;
    k_se_emit<<<nblk(nw, 128), 128, 0, st>>>(cs, ce, os, oe, (uint32_t)nw, req, kind[0].pk, kind[0].sig, kind[0].ref, kind[1].pk, kind[1].sig, kind[1].ref);
    CK(cudaGetLastError());
    ctx->launches++;
    for (int e = 0; e < 2; e++) {
      const Kind& k = kind[e];
      if (!k.n) continue;
      k_se_msgs<<<nblk(k.n, 128), 128, 0, st>>>(v, work, req, reu, k.ref, (uint32_t)k.n, e == 1, (uint32_t*)k.msg);
      CK(cudaGetLastError());
      ctx->launches++;
      rc = kgv_verify_items(ctx, sc, k.pk, k.msg, k.sig, k.n, e == 1, k.st, k.dig, k.idx, k.nm, st);
      if (rc) return rc;
      k_se_append<<<nblk(k.n, 128), 128, 0, st>>>(k.ref, k.st, (uint32_t)k.n, nlog, logs);
      CK(cudaGetLastError());
      ctx->launches++;
    }
  }
  if (rounds_out) *rounds_out = round;
  ctx->last_script_rounds = round;
  k_se_finalize<<<nblk(nl, 128), 128, 0, st>>>(v, dlist, nl, off, status, dres, patch);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

// the populated entries of a caller's batch.  An entry marked absent (pad_[0] != 0) is given an empty script: its offset is not range-checked
// for a host batch, and a transaction with a missing outpoint has no script result in the reference anyway (MissingTxOutpoints comes first).
__global__ void k_se_entries(const kgv_utxo_entry* __restrict__ in, const uint8_t* __restrict__ bytes, size_t n, DevEntry* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const kgv_utxo_entry e = in[i];
  const bool found = e.pad_[0] == 0;
  DevEntry d;
  d.amount = e.amount; d.block_daa_score = e.block_daa_score; d.script = bytes + (found ? e.script_off : 0); d.script_len = found ? e.script_len : 0;
  d.spk_version = e.spk_version; d.is_coinbase = e.is_coinbase; d.found = found ? 1 : 0;
  out[i] = d;
}

extern "C" int kgv_debug_script_rounds(const kgv_ctx* ctx, uint32_t* rounds) {
  if (!ctx || !rounds) return KGV_ERR_ARG;
  *rounds = ctx->last_script_rounds;
  return KGV_OK;
}

extern "C" int kgv_check_scripts(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* tx_indices, size_t n, kgv_tx_result* results) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || !batch->entries || (n && (!tx_indices || !results))) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (n == 0) return KGV_OK;
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  // the indices are range-checked here whatever their side: device indices are read through a host copy
  std::vector<uint32_t> idx_host;
  const uint32_t* hidx = tx_indices;
  if (io.is_device(tx_indices)) {
    idx_host.resize(n);
    CK(cudaMemcpyAsync(idx_host.data(), tx_indices, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    hidx = idx_host.data();
  }
  for (size_t i = 0; i < n; i++)
    if (hidx[i] >= batch->n_txs) { ctx->err = "kgv_check_scripts: a transaction index is out of range"; return KGV_ERR_ARG; }
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, true);
  if (rc) return rc;
  const size_t ni = d.n_inputs;
  DevEntry* dent;
  kgv_tx_result* dres;
  rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap, [&](kgv_carve& c) { dent = c.take<DevEntry>(ni); dres = c.take<kgv_tx_result>(n); });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const uint32_t* dlist;
  io.in(tx_indices, n * 4, &dlist);
  if ((rc = io.stage())) return rc;
  if (ni) {
    k_se_entries<<<nblk(ni, 128), 128, 0, st>>>(d.entries, d.bytes, ni, dent);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  BatchView v{d.txs, d.inputs, d.outputs, dent, d.bytes};
  rc = kgv_script_engine_run(ctx, v, d.n_txs, dlist, n, dres, false, nullptr);
  if (rc) return rc;
  if ((rc = io.copy_out(results, dres, n * sizeof(kgv_tx_result)))) return rc;
  return io.finish();
}
