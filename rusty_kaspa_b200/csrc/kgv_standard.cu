// kgv_standard.cu — the mempool's standardness policy for a batch (rule bodies in kgv_standard.cuh) and its three public calls,
// kgv_check_txs_standard_in_isolation, kgv_check_txs_standard_in_context and kgv_outputs_dust.  kgv_validate_mempool_txs_with_policy
// (kgv_validate.cu) runs the two transaction kernels around its pipeline.
//
//   k_tx_standard_isolation  one warp per tx : version, masses, then the lanes stride over the inputs (signature-script sizes) and the
//                                              outputs (spk version, class, dust), 32 at a time; the first offender is the lowest set bit
//                                              of a ballot.  Each lane walks its own output script (for is_unspendable) serially.
//   k_tx_standard_context    one warp per tx : storage mass, then the lanes stride over the inputs: the entry's class and, for P2SH, the
//                                              signature-script and redeem-script walks.  The fee check sits between input 0 and input 1,
//                                              where the reference's loop puts it.
//   k_outputs_dust           one thread per output
#include "kgv_internal.h"
#include "kgv_isolation.cuh"
#include "kgv_standard.cuh"

#include <cstdio>
#include <cstring>

using namespace kgv;

static_assert(sizeof(kgv_mempool_policy) == 16, "kgv_mempool_policy is 16 bytes");


constexpr int STD_WARPS = 4;  // transactions per block of the two transaction kernels

// gate: only a failure is written to res (kgv_validate_mempool_txs_with_policy: it overrides the isolation verdict there); detail is
// written for every tx
__global__ void __launch_bounds__(32 * STD_WARPS)
k_tx_standard_isolation(BatchView b, uint32_t n_txs, kgv_mempool_policy p, const kgv_tx_masses* __restrict__ masses, bool gate,
                        kgv_tx_result* __restrict__ res, uint64_t* __restrict__ detail) {
  const uint32_t ti = blockIdx.x * STD_WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (ti >= n_txs) return;  // uniform per warp
  const kgv_tx t = b.txs[ti];
  const kgv_tx_masses m = masses[ti];
  kgv_tx_result out = iso_result(KGV_TX_OK, 0);
  uint64_t det = 0;
  if (t.version < p.minimum_standard_transaction_version || t.version > p.maximum_standard_transaction_version) {
    out = iso_result(KGV_TX_REJECT_VERSION, 0); det = t.version;
  } else if (m.compute_mass > STD_MAX_TRANSACTION_MASS) {
    out = iso_result(KGV_TX_REJECT_COMPUTE_MASS, 0); det = m.compute_mass;
  } else if (m.transient_mass > STD_MAX_TRANSACTION_MASS) {
    out = iso_result(KGV_TX_REJECT_TRANSIENT_MASS, 0); det = m.transient_mass;
  } else {
    const kgv_input* in = b.inputs + t.first_input;
    const uint32_t i = warp_first(t.n_inputs, lane, [&](uint32_t x) { return in[x].sigscript_len > STD_MAX_SIGNATURE_SCRIPT_SIZE; });
    if (i < t.n_inputs) {
      out = iso_result(KGV_TX_REJECT_SIGNATURE_SCRIPT_SIZE, i); det = in[i].sigscript_len;
    } else {
      for (uint32_t base = 0; base < t.n_outputs; base += 32) {
        const uint32_t o = base + lane;
        uint32_t code = 0;
        uint64_t value = 0;
        if (o < t.n_outputs) {
          const kgv_output op = b.outputs[t.first_output + o];
          const uint8_t* s = b.bytes + op.script_off;
          value = op.value;
          if (op.spk_version > 0) code = KGV_TX_REJECT_SCRIPT_PUBLIC_KEY_VERSION;
          else if (script_class(op.spk_version, s, op.script_len) == SCLASS_NONSTANDARD) code = KGV_TX_REJECT_OUTPUT_SCRIPT_CLASS;
          else if (output_is_dust(op.value, s, op.script_len, p.minimum_relay_transaction_fee)) code = KGV_TX_REJECT_DUST;
        }
        const unsigned bad = __ballot_sync(ISO_FULL, code != 0);
        if (bad) {
          const int j = __ffs(bad) - 1;
          const uint32_t cj = __shfl_sync(ISO_FULL, code, j);
          const uint64_t vj = __shfl_sync(ISO_FULL, value, j);
          out = iso_result((uint8_t)cj, base + j);
          det = cj == KGV_TX_REJECT_DUST ? vj : 0;
          break;
        }
      }
    }
  }
  if (lane == 0) {
    if (!gate || out.status != KGV_TX_OK) res[ti] = out;
    if (detail) detail[ti] = det;
  }
}

// the spent entries, as the caller's batch holds them or as a validation call populated them
struct EntriesOfBatch {
  const kgv_utxo_entry* e;
  const uint8_t* bytes;
  __device__ __forceinline__ uint8_t cls(uint32_t i, const uint8_t*& s, uint32_t& n) const {
    const kgv_utxo_entry x = e[i];
    s = bytes + x.script_off; n = x.script_len;
    return script_class(x.spk_version, s, n);
  }
};
struct EntriesOfView {
  const DevEntry* e;
  __device__ __forceinline__ uint8_t cls(uint32_t i, const uint8_t*& s, uint32_t& n) const {
    s = e[i].script; n = e[i].script_len;
    return script_class(e[i].spk_version, s, n);
  }
};

// fee == null (kgv_validate_mempool_txs_with_policy): only the txs whose res status is KGV_TX_OK are checked, their fee is res[ti].fee and
// only a failure is written to res.  *overflow is set when a reached fee check's mass * fee overflows u64.
template <class E>
__global__ void __launch_bounds__(32 * STD_WARPS)
k_tx_standard_context(BatchView b, E ent, uint32_t n_txs, kgv_mempool_policy p, const kgv_tx_masses* __restrict__ masses,
                      const uint64_t* __restrict__ storage_mass, const uint64_t* __restrict__ fee, kgv_tx_result* __restrict__ res,
                      uint64_t* __restrict__ detail, unsigned long long* __restrict__ overflow) {
  const uint32_t ti = blockIdx.x * STD_WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (ti >= n_txs) return;  // uniform per warp
  uint64_t f;
  if (fee) {
    f = fee[ti];
  } else {
    const kgv_tx_result r = res[ti];
    if (r.status != KGV_TX_OK) return;
    f = r.fee;
  }
  const kgv_tx t = b.txs[ti];
  kgv_tx_result out = iso_result(KGV_TX_OK, 0);
  out.fee = f;
  uint64_t det = 0;
  const uint64_t sm = storage_mass[ti];
  if (sm > STD_MAX_TRANSACTION_MASS) {
    out.status = KGV_TX_REJECT_STORAGE_MASS; det = sm;
  } else {
    for (uint32_t base = 0; base < t.n_inputs; base += 32) {
      const uint32_t i = base + lane;
      uint32_t code = 0;
      uint64_t ops = 0;
      if (i < t.n_inputs) {
        const uint32_t a = t.first_input + i;
        const uint8_t* s;
        uint32_t n;
        const uint8_t c = ent.cls(a, s, n);
        if (c == SCLASS_NONSTANDARD) {
          code = KGV_TX_REJECT_INPUT_SCRIPT_CLASS;
        } else if (c == SCLASS_SCRIPT_HASH) {
          const kgv_input in = b.inputs[a];
          ops = p2sh_sig_op_bound(b.bytes + in.sigscript_off, in.sigscript_len);
          if (ops > STD_MAX_P2SH_SIG_OPS) code = KGV_TX_REJECT_SIGNATURE_COUNT;
        }
      }
      const unsigned bad = __ballot_sync(ISO_FULL, code != 0);
      if (base == 0) {
        if (bad & 1u) {
          out.status = (uint8_t)__shfl_sync(ISO_FULL, code, 0); det = __shfl_sync(ISO_FULL, ops, 0);
          break;
        }
        // input 0 passed: the reference's loop checks the fee next
        uint64_t min_fee;
        if (!min_relay_fee(masses[ti].compute_mass, p.minimum_relay_transaction_fee, min_fee)) {
          if (lane == 0) atomicOr(overflow, 1ull);
        } else if (f < min_fee) {
          out.status = KGV_TX_REJECT_INSUFFICIENT_FEE; det = min_fee;
          break;
        }
      }
      if (bad) {
        const int j = __ffs(bad) - 1;
        out.status = (uint8_t)__shfl_sync(ISO_FULL, code, j); out.fail_input = base + j; det = __shfl_sync(ISO_FULL, ops, j);
        break;
      }
    }
  }
  if (lane == 0) {
    if (fee || out.status != KGV_TX_OK) res[ti] = out;
    if (detail) detail[ti] = det;
  }
}

__global__ void k_outputs_dust(const kgv_output* __restrict__ outs, const uint8_t* __restrict__ bytes, size_t n, uint64_t fee, uint8_t* __restrict__ is_dust) {
  const size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n) return;
  const kgv_output x = outs[o];
  is_dust[o] = output_is_dust(x.value, bytes + x.script_off, x.script_len, fee) ? 1 : 0;
}

static unsigned tx_blocks(size_t nt) { return (unsigned)((nt + STD_WARPS - 1) / STD_WARPS); }

int kgv_standard_isolation_run(kgv_ctx* ctx, const kgv_dev_batch& d, const kgv_mempool_policy& p, const kgv_tx_masses* dmasses, bool gate,
                               kgv_tx_result* dres, uint64_t* ddetail, cudaStream_t st) {
  if (d.n_txs == 0) return KGV_OK;
  const BatchView v{d.txs, d.inputs, d.outputs, nullptr, d.bytes};
  k_tx_standard_isolation<<<tx_blocks(d.n_txs), 32 * STD_WARPS, 0, st>>>(v, (uint32_t)d.n_txs, p, dmasses, gate, dres, ddetail);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

int kgv_standard_context_run(kgv_ctx* ctx, const kgv_dev_batch& d, const DevEntry* dent, const kgv_mempool_policy& p, const kgv_tx_masses* dmasses,
                             const uint64_t* dsmass, const uint64_t* dfee, kgv_tx_result* dres, uint64_t* ddetail, unsigned long long* dflag,
                             cudaStream_t st) {
  if (d.n_txs == 0) return KGV_OK;
  const BatchView v{d.txs, d.inputs, d.outputs, nullptr, d.bytes};
  const unsigned g = tx_blocks(d.n_txs);
  if (dent)
    k_tx_standard_context<<<g, 32 * STD_WARPS, 0, st>>>(v, EntriesOfView{dent}, (uint32_t)d.n_txs, p, dmasses, dsmass, dfee, dres, ddetail, dflag);
  else
    k_tx_standard_context<<<g, 32 * STD_WARPS, 0, st>>>(v, EntriesOfBatch{d.entries, d.bytes}, (uint32_t)d.n_txs, p, dmasses, dsmass, dfee, dres, ddetail, dflag);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

extern "C" int kgv_check_txs_standard_in_isolation(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_mempool_policy* policy, const kgv_tx_masses* masses,
                                                    kgv_tx_result* results, uint64_t* detail) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || !policy || (batch->n_txs && (!results || !masses))) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_check_txs_standard_in_isolation", "policy", policy)) return rc;
  if (batch->n_txs == 0) return KGV_OK;
  if (batch->n_txs > 0xFFFFFFFFull) { ctx->err = "kgv_check_txs_standard_in_isolation: more than 2^32 - 1 transactions"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_check_txs_standard_in_isolation", {results, batch->txs, masses, detail})) return rc;
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  const size_t nt = d.n_txs;
  const kgv_tx_masses* dm;
  kgv_tx_result* dres;
  uint64_t* ddet;
  io.in(masses, nt * sizeof(kgv_tx_masses), &dm);
  io.out(results, nt * sizeof(kgv_tx_result), &dres);
  io.out(detail, nt * 8, &ddet);
  if ((rc = io.stage())) return rc;
  if ((rc = kgv_standard_isolation_run(ctx, d, *policy, dm, false, dres, ddet, ctx->stream))) return rc;
  return io.finish();
}

extern "C" int kgv_check_txs_standard_in_context(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_mempool_policy* policy, const kgv_tx_masses* masses,
                                                  const uint64_t* storage_mass, const uint64_t* fee, kgv_tx_result* results, uint64_t* detail) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || !policy || (batch->n_txs && (!results || !masses || !storage_mass || !fee))) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_check_txs_standard_in_context", "policy", policy)) return rc;
  if (batch->n_txs == 0) return KGV_OK;
  if (batch->n_inputs && !batch->entries) { ctx->err = "kgv_check_txs_standard_in_context: batch->entries is required"; return KGV_ERR_ARG; }
  if (batch->n_txs > 0xFFFFFFFFull) { ctx->err = "kgv_check_txs_standard_in_context: more than 2^32 - 1 transactions"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_check_txs_standard_in_context", {results, batch->txs, masses, storage_mass, fee, detail})) return rc;
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, batch->n_inputs != 0);
  if (rc) return rc;
  const size_t nt = d.n_txs;
  const kgv_tx_masses* dm;
  const uint64_t *dsm, *dfee;
  kgv_tx_result* dres;
  uint64_t* ddet;
  unsigned long long flag = 0, *dflag;  // a host scalar: finish() always synchronises to read it
  io.in(masses, nt * sizeof(kgv_tx_masses), &dm);
  io.in(storage_mass, nt * 8, &dsm);
  io.in(fee, nt * 8, &dfee);
  io.out(results, nt * sizeof(kgv_tx_result), &dres);
  io.out(detail, nt * 8, &ddet);
  io.out(&flag, 8, &dflag);
  if ((rc = io.stage())) return rc;
  CK(cudaMemsetAsync(dflag, 0, 8, ctx->stream));
  if ((rc = kgv_standard_context_run(ctx, d, nullptr, *policy, dm, dsm, dfee, dres, ddet, dflag, ctx->stream))) return rc;
  if ((rc = io.finish())) return rc;
  if (flag) { ctx->err = "kgv_check_txs_standard_in_context: compute mass * minimum_relay_transaction_fee overflows u64"; return KGV_ERR_ARG; }
  return KGV_OK;
}

extern "C" int kgv_outputs_dust(kgv_ctx* ctx, const kgv_tx_batch* batch, uint64_t minimum_relay_transaction_fee, uint8_t* is_dust) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || (batch->n_outputs && !is_dust)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (batch->n_outputs == 0) return KGV_OK;
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_outputs_dust", {is_dust, batch->outputs})) return rc;
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  const size_t no = d.n_outputs;
  uint8_t* out;
  io.out(is_dust, no, &out);
  if ((rc = io.stage())) return rc;
  k_outputs_dust<<<(unsigned)((no + 255) / 256), 256, 0, ctx->stream>>>(d.outputs, d.bytes, no, minimum_relay_transaction_fee, out);
  CK(cudaGetLastError());
  ctx->launches++;
  return io.finish();
}
