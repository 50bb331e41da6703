// kgv_replay_impl.cuh — kgv_replay_window: the caller side of the hot path as ONE library call (included by kgv_validate.cu,
// whose kernels it reuses).
//
// Reference: VirtualStateProcessor::calculate_utxo_state / verify_expected_utxo_state
// (consensus/src/pipeline/virtual_processor/utxo_validation.rs:110-173,182-228): the blocks of a mergeset are processed
// SEQUENTIALLY against `selected_parent_utxo_view.compose(&ctx.mergeset_diff)`, the transactions of one block in parallel
// (:262-309), and every accepted transaction is folded into the diff (UtxoDiff::add_transaction, utxo_diff.rs:233-247)
// before the next block is looked at.  simpa prints the rate of exactly this loop (simpa/src/main.rs:454-460).
//
// A 10-BPS block carries a few hundred signatures - three orders of magnitude too few for an H100 - but signatures are
// context free given the spent output (SURVEY.md §0-6: the sighash reads only the entry's script_public_key and amount,
// sighash.rs:252-255, and both are fixed by the outpoint).  So the window is processed in two device-resident passes:
//
//   pre-check   every script of the window in ONE batch (plan/sighash/verify/resolve of kgv_validate.cu, millions of
//               signature checks per launch).  Spent outputs come from the UTXO table or, when the output is created inside
//               the window, from the creating transaction (found through a window hash map  tx id -> tx index  built on the
//               device).  Which of the two exists at the spending block's position is irrelevant for the script verdict.
//   in-order    whatever depends only on the outpoint is resolved for the whole window in parallel; one persistent
//               single-CTA kernel then walks the blocks deciding only whether each input's outpoint still exists at its
//               block's position (accept = context ok && scripts ok), and parallel passes erase the spent entries and insert
//               the created ones that survive the window (see "The in-order pass" below).
//
// Result per transaction: the context verdict when the context rules fail, else the script verdict - the order
// validate_populated_transaction_and_get_fee reports them in (tx_validation_in_utxo_context.rs:34-61).

// ---------------------------------------------------------------------------------------------
// window map: tx id -> tx index (open addressing over indices; the ids array holds the keys)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t wm_hash(const uint64_t* id) { return id[0] ^ (id[1] * 0x9E3779B97F4A7C15ull) ^ (id[2] >> 17) ^ (id[3] << 13); }
__device__ __forceinline__ bool id_eq(const uint64_t* a, const uint64_t* b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2] && a[3] == b[3]; }

__global__ void k_wm_insert(const uint64_t* __restrict__ ids, uint32_t n_txs, uint32_t* __restrict__ wm, uint64_t wm_mask, uint8_t* __restrict__ has_sibling) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_txs) return;
  const uint64_t* id = ids + 4 * (size_t)t;
  uint64_t i = wm_hash(id) & wm_mask;
  for (uint64_t p = 0; p <= wm_mask; p++, i = (i + 1) & wm_mask) {
    uint32_t cur = atomicCAS(&wm[i], 0u, t + 1);
    if (cur == 0u) return;
    // the same transaction may sit in several parallel blocks of a DAG: one representative is enough (identical outputs)
    if (id_eq(ids + 4 * (size_t)(cur - 1), id)) { has_sibling[cur - 1] = 1; return; }
  }
}
__device__ __forceinline__ int wm_find(const uint64_t* __restrict__ ids, const uint32_t* __restrict__ wm, uint64_t wm_mask, const uint64_t* id) {
  uint64_t i = wm_hash(id) & wm_mask;
  for (uint64_t p = 0; p <= wm_mask; p++, i = (i + 1) & wm_mask) {
    uint32_t cur = wm[i];
    if (cur == 0u) return -1;
    if (id_eq(ids + 4 * (size_t)(cur - 1), id)) return (int)(cur - 1);
  }
  return -1;
}

// per-transaction block index and the pre-check's starting status
#define KGV_PRE_SKIPPED 0xFEu  // not script-checked in the pre-pass (coinbase position, SkipScriptChecks block)
__global__ void k_replay_tx_block(const kgv_replay_block* __restrict__ blocks, uint32_t n_blocks, uint32_t* __restrict__ tx_block) {
  uint32_t bi = blockIdx.x;
  if (bi >= n_blocks) return;
  kgv_replay_block bl = blocks[bi];
  for (uint32_t j = threadIdx.x; j < bl.n_txs; j += blockDim.x) tx_block[bl.first_tx + j] = bi;
}
__global__ void k_replay_pre_status(BatchView b, uint32_t n_txs, const kgv_replay_block* __restrict__ blocks, const uint32_t* __restrict__ tx_block,
                                    kgv_tx_result* __restrict__ pre) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  kgv_replay_block bl = blocks[tx_block[ti]];
  const kgv_tx& t = b.txs[ti];
  kgv_tx_result r;
  r.fee = 0; r.fail_input = 0; r.status = KGV_TX_OK; r.script_err = 0; r.pad_[0] = r.pad_[1] = 0;
  if (ti == bl.first_tx || tx_is_coinbase(t) || (bl.flags & KGV_REPLAY_SKIP_SCRIPTS)) r.status = KGV_PRE_SKIPPED;
  else {
    const DevEntry* ent = b.entries + t.first_input;
    for (uint32_t i = 0; i < t.n_inputs; i++)
      if (!ent[i].found) { r.status = KGV_TX_MISSING_OUTPOINTS; break; }  // cannot exist at its block's position either
  }
  pre[ti] = r;
}
// per-block ranges, computed in parallel before the walk so that it never chases tx records to find them
struct __align__(16) ReplayRange {  // 48 bytes: a whole number of 16-byte units (the walk fetches these with bulk copies)
  uint32_t t0, t1, i0, i1, o0, o1, flags, pad_;
  uint64_t pov;
  uint64_t pad2_;
};
static_assert(sizeof(ReplayRange) == 48, "ReplayRange layout");
__global__ void k_replay_ranges(const kgv_replay_block* __restrict__ blocks, uint32_t n_blocks, const kgv_tx* __restrict__ txs, ReplayRange* __restrict__ out) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_blocks) return;
  kgv_replay_block bl = blocks[b];
  ReplayRange r;
  r.t0 = bl.first_tx; r.t1 = bl.first_tx + bl.n_txs; r.flags = bl.flags; r.pad_ = 0; r.pov = bl.pov_daa_score; r.pad2_ = 0;
  r.i0 = r.i1 = r.o0 = r.o1 = 0;
  if (bl.n_txs) {
    const kgv_tx& tf = txs[r.t0];
    const kgv_tx& tl = txs[r.t1 - 1];
    r.i0 = tf.first_input; r.i1 = tl.first_input + tl.n_inputs; r.o0 = tf.first_output; r.o1 = tl.first_output + tl.n_outputs;
  }
  out[b] = r;
}

// ---------------------------------------------------------------------------------------------
// The in-order pass, reduced to what is inherently sequential.
//
// Within a window, whether an input's outpoint EXISTS at its block's position depends on the acceptance of earlier transactions - that is the
// only sequential dependence of calculate_utxo_state.  Everything else is a function of the outpoint alone (a txid commits to its outputs, so the
// spent entry's amount / script / coinbase flag are the same wherever it comes from) and is computed for the whole window in parallel:
//   k_replay_sources   per input : where its outpoint can come from - a table slot present at window start, or output k of window transaction j
//                                  (through the window map; several blocks of a DAG may carry the same transaction: one representative per id) -
//                                  and the index of the shared "spent" flag of that outpoint (inputs probing one slot agree on it through a pointer map)
//   k_replay_static    per tx    : the context rules that read only amounts / lengths (input sum, spend, fee, storage mass) -> a static verdict,
//                                  plus "needs the entry's DAA score" (spends a coinbase / carries a relative lock)
// The walk itself (one CTA, state in shared-memory bitmaps: spent outpoints, accepted transactions) then does per block: every transaction
// checks its inputs' flags (a few dozen instructions, no table access, no division), accepted ones set theirs after a barrier.  ~1 k cycles
// per block (measured, DESIGN.md §4).  Afterwards, again in parallel over the window:
//   k_replay_finish_inputs   every spent entry is captured (MuHash consumers) and erased from the table
//   k_replay_finish_outputs  every output of an accepted transaction that is still unspent at the end of the window is inserted
//   k_replay_finish_results  verdicts are assembled (dynamic verdict, else static, else the script verdict of the pre-check)
// Outputs created AND spent inside the window never touch the table.
// ---------------------------------------------------------------------------------------------
#define RS_NONE 0u
#define RS_TABLE 1u
#define RS_WINDOW 2u
#define RS_FLAG_MASK 0x3FFFFFFFu
struct ReplaySrc {      // per input (8 bytes: the walk stages these)
  uint32_t flag;        // bits 30-31: RS_*; bits 0-29: index of the outpoint's spent flag - TABLE: first input of the window probing the same slot; WINDOW: global index of the creating output
  uint32_t src_tx;      // WINDOW: representative index of the creating transaction
};
struct __align__(16) ReplayTxInfo {   // per transaction (16 bytes)
  uint32_t first_input;
  uint32_t n_inputs;
  uint32_t rep;           // representative instance of this transaction id inside the window (itself unless a DAG sibling carries the same transaction)
  uint8_t static_status;  // KGV_TX_OK or the first failing rule that does not depend on the walk
  uint8_t bits;           // 1: coinbase (position 0 / subnetwork)  2: DAA-score rules depend on the walk  4: scripts ok (pre-check)  8: sibling blocks carry this transaction too
  uint16_t pad_;
};
__device__ __forceinline__ uint32_t rs_kind(const ReplaySrc& r) { return r.flag >> 30; }

// pointer map: table slot -> smallest input index of the window that found it (inputs spending one outpoint share one flag)
__device__ __forceinline__ uint64_t slotmap_hash(unsigned long long k) {
  uint64_t h = (k >> 7) * 0x9E3779B97F4A7C15ull;
  return h ^ (h >> 31);
}
__global__ void k_slotmap_insert(const ReplaySrc* __restrict__ src, UtxoSlot* const* __restrict__ slot, size_t n_inputs, unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals,
                                 uint64_t mask) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs || rs_kind(src[i]) != RS_TABLE) return;
  const unsigned long long k = (unsigned long long)(uintptr_t)slot[i];
  for (uint64_t p = 0, j = slotmap_hash(k) & mask; p <= mask; p++, j = (j + 1) & mask) {
    unsigned long long cur = atomicCAS(&keys[j], 0ull, k);
    if (cur == 0ull || cur == k) { atomicMin(&vals[j], (uint32_t)i); return; }
  }
}
__global__ void k_slotmap_lookup(UtxoSlot* const* __restrict__ slot, size_t n_inputs, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals, uint64_t mask,
                                 ReplaySrc* __restrict__ src) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs || rs_kind(src[i]) != RS_TABLE) return;
  const unsigned long long k = (unsigned long long)(uintptr_t)slot[i];
  for (uint64_t p = 0, j = slotmap_hash(k) & mask; p <= mask; p++, j = (j + 1) & mask)
    if (keys[j] == k) { src[i].flag = (RS_TABLE << 30) | vals[j]; return; }
}
// sources of every input + the entry the pre-check (and the static rules) read
__global__ void k_replay_sources(TableView t, BatchView b, size_t n_inputs, const uint64_t* __restrict__ ids, const uint32_t* __restrict__ wm, uint64_t wm_mask, const uint32_t* __restrict__ tx_block,
                                 const ReplayRange* __restrict__ ranges, DevEntry* __restrict__ dent, UtxoSlot** __restrict__ slot, ReplaySrc* __restrict__ src) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs) return;
  const kgv_input& in = b.inputs[i];
  uint32_t k[9];
  input_key(k, in);
  SlotHead h;
  UtxoSlot* s = table_find(t, k, h);
  DevEntry d;
  ReplaySrc r;
  r.flag = RS_NONE << 30; r.src_tx = 0;
  if (s) { head_to_entry(d, t, s, h); r.flag = RS_TABLE << 30; }
  else {
    entry_absent(d);
    uint64_t id[4];
#pragma unroll
    for (int w = 0; w < 4; w++) id[w] = (uint64_t)k[2 * w] | ((uint64_t)k[2 * w + 1] << 32);
    int j = wm_find(ids, wm, wm_mask, id);
    if (j >= 0) {
      const kgv_tx& stx = b.txs[j];
      if (in.prev_index < stx.n_outputs) {
        const kgv_output& o = b.outputs[stx.first_output + in.prev_index];
        d.amount = o.value; d.script = b.bytes + o.script_off; d.script_len = o.script_len; d.spk_version = o.spk_version;
        d.is_coinbase = (tx_is_coinbase(stx) || ranges[tx_block[j]].t0 == (uint32_t)j) ? 1 : 0;  // the entry an accepted coinbase (position 0) leaves behind
        d.found = 1;
        r.flag = (RS_WINDOW << 30) | (stx.first_output + in.prev_index);
        r.src_tx = (uint32_t)j;
      }
    }
  }
  dent[i] = d;
  slot[i] = s;
  src[i] = r;
}
// static rules per transaction (entries as populated for the pre-check) + the pre-check's script verdict folded into one record.
// A transaction whose DAA-score rules (coinbase maturity, relative locks) involve only entries whose DAA score is known up front is decided
// here completely; one that involves an entry created by a transaction SEVERAL sibling blocks carry leaves those two rules to the walk (bits & 2), which then applies the rules in the
// reference's order: maturity, [amounts, mass = static_status], sequence locks.
__global__ void k_replay_static(BatchView b, uint32_t n_txs, kgv_params prm, const ReplayRange* __restrict__ ranges, const uint32_t* __restrict__ tx_block,
                                const kgv_tx_result* __restrict__ pre, const ReplaySrc* __restrict__ src, const uint64_t* __restrict__ ids, const uint32_t* __restrict__ wm, uint64_t wm_mask,
                                const uint8_t* __restrict__ has_sibling, ReplayTxInfo* __restrict__ info, uint64_t* __restrict__ fee, uint32_t* __restrict__ sfail) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  const kgv_tx& t = b.txs[ti];
  ReplayTxInfo o;
  o.first_input = t.first_input; o.n_inputs = t.n_inputs; o.static_status = KGV_TX_OK; o.bits = 0; o.pad_ = 0;
  {
    int j = wm_find(ids, wm, wm_mask, ids + 4 * (size_t)ti);
    o.rep = j >= 0 ? (uint32_t)j : ti;
    if (has_sibling[o.rep]) o.bits |= 8;
  }
  const ReplayRange r = ranges[tx_block[ti]];
  const bool cb = ti == r.t0 || tx_is_coinbase(t);
  if (cb) o.bits |= 1;
  if (pre[ti].status == KGV_TX_OK) o.bits |= 4;
  uint64_t f = 0;
  uint32_t fail = 0;
  if (!cb) {
    const DevEntry* ent = b.entries + t.first_input;
    const ReplaySrc* sr = src + t.first_input;
    // DAA score of the entry input i spends: the table's, or - created inside the window - the pov of the block that accepts the creator.  A creator
    // with a single instance in the window can only be accepted in its own block; one that several sibling blocks carry is left to the walk.
    auto entry_daa = [&](uint32_t i) -> uint64_t { return rs_kind(sr[i]) == RS_WINDOW ? ranges[tx_block[sr[i].src_tx]].pov : ent[i].block_daa_score; };
    bool all = true, dyn = false;
    for (uint32_t i = 0; i < t.n_inputs; i++) {
      all = all && ent[i].found;
      const bool needs_daa = ent[i].is_coinbase || !(b.inputs[t.first_input + i].sequence & (1ull << 63));
      dyn = dyn || (needs_daa && rs_kind(sr[i]) == RS_WINDOW && has_sibling[sr[i].src_tx]);
    }
    if (dyn) o.bits |= 2;
    if (all) {  // the order of tx_context_rules (kgv_context.cuh)
      uint8_t st = KGV_TX_OK;
      if (!dyn)
        for (uint32_t i = 0; i < t.n_inputs; i++)
          if (ent[i].is_coinbase && entry_daa(i) + prm.coinbase_maturity > r.pov) { st = KGV_TX_IMMATURE_COINBASE; fail = i; break; }
      uint64_t total_in = 0;
      for (uint32_t i = 0; i < t.n_inputs && st == KGV_TX_OK; i++) {
        if (ck_add(total_in, ent[i].amount, total_in)) st = KGV_TX_INPUT_AMOUNT_OVERFLOW;
        else if (total_in > prm.max_sompi) st = KGV_TX_INPUT_AMOUNT_TOO_HIGH;
      }
      if (st == KGV_TX_OK) {
        uint64_t total_out = 0;
        for (uint32_t i = 0; i < t.n_outputs; i++) total_out += b.outputs[t.first_output + i].value;
        if (total_in < total_out) st = KGV_TX_SPEND_TOO_HIGH;
        else f = total_in - total_out;
      }
      if (st == KGV_TX_OK) {
        uint64_t mass;
        const kgv_output* outs = b.outputs + t.first_output;
        bool ok = storage_mass(mass, false, t.n_inputs, t.n_outputs, [&](uint32_t i) -> const DevEntry& { return ent[i]; },
                               [&](uint32_t i, uint64_t& v, uint32_t& l) { v = outs[i].value; l = outs[i].script_len; }, prm.storage_mass_parameter);
        if (!ok) st = KGV_TX_MASS_INCOMPUTABLE;
        else if (mass != t.mass) st = KGV_TX_WRONG_MASS;
      }
      if (st == KGV_TX_OK && !dyn)
        for (uint32_t i = 0; i < t.n_inputs; i++) {
          const uint64_t seq = b.inputs[t.first_input + i].sequence;
          if (seq & (1ull << 63)) continue;
          const long long lock = (long long)entry_daa(i) + (long long)(seq & 0xFFFFFFFFull) - 1;
          if (lock >= (long long)r.pov) { st = KGV_TX_SEQUENCE_LOCK; break; }
        }
      o.static_status = st;
    }
  }
  info[ti] = o;
  fee[ti] = f;
  sfail[ti] = fail;
}

// The walk.  One CTA of 256 threads (a 10-BPS block carries ~150 transactions; every extra warp only adds issue pressure to the one SM).  Each
// block's records (16 bytes per transaction, 8 per input) and the range record two blocks ahead are fetched into shared memory by the copy
// engine - cp.async.bulk issued by thread 0, completion on an mbarrier - ONE block ahead of their use: no thread spends instructions or
// registers on staging, and the global-memory latency hides behind the current block's decide / commit.
#define RW_THREADS 256u
#define RW_MAXT 512u
#define RW_MAXI 1024u
#define RW_STAGE_BYTES (RW_MAXT * 16u + (RW_MAXI + 2u) * 8u)  // one staging buffer (inputs are copied from an even index: one entry of slack either side)
#define RW_FIXED_BYTES (2u * RW_STAGE_BYTES + 3u * 48u + 16u) // two staging buffers, a ring of three range records, two mbarriers
struct WalkArgs {
  const ReplayRange* ranges;
  uint32_t n_blocks;
  const ReplayTxInfo* info;
  const ReplaySrc* src;
  const DevEntry* dent;       // entries of the pre-check (DAA score / coinbase flag), rare path only
  const kgv_input* inputs;    // sequence numbers, rare path only
  volatile unsigned long long* acc_pov;  // per representative tx: pov of the block that accepted it
  uint8_t* w_status;          // verdict of the transactions whose DAA-score rules the walk decides (bits & 2)
  uint32_t* w_fail;           // failing input for such an ImmatureCoinbaseSpend
  uint8_t* accept;            // scratch for blocks beyond 256 transactions
  uint32_t* bm_spent_in;      // global copies of the bitmaps (written at the end; used directly when they do not fit shared memory)
  uint32_t* bm_spent_out;
  uint32_t* bm_accepted;      // per representative transaction
  uint32_t* bm_exists;        // per transaction: every input existed at its block's position
  uint32_t words_in, words_out, words_tx;
  uint64_t coinbase_maturity;
  unsigned long long* stats;
  int use_smem;
};
__device__ __forceinline__ bool bm_get(const uint32_t* bm, uint32_t i) { return (*(const volatile uint32_t*)&bm[i >> 5] >> (i & 31)) & 1u; }
__device__ __forceinline__ void bm_set(uint32_t* bm, uint32_t i) { atomicOr(&bm[i >> 5], 1u << (i & 31)); }

// decide / commit of one block.  Force-inlined into call sites whose pointer arguments have a KNOWN address space (shared staging + shared bitmaps
// on the common path): with pointers selected at run time the compiler falls back to generic loads and to a compare-and-swap loop per atomicOr,
// which cost 3x the whole walk (measured: 3.7 k -> cycles per block, DESIGN.md §4).
__device__ __forceinline__ bool walk_decide(const WalkArgs& a, const ReplayRange& bl, const ReplayTxInfo* p_info, const ReplaySrc* p_src, const uint32_t* spent_in,
                                            const uint32_t* spent_out, const uint32_t* accepted, uint32_t* exists, uint32_t tid, uint32_t nth, uint32_t& n_acc) {
  const bool verify_only = (bl.flags & KGV_REPLAY_VERIFY_ONLY) != 0;
  bool acc_first = false;  // the verdict of this thread's first transaction stays in a register (blocks beyond 256 transactions re-read the others)
  for (uint32_t ti = bl.t0 + tid; ti < bl.t1; ti += nth) {
    const ReplayTxInfo o = p_info[ti];
    uint8_t st = KGV_TX_OK;
    bool acc;
    if (o.bits & 1) {
      acc = (ti == bl.t0) && (bl.flags & KGV_REPLAY_ACCEPT_COINBASE);
    } else {
      for (uint32_t i = 0; i < o.n_inputs; i++) {
        const ReplaySrc sr = p_src[o.first_input + i];
        const uint32_t kd = rs_kind(sr), fl = sr.flag & RS_FLAG_MASK;
        bool ex = false;
        if (kd == RS_TABLE) ex = !bm_get(spent_in, fl);
        else if (kd == RS_WINDOW) ex = bm_get(accepted, sr.src_tx) && !bm_get(spent_out, fl);
        if (!ex) { st = KGV_TX_MISSING_OUTPOINTS; break; }
      }
      if (st == KGV_TX_OK && (o.bits & 2)) {  // rare: coinbase maturity (tx_validation_in_utxo_context.rs:75-91) on an entry whose creator sibling blocks share
        for (uint32_t i = 0; i < o.n_inputs; i++) {
          const uint32_t gi = o.first_input + i;
          const DevEntry& e = a.dent[gi];
          const ReplaySrc sr = p_src[gi];
          const uint64_t daa = rs_kind(sr) == RS_TABLE ? e.block_daa_score : a.acc_pov[sr.src_tx];
          if (e.is_coinbase && daa + a.coinbase_maturity > bl.pov) { st = KGV_TX_IMMATURE_COINBASE; a.w_fail[ti] = i; break; }
        }
      }
      if (st == KGV_TX_OK) st = o.static_status;
      if (st == KGV_TX_OK && (o.bits & 2)) {  // rare: relative sequence locks (:130-155)
        for (uint32_t i = 0; i < o.n_inputs; i++) {
          const uint32_t gi = o.first_input + i;
          const uint64_t seq = a.inputs[gi].sequence;
          if (seq & (1ull << 63)) continue;
          const ReplaySrc sr = p_src[gi];
          const uint64_t daa = rs_kind(sr) == RS_TABLE ? a.dent[gi].block_daa_score : a.acc_pov[sr.src_tx];
          const long long lock = (long long)daa + (long long)(seq & 0xFFFFFFFFull) - 1;
          if (lock >= (long long)bl.pov) { st = KGV_TX_SEQUENCE_LOCK; break; }
        }
      }
      if (st != KGV_TX_MISSING_OUTPOINTS) bm_set(exists, ti);
      if (o.bits & 2) a.w_status[ti] = st;  // rare
      acc = st == KGV_TX_OK && ((bl.flags & KGV_REPLAY_SKIP_SCRIPTS) || (o.bits & 4));
    }
    if (verify_only) acc = false;
    if (ti == bl.t0 + tid) acc_first = acc;
    else a.accept[ti] = acc ? 1 : 0;        // blocks beyond 256 transactions only
    if (acc && !(o.bits & 1)) n_acc++;
  }
  return acc_first;
}
// accepted transactions spend their inputs and become visible to later blocks (UtxoDiff::add_transaction, utxo_diff.rs:233-247)
__device__ __forceinline__ void walk_commit(const WalkArgs& a, const ReplayRange& bl, const ReplayTxInfo* p_info, const ReplaySrc* p_src, uint32_t* spent_in, uint32_t* spent_out,
                                            uint32_t* accepted, uint32_t tid, uint32_t nth, bool acc_first) {
  if (bl.flags & KGV_REPLAY_VERIFY_ONLY) return;
  for (uint32_t ti = bl.t0 + tid; ti < bl.t1; ti += nth) {
    if (ti == bl.t0 + tid ? !acc_first : !a.accept[ti]) continue;  // (written by this very thread in walk_decide)
    const ReplayTxInfo o = p_info[ti];
    for (uint32_t i = 0; i < o.n_inputs; i++) {
      const ReplaySrc sr = p_src[o.first_input + i];
      if (rs_kind(sr) == RS_TABLE) bm_set(spent_in, sr.flag & RS_FLAG_MASK);
      else bm_set(spent_out, sr.flag & RS_FLAG_MASK);
    }
    bm_set(accepted, o.rep);
    if (o.bits & 8) a.acc_pov[o.rep] = bl.pov;  // rare: which sibling's block accepted it is only known here
  }
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {  // 16-byte aligned addresses and size
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}

// BM_SHARED: the four bitmaps live in shared memory (windows up to ~1.4 M flags); otherwise they are the global copies.
template <bool BM_SHARED>
__global__ void __launch_bounds__(RW_THREADS, 1) k_replay_walk(WalkArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];  // cp.async.bulk needs 16-byte destinations; every offset below is a multiple of 16
  const uint32_t tid = threadIdx.x, nth = blockDim.x;
  uint8_t* const stage0 = smem_raw;
  uint8_t* const stage1 = smem_raw + RW_STAGE_BYTES;
  ReplayRange* const ring = (ReplayRange*)(smem_raw + 2 * RW_STAGE_BYTES);
  uint64_t* const mbar = (uint64_t*)(smem_raw + 2 * RW_STAGE_BYTES + 3 * 48);
  // The loop below issues NO global store on its common path: its whole output is the four bitmaps, written out once at the end;
  // k_replay_verdicts turns them into per-transaction verdicts.
  const uint32_t bm_words = a.words_in + a.words_out + 2 * a.words_tx;
  uint32_t* const sm_bm = (uint32_t*)(smem_raw + RW_FIXED_BYTES);
  if (BM_SHARED)
    for (uint32_t w = tid; w < bm_words; w += nth) sm_bm[w] = 0;
  __shared__ unsigned int s_acc;
  uint32_t n_acc = 0;  // per thread, reduced once at the end
  auto fits = [](const ReplayRange& r) { return r.t1 - r.t0 <= RW_MAXT && r.i1 - r.i0 <= RW_MAXI; };
  // copy group G(b) = { records of block b, range record of block b+1 }, completing on mbar[b & 1]; issued by thread 0 with range(b) in hand
  auto issue_group = [&](uint32_t b, const ReplayRange& r) {
    uint8_t* st = (b & 1) ? stage1 : stage0;
    uint64_t* bar = &mbar[b & 1];
    const uint32_t nt = r.t1 - r.t0, ie = r.i0 & ~1u, ni2 = (r.i1 - ie + 1u) & ~1u;
    const bool data = fits(r) && nt;
    const bool next = b + 1 < a.n_blocks;
    const uint32_t bytes = (data ? nt * 16u + ni2 * 8u : 0u) + (next ? 48u : 0u);
    mbar_expect_tx(bar, bytes);
    if (data) {
      bulk_g2s(st, a.info + r.t0, nt * 16u, bar);
      if (ni2) bulk_g2s(st + RW_MAXT * 16u, a.src + ie, ni2 * 8u, bar);
    }
    if (next) bulk_g2s(&ring[(b + 1) % 3], a.ranges + b + 1, 48u, bar);
  };
  if (tid == 0) {
    s_acc = 0;
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    ring[0] = a.ranges[0];
  }
  __syncthreads();
  if (tid == 0) issue_group(0, ring[0]);
  for (uint32_t bi = 0; bi < a.n_blocks; bi++) {
    mbar_wait(&mbar[bi & 1], (bi >> 1) & 1);  // records of this block + range of the next one have landed
    const ReplayRange bl = ring[bi % 3];
    if (tid == 0 && bi + 1 < a.n_blocks) issue_group(bi + 1, ring[(bi + 1) % 3]);  // its buffers were last read before the barrier that ended iteration bi-1
    const bool staged = fits(bl);
    const uint8_t* sp = (bi & 1) ? stage1 : stage0;
    bool acc_first;
    // ---- decide: every transaction reads the flags of its inputs (state as of the previous block); barrier; commit
    if (BM_SHARED && staged) {
      uint32_t *spent_in = sm_bm, *spent_out = sm_bm + a.words_in, *accepted = spent_out + a.words_out, *exists = accepted + a.words_tx;
      const ReplayTxInfo* p_info = (const ReplayTxInfo*)sp - bl.t0;
      const ReplaySrc* p_src = (const ReplaySrc*)(sp + RW_MAXT * 16u) - (bl.i0 & ~1u);
      acc_first = walk_decide(a, bl, p_info, p_src, spent_in, spent_out, accepted, exists, tid, nth, n_acc);
      __syncthreads();
      walk_commit(a, bl, p_info, p_src, spent_in, spent_out, accepted, tid, nth, acc_first);
    } else if (BM_SHARED) {  // a block too large for the staging area: records straight from global memory
      uint32_t *spent_in = sm_bm, *spent_out = sm_bm + a.words_in, *accepted = spent_out + a.words_out, *exists = accepted + a.words_tx;
      acc_first = walk_decide(a, bl, a.info, a.src, spent_in, spent_out, accepted, exists, tid, nth, n_acc);
      __syncthreads();
      walk_commit(a, bl, a.info, a.src, spent_in, spent_out, accepted, tid, nth, acc_first);
    } else {                 // a window too large for shared-memory bitmaps
      const ReplayTxInfo* p_info = staged ? (const ReplayTxInfo*)sp - bl.t0 : a.info;
      const ReplaySrc* p_src = staged ? (const ReplaySrc*)(sp + RW_MAXT * 16u) - (bl.i0 & ~1u) : a.src;
      acc_first = walk_decide(a, bl, p_info, p_src, a.bm_spent_in, a.bm_spent_out, a.bm_accepted, a.bm_exists, tid, nth, n_acc);
      __syncthreads();
      walk_commit(a, bl, p_info, p_src, a.bm_spent_in, a.bm_spent_out, a.bm_accepted, tid, nth, acc_first);
    }
    __syncthreads();
  }
  if (BM_SHARED)
    for (uint32_t w = tid; w < bm_words; w += nth) a.bm_spent_in[w] = sm_bm[w];  // the global copies are laid out back to back like the shared ones
  for (int off = 16; off; off >>= 1) n_acc += __shfl_down_sync(0xFFFFFFFFu, n_acc, off);
  if ((tid & 31) == 0 && n_acc) atomicAdd(&s_acc, n_acc);
  __syncthreads();
  if (tid == 0) a.stats[0] = s_acc;
}

// bitmaps of the walk -> per-transaction verdict of the UTXO-context rules, the acceptance flag, and the DAA score accepted outputs carry
__global__ void k_replay_verdicts(uint32_t n_txs, const ReplayRange* __restrict__ ranges, const uint32_t* __restrict__ tx_block, const ReplayTxInfo* __restrict__ info,
                                  const uint32_t* __restrict__ bm_exists, uint8_t* __restrict__ w_status, uint8_t* __restrict__ accept, unsigned long long* __restrict__ acc_pov) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  const ReplayTxInfo o = info[ti];
  const ReplayRange bl = ranges[tx_block[ti]];
  uint8_t st;
  bool acc;
  if (o.bits & 1) {
    st = KGV_TX_SKIPPED_COINBASE;
    acc = (ti == bl.t0) && (bl.flags & KGV_REPLAY_ACCEPT_COINBASE);
  } else {
    st = !bm_get(bm_exists, ti) ? KGV_TX_MISSING_OUTPOINTS : ((o.bits & 2) ? w_status[ti] : o.static_status);
    acc = st == KGV_TX_OK && ((bl.flags & KGV_REPLAY_SKIP_SCRIPTS) || (o.bits & 4));
  }
  if (bl.flags & KGV_REPLAY_VERIFY_ONLY) acc = false;
  w_status[ti] = st;
  accept[ti] = acc ? 1 : 0;
  if (acc && !(o.bits & 8)) acc_pov[o.rep] = bl.pov;  // (a transaction sibling blocks share: written by the walk)
}

// spent entries: captured for the MuHash consumers (entry as it was when spent), then erased from the table
__global__ void k_replay_finish_inputs(TableView t, BatchView b, size_t n_inputs, const uint32_t* __restrict__ itx, const uint8_t* __restrict__ accept,
                                       UtxoSlot* const* __restrict__ slot, const ReplaySrc* __restrict__ src, const unsigned long long* __restrict__ acc_pov, DevEntry* __restrict__ dent,
                                       uint8_t* __restrict__ spent_scripts) {
  __shared__ int s_live, s_tomb;
  if (threadIdx.x == 0) { s_live = 0; s_tomb = 0; }
  __syncthreads();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_inputs && accept[itx[i]]) {
  DevEntry d = dent[i];
  const uint32_t kd = rs_kind(src[i]);
  if (kd == RS_TABLE) {
    UtxoSlot* s = slot[i];
    if (d.script_len <= INLINE_SCRIPT) {  // the slot is about to be tombstoned (and may be reused): keep the script bytes
      uint32_t* dst = (uint32_t*)(spent_scripts + 72 * i);
      const uint32_t* sp = (const uint32_t*)((const uint8_t*)s + SLOT_SCRIPT_BYTE);
      const uint32_t nw = (d.script_len + 3) >> 2;
      for (uint32_t w = 0; w < nw; w++) dst[w] = __ldcg(sp + w);
      d.script = (const uint8_t*)dst;
      dent[i] = d;
    }
    uint32_t k[9];
    input_key(k, b.inputs[i]);
    table_erase_found(t, k, s, s >= t.slots && s <= t.slots + t.mask, &s_live, &s_tomb);
  } else if (kd == RS_WINDOW) {
    d.block_daa_score = acc_pov[src[i].src_tx];  // the entry existed with the accepting block's DAA score (utxo_diff.rs:240-245)
    dent[i] = d;
  }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_live) atomicAdd(&t.counters[0], (unsigned long long)(long long)s_live);
    if (s_tomb) atomicAdd(&t.counters[1], (unsigned long long)(long long)s_tomb);
  }
}
// outputs of accepted transactions that nobody spent inside the window
__global__ void k_replay_finish_outputs(TableView t, BatchView b, size_t n_outputs, const uint32_t* __restrict__ otx, const uint8_t* __restrict__ accept,
                                        const uint32_t* __restrict__ bm_spent_out, const uint64_t* __restrict__ ids, const unsigned long long* __restrict__ acc_pov,
                                        const ReplayTxInfo* __restrict__ info) {
  __shared__ int s_live, s_tomb;
  if (threadIdx.x == 0) { s_live = 0; s_tomb = 0; }
  __syncthreads();
  size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o < n_outputs) {
    const uint32_t ti = otx[o];
    const uint32_t r = info[ti].rep;
    // the representative instance stores the outputs (several accepted instances of one id would store the same entries)
    if (accept[ti] && (r == ti || !accept[r])) {
      const kgv_tx& tx = b.txs[ti];
      const uint32_t k_out = (uint32_t)(o - tx.first_output);
      if (!bm_get(bm_spent_out, b.txs[r].first_output + k_out)) {
        const kgv_output& out = b.outputs[o];
        uint32_t k[9];
#pragma unroll
        for (int w = 0; w < 4; w++) { uint64_t q = ids[4 * (size_t)ti + w]; k[2 * w] = (uint32_t)q; k[2 * w + 1] = (uint32_t)(q >> 32); }
        k[8] = k_out;
        table_put(t, k, out.value, acc_pov[r], out.spk_version, (info[ti].bits & 1) ? 1u : 0u, b.bytes + out.script_off, out.script_len, &s_live, &s_tomb);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_live) atomicAdd(&t.counters[0], (unsigned long long)(long long)s_live);
    if (s_tomb) atomicAdd(&t.counters[1], (unsigned long long)(long long)s_tomb);
  }
}
__global__ void k_replay_finish_results(uint32_t n_txs, const ReplayRange* __restrict__ ranges, const uint32_t* __restrict__ tx_block, const ReplayTxInfo* __restrict__ info,
                                        const uint8_t* __restrict__ w_status, const uint32_t* __restrict__ w_fail, const uint32_t* __restrict__ sfail,
                                        const uint64_t* __restrict__ fee, const kgv_tx_result* __restrict__ pre, kgv_tx_result* __restrict__ res) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  kgv_tx_result r;
  r.fee = 0; r.fail_input = 0; r.status = w_status[ti]; r.script_err = 0; r.pad_[0] = r.pad_[1] = 0;
  if (r.status == KGV_TX_IMMATURE_COINBASE) r.fail_input = (info[ti].bits & 2) ? w_fail[ti] : sfail[ti];
  const uint8_t st = r.status;
  // the fee is known once the amounts passed (tx_context_rules sets it before the mass / sequence-lock rules)
  if (st == KGV_TX_OK || st == KGV_TX_MASS_INCOMPUTABLE || st == KGV_TX_WRONG_MASS || st == KGV_TX_SEQUENCE_LOCK) r.fee = fee[ti];
  if (st == KGV_TX_OK && !(ranges[tx_block[ti]].flags & KGV_REPLAY_SKIP_SCRIPTS)) {
    const kgv_tx_result p = pre[ti];
    if (p.status != KGV_TX_OK && p.status != KGV_PRE_SKIPPED) { r.status = p.status; r.script_err = p.script_err; r.fail_input = p.fail_input; }
  }
  res[ti] = r;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
extern "C" int kgv_replay_window(kgv_ctx* ctx, kgv_utxo_table* table, const kgv_tx_batch* batch, const kgv_replay_block* blocks, size_t n_blocks,
                                 const kgv_params* prm, kgv_tx_result* results, uint8_t* accept, kgv_replay_stats* stats) {
  if (!ctx || !table) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || !prm || (n_blocks && !blocks) || (batch->n_txs && !results)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"blocks", blocks}, {"params", prm}, {"stats", stats}})
    if (int rc = kgv_host_only(ctx, "kgv_replay_window", what, p)) return rc;
  if (stats) { stats->n_accepted = 0; stats->n_sig_checks = 0; stats->n_host_vm = 0; stats->pre_check_ms = 0; stats->in_order_ms = 0; }
  if (batch->n_txs == 0 || n_blocks == 0) return KGV_OK;
  if (n_blocks > 0xFFFFFFFFull) { ctx->err = "too many blocks"; return KGV_ERR_ARG; }
  if (batch->n_inputs > RS_FLAG_MASK || batch->n_outputs > RS_FLAG_MASK) { ctx->err = "a replay window holds at most 2^30 - 1 inputs / outputs"; return KGV_ERR_LIMIT; }
  // the blocks must tile the batch in order (block b = transactions [first_tx, first_tx + n_txs))
  {
    uint64_t at = 0;
    for (size_t i = 0; i < n_blocks; i++) {
      if (blocks[i].first_tx != at || blocks[i].flags > 7u) { ctx->err = "kgv_replay_window: replay blocks must tile the batch contiguously, in order, with known flags"; return KGV_ERR_ARG; }
      at += blocks[i].n_txs;
    }
    if (at != batch->n_txs) { ctx->err = "kgv_replay_window: replay blocks do not cover the batch"; return KGV_ERR_ARG; }
  }
  CK(cudaSetDevice(ctx->device));
  // a write on the table replayed into, a read on the layers below it: mempool calls on the base run beside a replay into a view over it
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_replay_window", table, table)) return rc;
  int rc = utxo_reserve(ctx, table, batch->n_outputs + (table->base ? batch->n_inputs : 0), batch->n_bytes + 8 * (uint64_t)batch->n_outputs);
  if (rc) return rc;
  kgv_dev_batch d;
  rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  const size_t nt = d.n_txs, ni = d.n_inputs, no = d.n_outputs;
  uint64_t wm_cap = 1024;
  while (wm_cap < 2 * nt) wm_cap <<= 1;
  // state of the walk
  uint64_t sm_cap = 1024;
  while (sm_cap < 2 * ni) sm_cap <<= 1;
  const uint32_t words_in = (uint32_t)((ni + 31) / 32), words_out = (uint32_t)((no + 31) / 32), words_tx = (uint32_t)((nt + 31) / 32);
  const size_t bm_words = (size_t)words_in + words_out + 2 * (size_t)words_tx;
  uint64_t *ids, *fee;
  uint32_t *wm, *txb, *itx, *otx, *sfail, *wfl, *bm, *smv;
  kgv_tx_result *pre, *res;
  uint8_t *dacc, *scr, *sib, *wst;
  unsigned long long *cnt, *apov, *smk;
  kgv_replay_block* dblk;
  DevEntry* dent;
  UtxoSlot** slotp;
  ReplayRange* ranges;
  ReplaySrc* src;
  ReplayTxInfo* info;
  rc = kgv_reserve_carved(ctx, &ctx->d_replay, &ctx->d_replay_cap, [&](kgv_carve& c) {
    // window state
    ids = c.take<uint64_t>(nt * 4); wm = c.take<uint32_t>(wm_cap); dblk = c.take<kgv_replay_block>(n_blocks);
    txb = c.take<uint32_t>(nt); itx = c.take<uint32_t>(ni); otx = c.take<uint32_t>(no); dent = c.take<DevEntry>(ni);
    pre = c.take<kgv_tx_result>(nt); res = c.take<kgv_tx_result>(nt); dacc = c.take<uint8_t>(nt);
    scr = c.take<uint8_t>(ni * 72); slotp = c.take<UtxoSlot*>(ni); ranges = c.take<ReplayRange>(n_blocks); cnt = c.take<unsigned long long>(8);
    // state of the walk
    sib = c.take<uint8_t>(nt); src = c.take<ReplaySrc>(ni); sfail = c.take<uint32_t>(nt); info = c.take<ReplayTxInfo>(nt);
    fee = c.take<uint64_t>(nt); wst = c.take<uint8_t>(nt); wfl = c.take<uint32_t>(nt); apov = c.take<unsigned long long>(nt);
    bm = c.take<uint32_t>(bm_words); smk = c.take<unsigned long long>(sm_cap); smv = c.take<uint32_t>(sm_cap);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if (stats) {
    for (cudaEvent_t& e : ctx->ev_time) if (!e) CK(cudaEventCreate(&e));
    CK(cudaEventRecord(ctx->ev_time[0], st));
  }
  // KGV_DEBUG: device time between marks, printed at the end of the call
  std::vector<std::pair<const char*, cudaEvent_t>> marks;
  auto mark = [&](const char* name) {
    if (!kgv_debug_on()) return;
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return;
    cudaEventRecord(e, st);
    marks.push_back({name, e});
  };
  mark("start");
  CK(cudaMemcpyAsync(dblk, blocks, n_blocks * sizeof(kgv_replay_block), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(wm, 0, wm_cap * 4, st));
  CK(cudaMemsetAsync(cnt, 0, 64, st));
  if ((rc = kgv_tx_digests_run(ctx, d, nt, ids, false))) return rc;
  CK(cudaMemsetAsync(sib, 0, nt, st));
  k_wm_insert<<<nblk(nt, 128), 128, 0, st>>>(ids, (uint32_t)nt, wm, wm_cap - 1, sib);
  CK(cudaGetLastError());
  k_input_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, itx);
  CK(cudaGetLastError());
  k_output_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, otx);
  CK(cudaGetLastError());
  k_replay_tx_block<<<(unsigned)n_blocks, 128, 0, st>>>(dblk, (uint32_t)n_blocks, txb);
  CK(cudaGetLastError());
  k_replay_ranges<<<nblk(n_blocks, 128), 128, 0, st>>>(dblk, (uint32_t)n_blocks, d.txs, ranges);
  CK(cudaGetLastError());
  ctx->launches += 5;
  // ---- pre-check of every script of the window
  BatchView v{d.txs, d.inputs, d.outputs, dent, d.bytes};
  auto find_sources = [&]() -> int {
    if (!ni) return KGV_OK;
    k_replay_sources<<<nblk(ni, 128), 128, 0, st>>>(view_of(table), v, ni, ids, wm, wm_cap - 1, txb, ranges, dent, slotp, src);
    CK(cudaGetLastError());
    ctx->launches++;
    return KGV_OK;
  };
  mark("ids+window map+ranges");
  rc = find_sources();
  if (rc) return rc;
  mark("sources");
  k_replay_pre_status<<<nblk(nt, 128), 128, 0, st>>>(v, (uint32_t)nt, dblk, txb, pre);
  CK(cudaGetLastError());
  ctx->launches++;
  STAGE("replay pre-status");
  uint64_t n_items = 0;
  rc = kgv_scripts_phase(ctx, v, nt, ni, itx, pre, &n_items);
  if (rc) return rc;
  mark("scripts phase");
  k_count_status<<<nblk(nt, 256), 256, 0, st>>>(pre, (uint32_t)nt, KGV_TX_NEEDS_HOST_VM, cnt + 1);
  CK(cudaGetLastError());
  ctx->launches++;
  unsigned long long n_vm = 0;
  CK(cudaMemcpyAsync(&n_vm, cnt + 1, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (n_vm) {
    // non-standard scripts: the device script engine decides them on the entries the pre-check populated
    rc = kgv_script_engine_run(ctx, v, nt, nullptr, (size_t)n_vm, pre, true, nullptr);
    if (rc) return rc;
  }
  mark("script engine");
  if (stats) CK(cudaEventRecord(ctx->ev_time[1], st));
  // ---- the walk
  CK(cudaMemsetAsync(bm, 0, bm_words * 4, st));
  CK(cudaMemsetAsync(apov, 0, nt * 8, st));
  if (ni) {
    CK(cudaMemsetAsync(smk, 0, sm_cap * 8, st));
    CK(cudaMemsetAsync(smv, 0xFF, sm_cap * 4, st));
    k_slotmap_insert<<<nblk(ni, 256), 256, 0, st>>>(src, slotp, ni, smk, smv, sm_cap - 1);
    CK(cudaGetLastError());
    k_slotmap_lookup<<<nblk(ni, 256), 256, 0, st>>>(slotp, ni, smk, smv, sm_cap - 1, src);
    CK(cudaGetLastError());
    ctx->launches += 2;
  }
  mark("slot map");
  k_replay_static<<<nblk(nt, 128), 128, 0, st>>>(v, (uint32_t)nt, *prm, ranges, txb, pre, src, ids, wm, wm_cap - 1, sib, info, fee, sfail);
  CK(cudaGetLastError());
  ctx->launches++;
  mark("static rules");
  WalkArgs w;
  w.ranges = ranges; w.n_blocks = (uint32_t)n_blocks; w.info = info; w.src = src; w.dent = dent; w.inputs = d.inputs;
  w.acc_pov = apov; w.w_status = wst; w.w_fail = wfl; w.accept = dacc;
  w.bm_spent_in = bm; w.bm_spent_out = bm + words_in; w.bm_accepted = bm + words_in + words_out; w.bm_exists = bm + words_in + words_out + words_tx;
  w.words_in = words_in; w.words_out = words_out; w.words_tx = words_tx;
  w.coinbase_maturity = prm->coinbase_maturity; w.stats = cnt;
  const size_t stage_bytes = RW_FIXED_BYTES, walk_smem = stage_bytes + bm_words * 4;
  w.use_smem = walk_smem <= 200 * 1024;
  static bool walk_set = false;
  if (!walk_set) { CK(cudaFuncSetAttribute(k_replay_walk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); walk_set = true; }
  if (w.use_smem) k_replay_walk<true><<<1, RW_THREADS, walk_smem, st>>>(w);
  else k_replay_walk<false><<<1, RW_THREADS, stage_bytes, st>>>(w);
  CK(cudaGetLastError());
  ctx->launches++;
  mark("walk");
  k_replay_verdicts<<<nblk(nt, 256), 256, 0, st>>>((uint32_t)nt, ranges, txb, info, w.bm_exists, wst, dacc, apov);
  CK(cudaGetLastError());
  ctx->launches++;
  const TableView tv = view_of(table);
  if (ni) {
    k_replay_finish_inputs<<<nblk(ni, 128), 128, 0, st>>>(tv, v, ni, itx, dacc, slotp, src, apov, dent, scr);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  if (no) {
    k_replay_finish_outputs<<<nblk(no, 128), 128, 0, st>>>(tv, v, no, otx, dacc, bm + words_in, ids, apov, info);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  mark("finish inputs+outputs");
  k_replay_finish_results<<<nblk(nt, 256), 256, 0, st>>>((uint32_t)nt, ranges, txb, info, wst, wfl, sfail, fee, pre, res);
  CK(cudaGetLastError());
  ctx->launches++;
  mark("finish results");
  if (stats) CK(cudaEventRecord(ctx->ev_time[2], st));
  STAGE("replay in-order");
  if (!marks.empty()) {
    cudaStreamSynchronize(st);
    fprintf(stderr, "[kgv] replay window, device ms:");
    for (size_t i = 1; i < marks.size(); i++) {
      float ms = 0;
      cudaEventElapsedTime(&ms, marks[i - 1].second, marks[i].second);
      fprintf(stderr, "  %s %.3f", marks[i].first, ms);
    }
    fprintf(stderr, "\n");
    for (auto& m : marks) cudaEventDestroy(m.second);
  }
  kgv_io io(ctx);
  unsigned long long n_acc = 0;
  if ((rc = io.copy_out(results, res, nt * sizeof(kgv_tx_result)))) return rc;
  if (accept && (rc = io.copy_out(accept, dacc, nt))) return rc;
  if (stats && (rc = io.copy_out(&n_acc, cnt, 8))) return rc;
  if ((rc = io.finish())) return rc;
  ctx->last_replay.valid = true;
  ctx->last_replay.txs = d.txs; ctx->last_replay.inputs = d.inputs; ctx->last_replay.outputs = d.outputs; ctx->last_replay.bytes = d.bytes;
  ctx->last_replay.nt = nt; ctx->last_replay.ni = ni; ctx->last_replay.no = no; ctx->last_replay.n_blocks = n_blocks;
  ctx->last_replay.ids = ids; ctx->last_replay.itx = itx; ctx->last_replay.otx = otx; ctx->last_replay.ent = dent; ctx->last_replay.acc = dacc;
  ctx->last_replay.txb = txb; ctx->last_replay.rng = ranges;
  ctx->last_replay.src = src; ctx->last_replay.inf = info; ctx->last_replay.apv = apov;
  ctx->last_replay.blk = dblk; ctx->last_replay.res = res;
  ctx->last_replay.table = table; ctx->last_replay.rehashes = kgv_chain_rehashes(table);
  ctx->last_replay.block_flags.resize(n_blocks); ctx->last_replay.block_n_txs.resize(n_blocks);
  for (size_t i = 0; i < n_blocks; i++) { ctx->last_replay.block_flags[i] = blocks[i].flags; ctx->last_replay.block_n_txs[i] = blocks[i].n_txs; }
  if (stats) {
    stats->n_accepted = n_acc; stats->n_sig_checks = n_items; stats->n_host_vm = n_vm;
    CK(cudaEventElapsedTime(&stats->pre_check_ms, ctx->ev_time[0], ctx->ev_time[1]));
    CK(cudaEventElapsedTime(&stats->in_order_ms, ctx->ev_time[1], ctx->ev_time[2]));
  }
  return KGV_OK;
}


// ---------------------------------------------------------------------------------------------
// kgv_replay_muhash: MuHash::from_transaction of everything the last kgv_replay_window call accepted, combined per group of
// blocks (the mergeset of one chain block): what calculate_utxo_state folds into ctx.multiset_hash (utxo_validation.rs:120,144).
// Spent entries are the ones k_replay_finish_inputs captured (kept in the window state with their scripts).
// ---------------------------------------------------------------------------------------------
__global__ void k_replay_tx_pov(const ReplayRange* __restrict__ ranges, const uint32_t* __restrict__ tx_block, uint32_t n_txs, uint64_t* __restrict__ tx_pov, uint8_t* __restrict__ tx_first) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_txs) return;
  const ReplayRange r = ranges[tx_block[t]];
  tx_pov[t] = r.pov;
  tx_first[t] = t == r.t0 ? 1 : 0;
}
__global__ void __launch_bounds__(128) k_muhash_replay_elements(BatchView b, size_t n_inputs, size_t n_outputs, const uint32_t* __restrict__ input_tx, const uint32_t* __restrict__ output_tx,
                                                                const uint8_t* __restrict__ accept, const uint64_t* __restrict__ txids, const uint64_t* __restrict__ tx_pov,
                                                                const uint8_t* __restrict__ tx_first, uint32_t* __restrict__ e_den, uint32_t* __restrict__ e_num) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_inputs) {
    const uint32_t ti = input_tx[g];
    const DevEntry& e = b.entries[g];
    if (!accept[ti] || !e.found) return;  // never multiplied (flagged off in the range product)
    const kgv_input& in = b.inputs[g];
    uint32_t k[9];
    input_key(k, in);
    uint64_t d[4];
    muhash_utxo_digest(d, k, in.prev_index, e.block_daa_score, e.amount, e.is_coinbase != 0, e.spk_version, e.script, e.script_len);
    muhash_expand_store(e_den, n_inputs, g, d);
    return;
  }
  g -= n_inputs;
  if (g >= n_outputs) return;
  const uint32_t ti = output_tx[g];
  if (!accept[ti]) return;
  const kgv_tx& tx = b.txs[ti];
  const kgv_output& out = b.outputs[g];
  uint32_t k[8];
#pragma unroll
  for (int w = 0; w < 4; w++) { k[2 * w] = (uint32_t)txids[4 * (size_t)ti + w]; k[2 * w + 1] = (uint32_t)(txids[4 * (size_t)ti + w] >> 32); }
  uint64_t d[4];
  muhash_utxo_digest(d, k, (uint32_t)(g - tx.first_output), tx_pov[ti], out.value, tx_first[ti] || tx_is_coinbase(tx), out.spk_version, b.bytes + out.script_off, out.script_len);
  muhash_expand_store(e_num, n_outputs, g, d);
}
__global__ void k_replay_group_ranges(const ReplayRange* __restrict__ ranges, const uint32_t* __restrict__ group_first, uint32_t n_groups, uint32_t* __restrict__ ilo, uint32_t* __restrict__ ihi,
                                      uint32_t* __restrict__ olo, uint32_t* __restrict__ ohi) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const uint32_t b0 = group_first[g], b1 = group_first[g + 1];
  uint32_t i0 = 0, i1 = 0, o0 = 0, o1 = 0;
  bool any = false;
  for (uint32_t b = b0; b < b1; b++) {  // empty blocks carry no range
    const ReplayRange r = ranges[b];
    if (r.t1 == r.t0) continue;
    if (!any) { i0 = r.i0; o0 = r.o0; any = true; }
    i1 = r.i1; o1 = r.o1;
  }
  ilo[g] = i0; ihi[g] = any ? i1 : i0; olo[g] = o0; ohi[g] = any ? o1 : o0;
}

void kgv_replay_muhash_work::carve(kgv_carve& c, size_t nt, size_t n_groups) {
  pov = c.take<uint64_t>(nt); first = c.take<uint8_t>(nt);
  ilo = c.take<uint32_t>(n_groups); ihi = c.take<uint32_t>(n_groups); olo = c.take<uint32_t>(n_groups); ohi = c.take<uint32_t>(n_groups);
}
int kgv_replay_muhash_run(kgv_ctx* ctx, const uint32_t* dgf, size_t n_groups, const kgv_replay_muhash_work& w, uint32_t* vals, cudaStream_t st) {
  const auto& L = ctx->last_replay;
  const size_t nt = L.nt, ni = L.ni, no = L.no;
  uint32_t *e_den = nullptr, *e_num = nullptr;
  int rc = kgv_mu_reserve(ctx, ni, no, &e_den, &e_num);
  if (rc) return rc;
  k_replay_tx_pov<<<nblk(nt, 256), 256, 0, st>>>(L.rng, L.txb, (uint32_t)nt, w.pov, w.first);
  CK(cudaGetLastError());
  BatchView v{(const kgv_tx*)L.txs, (const kgv_input*)L.inputs, (const kgv_output*)L.outputs, L.ent, (const uint8_t*)L.bytes};
  if (ni + no) {
    k_muhash_replay_elements<<<nblk(ni + no, 128), 128, 0, st>>>(v, ni, no, L.itx, L.otx, L.acc, L.ids, w.pov, w.first, e_den, e_num);
    CK(cudaGetLastError());
  }
  k_replay_group_ranges<<<nblk(n_groups, 128), 128, 0, st>>>(L.rng, dgf, (uint32_t)n_groups, w.ilo, w.ihi, w.olo, w.ohi);
  CK(cudaGetLastError());
  ctx->launches += 3;
  // an input of an accepted transaction is always found (the context rules saw it), so accept[itx[j]] alone selects the denominators
  rc = kgv_mu_range_products(ctx, e_num, no, L.acc, L.otx, w.olo, w.ohi, (uint32_t)n_groups, vals, 192, st);
  if (rc) return rc;
  rc = kgv_mu_range_products(ctx, e_den, ni, L.acc, L.itx, w.ilo, w.ihi, (uint32_t)n_groups, vals + 96, 192, st);
  if (rc) return rc;
  return kgv_mu_canonicalize(ctx, vals, 96, 2 * n_groups, st);
}

extern "C" int kgv_replay_muhash(kgv_ctx* ctx, const uint32_t* group_first_block, size_t n_groups, uint8_t* values768) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n_groups == 0) return KGV_OK;
  if (!group_first_block || !values768) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (!ctx->last_replay.valid) { ctx->err = "kgv_replay_muhash must directly follow the kgv_replay_window call it refers to"; return KGV_ERR_ARG; }
  const auto& L = ctx->last_replay;
  if (int rc = kgv_host_only(ctx, "kgv_replay_muhash", "group_first_block", group_first_block)) return rc;
  if (group_first_block[0] != 0 || group_first_block[n_groups] != L.n_blocks) { ctx->err = "groups must tile the blocks of the window"; return KGV_ERR_ARG; }
  for (size_t i = 0; i < n_groups; i++) if (group_first_block[i] > group_first_block[i + 1]) { ctx->err = "group offsets not monotone"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = kgv_last_replay_read(ctx, acc, "kgv_replay_muhash")) return rc;
  cudaStream_t st = ctx->stream;
  // scratch (d_work is free between validation calls)
  uint32_t *dgf, *vals;
  kgv_replay_muhash_work w;
  int rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap,
                              [&](kgv_carve& c) { dgf = c.take<uint32_t>(n_groups + 1); w.carve(c, L.nt, n_groups); vals = c.take<uint32_t>(n_groups * 192); });
  if (rc) return rc;
  CK(cudaMemcpyAsync(dgf, group_first_block, (n_groups + 1) * 4, cudaMemcpyHostToDevice, st));
  rc = kgv_replay_muhash_run(ctx, dgf, n_groups, w, vals, st);
  if (rc) return rc;
  kgv_io io(ctx);
  if ((rc = io.copy_out(values768, vals, n_groups * 768))) return rc;
  return io.finish();
}

// ---------------------------------------------------------------------------------------------
// kgv_replay_diffs: the UtxoDiff of every group of blocks of the last kgv_replay_window call - ctx.mergeset_diff of calculate_utxo_state
// (utxo_validation.rs:119,148), i.e. UtxoDiff::add_transaction (utxo_diff.rs:224-260) over the group's accepted transactions in order.  No table
// access: everything comes from the state the walk leaves behind (source records, representative / accepted instance, accepting DAA
// score, the spent entries dent holds with their scripts captured).
//   removal   an input of an accepted transaction, unless it spends an output whose creator was accepted in the SAME group (the pair cancels)
//   addition  an output of the accepted instance of a transaction, unless an accepted transaction of the same group spends it
// Removals come in window input order and additions in window output order, so every group is a contiguous range of each list and the result does
// not depend on scheduling.  Script bytes are laid out group after group, each as [its removals' scripts][its additions' scripts].
// ---------------------------------------------------------------------------------------------
struct DiffArgs {
  const kgv_tx* txs;
  const kgv_input* inputs;
  const kgv_output* outputs;
  const uint8_t* bytes;
  const DevEntry* dent;            // spent entry of every input as found at its block's position (window state)
  const uint64_t* ids;
  const uint32_t *itx, *otx, *txb;
  const ReplayRange* ranges;
  const uint8_t* accept;
  const ReplaySrc* src;
  const ReplayTxInfo* info;
  const unsigned long long* acc_pov;
  uint32_t nt, ni, no, n_blocks;
  uint32_t* acc_inst;              // per representative: the instance that was accepted
  uint32_t* bgrp;                  // per block: its group
  uint32_t* spg;                   // per window output (representative numbering): group of its accepted spender, ~0 if none
  uint32_t *gi, *go;               // per group (n_groups + 1): first input / first output
  uint32_t *rflag, *rlen;          // per input: removal?  its script length if so
  uint32_t *aflag, *alen;          // per output: addition?  its script length if so
  unsigned long long *rs, *rb, *as, *ab;  // exclusive scans of the four arrays above (n + 1 entries: the last one is the total)
};

// a transaction id is accepted at most once in a window (a second instance finds its inputs spent) unless one block carries it twice:
// the smallest accepted instance then stands for it
__global__ void k_diff_acc_inst(DiffArgs a) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti < a.nt && a.accept[ti]) atomicMin(&a.acc_inst[a.info[ti].rep], ti);
}
__global__ void k_diff_groups(DiffArgs a, const uint32_t* __restrict__ gf, uint32_t n_groups) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n_groups) return;
  const uint32_t b0 = gf[g];
  const uint32_t t = b0 < a.n_blocks ? a.ranges[b0].t0 : a.nt;  // (an empty block's range still starts at its first_tx)
  a.gi[g] = t < a.nt ? a.txs[t].first_input : a.ni;
  a.go[g] = t < a.nt ? a.txs[t].first_output : a.no;
  if (g < n_groups)
    for (uint32_t b = b0; b < gf[g + 1]; b++) a.bgrp[b] = g;
}
// at most one accepted transaction spends a window output (the walk's spent flag)
__global__ void k_diff_spender_group(DiffArgs a) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.ni) return;
  const uint32_t ti = a.itx[i];
  if (!a.accept[ti]) return;
  const ReplaySrc r = a.src[i];
  if (rs_kind(r) == RS_WINDOW) a.spg[r.flag & RS_FLAG_MASK] = a.bgrp[a.txb[ti]];
}
__global__ void k_diff_classify(DiffArgs a) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < a.ni) {
    const uint32_t ti = a.itx[g];
    uint32_t f = 0;
    if (a.accept[ti]) {  // an accepted input always has a source (the walk found it)
      const ReplaySrc r = a.src[g];
      f = !(rs_kind(r) == RS_WINDOW && a.bgrp[a.txb[a.acc_inst[r.src_tx]]] == a.bgrp[a.txb[ti]]);
    }
    a.rflag[g] = f;
    a.rlen[g] = f ? a.dent[g].script_len : 0;
    return;
  }
  g -= a.ni;
  if (g >= a.no) return;
  const uint32_t ti = a.otx[g];
  uint32_t f = 0;
  if (a.accept[ti]) {
    const uint32_t r = a.info[ti].rep;
    if (a.acc_inst[r] == ti) f = a.spg[a.txs[r].first_output + ((uint32_t)g - a.txs[ti].first_output)] != a.bgrp[a.txb[ti]];
  }
  a.aflag[g] = f;
  a.alen[g] = f ? a.outputs[g].script_len : 0;
}
// the four exclusive scans, one block each, as k_exclusive_scan2 (64-bit sums: the byte totals are checked against the 32-bit script_off)
__global__ void __launch_bounds__(1024) k_diff_scan4(DiffArgs a, unsigned long long* __restrict__ totals) {
  const uint32_t* in = blockIdx.x == 0 ? a.rflag : blockIdx.x == 1 ? a.rlen : blockIdx.x == 2 ? a.aflag : a.alen;
  unsigned long long* out = blockIdx.x == 0 ? a.rs : blockIdx.x == 1 ? a.rb : blockIdx.x == 2 ? a.as : a.ab;
  const size_t n = blockIdx.x < 2 ? a.ni : a.no;
  __shared__ unsigned long long part[1024];
  const size_t per = (n + 1023) / 1024;
  const size_t lo = (size_t)threadIdx.x * per;
  const size_t hi = lo + per < n ? lo + per : n;
  unsigned long long s = 0;
  for (size_t i = lo; i < hi; i++) s += in[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    unsigned long long t = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  unsigned long long run = part[threadIdx.x] - s;
  for (size_t i = lo; i < hi; i++) {
    const uint32_t v = in[i];
    out[i] = run;
    run += v;
  }
  if (threadIdx.x == 1023) { out[n] = part[1023]; totals[blockIdx.x] = part[1023]; }
}
__global__ void k_diff_ranges(DiffArgs a, uint32_t n_groups, kgv_diff_range* __restrict__ out) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const uint32_t i0 = a.gi[g], i1 = a.gi[g + 1], o0 = a.go[g], o1 = a.go[g + 1];
  kgv_diff_range r;
  r.first_remove = a.rs[i0]; r.n_remove = a.rs[i1] - a.rs[i0];
  r.first_add = a.as[o0]; r.n_add = a.as[o1] - a.as[o0];
  out[g] = r;
}
__device__ __forceinline__ void store_key36(uint8_t* p, const uint32_t* k) {
  if ((((uintptr_t)p) & 3) == 0) {
#pragma unroll
    for (int w = 0; w < 9; w++) ((uint32_t*)p)[w] = k[w];
  } else {
#pragma unroll
    for (int w = 0; w < 9; w++) { p[4 * w] = (uint8_t)k[w]; p[4 * w + 1] = (uint8_t)(k[w] >> 8); p[4 * w + 2] = (uint8_t)(k[w] >> 16); p[4 * w + 3] = (uint8_t)(k[w] >> 24); }
  }
}
__global__ void k_diff_gather(DiffArgs a, uint8_t* __restrict__ rem_keys, kgv_utxo_entry* __restrict__ rem_entries, uint8_t* __restrict__ add_keys,
                              kgv_utxo_entry* __restrict__ add_entries, uint8_t* __restrict__ bytes) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t k[9];
  kgv_utxo_entry e;
  e.pad_[0] = e.pad_[1] = e.pad_[2] = e.pad_[3] = e.pad_[4] = 0;
  const uint8_t* scr;
  uint8_t* dst;
  if (g < a.ni) {
    if (!a.rflag[g]) return;
    const uint32_t grp = a.bgrp[a.txb[a.itx[g]]];
    const size_t j = a.rs[g];
    const unsigned long long off = a.rb[g] + a.ab[a.go[grp]];
    input_key(k, a.inputs[g]);
    store_key36(rem_keys + 36 * j, k);
    const DevEntry d = a.dent[g];
    e.amount = d.amount; e.block_daa_score = d.block_daa_score; e.script_off = (uint32_t)off; e.script_len = d.script_len; e.spk_version = d.spk_version;
    e.is_coinbase = d.is_coinbase;
    rem_entries[j] = e;
    scr = d.script; dst = bytes + off;
  } else {
    g -= a.ni;
    if (g >= a.no || !a.aflag[g]) return;
    const uint32_t ti = a.otx[g];
    const uint32_t grp = a.bgrp[a.txb[ti]];
    const size_t j = a.as[g];
    const unsigned long long off = a.rb[a.gi[grp + 1]] + a.ab[g];
#pragma unroll
    for (int w = 0; w < 4; w++) { const uint64_t q = a.ids[4 * (size_t)ti + w]; k[2 * w] = (uint32_t)q; k[2 * w + 1] = (uint32_t)(q >> 32); }
    k[8] = (uint32_t)g - a.txs[ti].first_output;
    store_key36(add_keys + 36 * j, k);
    const kgv_output& o = a.outputs[g];
    const ReplayTxInfo inf = a.info[ti];
    // the entry k_replay_finish_outputs stores and k_muhash_replay_elements hashes: the accepting block's DAA score, coinbase by position or subnetwork
    e.amount = o.value; e.block_daa_score = a.acc_pov[inf.rep]; e.script_off = (uint32_t)off; e.script_len = o.script_len; e.spk_version = o.spk_version;
    e.is_coinbase = (inf.bits & 1) ? 1 : 0;
    add_entries[j] = e;
    scr = a.bytes + o.script_off; dst = bytes + off;
  }
  for (uint32_t b = 0; b < e.script_len; b++) dst[b] = scr[b];
}

extern "C" int kgv_replay_diffs(kgv_ctx* ctx, const uint32_t* group_first_block, size_t n_groups, kgv_diff_range* ranges, uint8_t* rem_keys36,
                                kgv_utxo_entry* rem_entries, uint8_t* add_keys36, kgv_utxo_entry* add_entries, uint8_t* bytes, size_t max_rem, size_t max_add,
                                size_t bytes_cap, size_t* n_rem_out, size_t* n_add_out, size_t* bytes_out) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!group_first_block || n_groups == 0) { ctx->err = "kgv_replay_diffs: no groups"; return KGV_ERR_ARG; }
  if (!ctx->last_replay.valid) { ctx->err = "kgv_replay_diffs refers to the last kgv_replay_window call, and none is current (another batch was staged or the table rehashed since)"; return KGV_ERR_ARG; }
  const auto& L = ctx->last_replay;
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"group_first_block", group_first_block}, {"n_rem_out", n_rem_out}, {"n_add_out", n_add_out},
                                {"bytes_out", bytes_out}})
    if (int rc = kgv_host_only(ctx, "kgv_replay_diffs", what, p)) return rc;
  if (group_first_block[0] != 0 || group_first_block[n_groups] != L.n_blocks) { ctx->err = "groups must tile the blocks of the window"; return KGV_ERR_ARG; }
  for (size_t i = 0; i < n_groups; i++) if (group_first_block[i] > group_first_block[i + 1]) { ctx->err = "group offsets not monotone"; return KGV_ERR_ARG; }
  const bool counting = !rem_keys36;
  kgv_io io(ctx);
  if (!counting) {
    if (!rem_entries || !add_keys36 || !add_entries || (bytes_cap && !bytes)) { ctx->err = "null buffer"; return KGV_ERR_ARG; }
    bool dev;
    if (int rc = io.one_side("kgv_replay_diffs", {rem_keys36, rem_entries, add_keys36, add_entries, bytes, ranges}, &dev)) return rc;
    if (dev && (((uintptr_t)rem_entries | (uintptr_t)add_entries) & 7)) { ctx->err = "kgv_replay_diffs: device entry arrays must be 8-byte aligned"; return KGV_ERR_ARG; }
  }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = kgv_last_replay_read(ctx, acc, "kgv_replay_diffs")) return rc;
  cudaStream_t st = ctx->stream;
  const size_t nt = L.nt, ni = L.ni, no = L.no;
  // scratch (d_work is free between validation calls)
  DiffArgs a;
  uint32_t* dgf;
  kgv_diff_range* drg;
  unsigned long long* dtot;
  int rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap, [&](kgv_carve& c) {
    a.acc_inst = c.take<uint32_t>(nt); a.bgrp = c.take<uint32_t>(L.n_blocks); a.spg = c.take<uint32_t>(no);
    dgf = c.take<uint32_t>(n_groups + 1); a.gi = c.take<uint32_t>(n_groups + 1); a.go = c.take<uint32_t>(n_groups + 1);
    a.rflag = c.take<uint32_t>(ni); a.rlen = c.take<uint32_t>(ni); a.aflag = c.take<uint32_t>(no); a.alen = c.take<uint32_t>(no);
    a.rs = c.take<unsigned long long>(ni + 1); a.rb = c.take<unsigned long long>(ni + 1);
    a.as = c.take<unsigned long long>(no + 1); a.ab = c.take<unsigned long long>(no + 1);
    drg = c.take<kgv_diff_range>(n_groups); dtot = c.take<unsigned long long>(8);
  });
  if (rc) return rc;
  // the diffs come back up to their sizes, known after the scan
  uint8_t *rk = nullptr, *ak = nullptr, *db = nullptr;
  kgv_utxo_entry *re = nullptr, *ae = nullptr;
  if (!counting) {
    io.out(rem_keys36, max_rem * 36, &rk);
    io.out(rem_entries, max_rem * sizeof(kgv_utxo_entry), &re);
    io.out(add_keys36, max_add * 36, &ak);
    io.out(add_entries, max_add * sizeof(kgv_utxo_entry), &ae);
    io.out(bytes, bytes_cap, &db);
    if ((rc = io.stage())) return rc;
  }
  a.txs = (const kgv_tx*)L.txs; a.inputs = (const kgv_input*)L.inputs; a.outputs = (const kgv_output*)L.outputs; a.bytes = (const uint8_t*)L.bytes;
  a.dent = L.ent; a.ids = L.ids; a.itx = L.itx; a.otx = L.otx; a.txb = L.txb;
  a.ranges = L.rng; a.accept = L.acc; a.src = L.src; a.info = L.inf; a.acc_pov = L.apv;
  a.nt = (uint32_t)nt; a.ni = (uint32_t)ni; a.no = (uint32_t)no; a.n_blocks = (uint32_t)L.n_blocks;
  CK(cudaMemcpyAsync(dgf, group_first_block, (n_groups + 1) * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(a.acc_inst, 0xFF, nt * 4, st));
  if (no) CK(cudaMemsetAsync(a.spg, 0xFF, no * 4, st));
  k_diff_acc_inst<<<nblk(nt, 256), 256, 0, st>>>(a);
  CK(cudaGetLastError());
  k_diff_groups<<<nblk(n_groups + 1, 128), 128, 0, st>>>(a, dgf, (uint32_t)n_groups);
  CK(cudaGetLastError());
  if (ni) { k_diff_spender_group<<<nblk(ni, 256), 256, 0, st>>>(a); CK(cudaGetLastError()); }
  if (ni + no) { k_diff_classify<<<nblk(ni + no, 256), 256, 0, st>>>(a); CK(cudaGetLastError()); }
  k_diff_scan4<<<4, 1024, 0, st>>>(a, dtot);
  CK(cudaGetLastError());
  k_diff_ranges<<<nblk(n_groups, 128), 128, 0, st>>>(a, (uint32_t)n_groups, drg);
  CK(cudaGetLastError());
  ctx->launches += 6 + (ni ? 1 : 0) + (ni + no ? 1 : 0);
  unsigned long long tot[4];
  CK(cudaMemcpyAsync(tot, dtot, sizeof tot, cudaMemcpyDeviceToHost, st));
  if (ranges && (rc = io.copy_out(ranges, drg, n_groups * sizeof(kgv_diff_range)))) return rc;
  CK(cudaStreamSynchronize(st));
  const size_t n_rem = (size_t)tot[0], n_add = (size_t)tot[2], n_bytes = (size_t)(tot[1] + tot[3]);
  if (n_rem_out) *n_rem_out = n_rem;
  if (n_add_out) *n_add_out = n_add;
  if (bytes_out) *bytes_out = n_bytes;
  if (n_bytes > 0xFFFFFFFFull) { ctx->err = "kgv_replay_diffs: the script bytes of the diffs exceed the 32-bit script_off"; return KGV_ERR_LIMIT; }
  if (counting) return KGV_OK;
  if (n_rem > max_rem || n_add > max_add || n_bytes > bytes_cap) { ctx->err = "kgv_replay_diffs: the caller's arrays are too small (sizes returned)"; return KGV_ERR_NOMEM; }
  if (ni + no == 0) return KGV_OK;
  k_diff_gather<<<nblk(ni + no, 128), 128, 0, st>>>(a, rk, re, ak, ae, db);
  CK(cudaGetLastError());
  ctx->launches++;
  io.trim(rem_keys36, n_rem * 36);
  io.trim(rem_entries, n_rem * sizeof(kgv_utxo_entry));
  io.trim(add_keys36, n_add * 36);
  io.trim(add_entries, n_add * sizeof(kgv_utxo_entry));
  io.trim(bytes, n_bytes);
  return io.finish();
}
