// tests/emu/zk_emu.cu — TEST INFRASTRUCTURE: runs the product's gate programs (the same
// __host__ __device__ functions the CUDA kernels call) serially on the CPU, so that kernel
// logic can be diffed against the oracle locally before spending a GPU call.  Never shipped,
// never used by the product (which has no CPU path); built by tests/emu_lib.py with
// `nvcc -x cu` host compilation only.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../zkevm-specs_b200/csrc/bytecode.cu"
#include "../../zkevm-specs_b200/csrc/copy.cu"
#include "../../zkevm-specs_b200/csrc/evm.cu"
#include "../../zkevm-specs_b200/csrc/exp.cu"
#include "../../zkevm-specs_b200/csrc/pi.cu"
#include "../../zkevm-specs_b200/csrc/assign.cu"
#include "../../zkevm-specs_b200/csrc/state.cu"
#include "../../zkevm-specs_b200/csrc/tx.cu"
#include "../../zkevm-specs_b200/csrc/keccak.cuh"

using namespace zk;

// tests toggle this to store every matrix in the packed format (each column at the smallest of
// the widths 0/1/2/4/8/16/32 bytes that holds its values) instead of canonical 32-byte cells
extern "C" int g_emu_packed = 0;
extern "C" long long g_emu_narrow_cols = 0;
extern "C" long long g_emu_narrow_runs = 0;  // EVM checks that took the narrow kernel form (StepCtx::narrow)  // columns stored narrower than 32 bytes so far (tests assert > 0)
struct Store {  // owns the packed copy of a matrix
  std::vector<unsigned char> buf;
  u64 off[ZK_MAX_COLS];
  unsigned char width[ZK_MAX_COLS];
  const unsigned char* base = nullptr;
};
// `want`: if every column fits these widths, store exactly them (the layout k_bytecode_table_expand writes)
static void store_matrix(Store& st, const u64* cells, u64 n_rows, u32 n_cols, bool allow_pack = true,
                         const unsigned char* want = nullptr) {
  if (!g_emu_packed || !allow_pack || n_rows == 0) {
    layout_canonical(st.off, st.width, n_cols, n_rows);
    st.base = (const unsigned char*)cells;
    return;
  }
  size_t total = 0;
  for (u32 c = 0; c < n_cols; c++) {
    const u64* col = cells + (u64)c * n_rows * 4;
    u64 m0 = 0, m1 = 0, m23 = 0;
    bool constant = true;
    for (u64 r = 0; r < n_rows; r++) {
      m0 |= col[4 * r];
      m1 |= col[4 * r + 1];
      m23 |= col[4 * r + 2] | col[4 * r + 3];
      constant = constant && !memcmp(col + 4 * r, col, 32);
    }
    unsigned w = 32;
    if (constant) w = 0;
    else if (!m23 && !m1) w = m0 < 256 ? 1 : (m0 < 65536 ? 2 : (m0 < (1ull << 32) ? 4 : 8));
    else if (!m23) w = 16;
    st.width[c] = (unsigned char)w;
    g_emu_narrow_cols += w < 32;
    st.off[c] = total;
    total += ((w ? (size_t)w * n_rows : 32) + 31) / 32 * 32;
  }
  if (want) {
    bool fits = true;
    for (u32 c = 0; c < n_cols; c++) fits = fits && (st.width[c] <= want[c]);
    if (fits) {
      total = 0;
      for (u32 c = 0; c < n_cols; c++) {
        st.width[c] = want[c];
        st.off[c] = total;
        total += ((size_t)want[c] * n_rows + 31) / 32 * 32;
      }
    }
  }
  st.buf.assign(total + 32, 0);
  for (u32 c = 0; c < n_cols; c++) {
    const u64* col = cells + (u64)c * n_rows * 4;
    unsigned char* dst = st.buf.data() + st.off[c];
    const unsigned w = st.width[c];
    if (w == 0) memcpy(dst, col, 32);
    else
      for (u64 r = 0; r < n_rows; r++) memcpy(dst + r * w, col + 4 * r, w);  // little-endian host
  }
  st.base = st.buf.data();
}
static WitnessDev make_witness(Store& st, const u64* cells, u64 n_rows, u32 n_cols, const unsigned char* flags) {
  store_matrix(st, cells, n_rows, n_cols);
  WitnessDev w;
  w.base = st.base;
  w.n_rows = n_rows;
  w.flags = flags;
  for (u32 c = 0; c < ZK_MAX_COLS; c++) {
    w.off[c] = c < n_cols ? st.off[c] : 0;
    w.width[c] = c < n_cols ? st.width[c] : 32;
  }
  return w;
}

struct IndexStore {
  std::vector<u64> slots;
  Store st;
};
static IndexDev build_index(const u64* cells, u64 n_rows, u32 n_cols, const u32* key_cols, u32 n_key,
                            const Fr& challenge, IndexStore& own, bool allow_pack = true, const unsigned char* want = nullptr) {
  std::vector<u64>& slots = own.slots;
  store_matrix(own.st, cells, n_rows, n_cols, allow_pack, want);
  IndexDev d;
  d.tab.base = own.st.base;
  d.tab.n_rows = n_rows;
  d.tab.n_cols = n_cols;
  d.tab.flags = nullptr;
  for (u32 c = 0; c < ZK_MAX_TABLE_COLS; c++) {
    d.tab.off[c] = c < n_cols ? own.st.off[c] : 0;
    d.tab.width[c] = c < n_cols ? own.st.width[c] : 32;
  }
  size_t cap = 64;
  while (cap < 2 * n_rows) cap <<= 1;
  slots.assign(cap, ZK_EMPTY_SLOT);
  d.slots = slots.data();
  d.mask = (u32)(cap - 1);
  d.n_key = n_key;
  {  // hash keys: a splitmix64 stream seeded by the lookup challenge (as api.cu:ensure_index)
    const Fr& c = challenge;
    u64 x = c.l[0] ^ (c.l[1] * 0x9E3779B97F4A7C15ull) ^ (c.l[2] * 0xC2B2AE3D27D4EB4Full) ^ (c.l[3] * 0x165667B19E3779F9ull);
    auto next = [&x]() {
      x += 0x9E3779B97F4A7C15ull;
      u64 z = x;
      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
      z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
      return z ^ (z >> 31);
    };
    for (int k = 0; k < 4; k++) d.hk[k] = next() | 1ull;
    for (u32 j = 0; j < ZK_MAX_KEY; j++) {
      d.key_cols[j] = j < n_key ? key_cols[j] : 0;
      d.hm[j] = next() | 1ull;
    }
  }
  d.pos_ok = nullptr;
  d.pos_kind = ZK_POS_NONE;
  d.tail_key = -1;
  d.tail_col = d.tail_val = 0;
  d.heads = nullptr;
  d.heads_mask = 0;
  d.heads_list = d.heads_count = nullptr;
  for (u64 r = 0; r < n_rows; r++) index_insert_row(d, r);
  return d;
}
// positional structure of a table, verified exactly like k_pos_verify does on the device
struct PosState {
  u32 ok[2] = {1, 0};
  std::vector<HeadEnt> heads;
  std::vector<u32> aux;
};
// bit 0: the bytecode table, bit 1: the rw table of the last emu_check_evm_x / emu_check_copy call passed the
// verify pass (its lookups took the positional path)
extern "C" int g_emu_pos_ok = 0;
extern "C" unsigned emu_heads_cap() { return ZK_HEADS_CAP; }
static void add_positional(IndexDev& d, u32 kind, PosState& st) {
  d.pos_kind = kind;
  if (kind == ZK_POS_RUNS) {  // the device's heads index, at its real size (4 MB)
    HeadEnt empty;
    memset(&empty, 0xFF, sizeof(empty));
    st.heads.assign(ZK_HEADS_CAP, empty);
    st.aux.assign(ZK_HEADS_CAP + 1, 0);
    d.heads = st.heads.data();
    d.heads_mask = ZK_HEADS_CAP - 1;
    d.heads_list = st.aux.data();
    d.heads_count = st.aux.data() + ZK_HEADS_CAP;
  }
  st.ok[0] = 1;
  st.ok[1] = (u32)d.tab.n_rows;
  if (kind == ZK_POS_DENSE && d.tab.n_cols == 14) {  // the rw table: Start padding rows may form a tail run
    d.tail_col = 2;
    d.tail_val = 1;
    for (u32 j = 0; j < d.n_key; j++)
      if (d.key_cols[j] == 2) d.tail_key = (int)j;
  }
  for (u64 r = 0; r < d.tab.n_rows; r++) {
    if (kind == ZK_POS_DENSE) pos_verify_dense_row(d, st.ok, r);
    else pos_verify_run_row(d, st.ok, r);
  }
  if (kind == ZK_POS_RUNS && d.tab.n_rows) {  // k_pos_runlen
    const u32 count = *d.heads_count < d.heads_mask + 1 ? *d.heads_count : d.heads_mask + 1;
    for (u32 k = 0; k <= count; k++) pos_runlen_entry(d, k, count);
  }
  d.pos_ok = st.ok;
}
extern "C" int g_emu_positional = 1;  // tests toggle this to run both lookup paths

static void init_result(ResultDev& res, uint32_t* ff, uint64_t* fc, int n) {
  for (int i = 0; i < n; i++) { ff[i] = 0xFFFFFFFFu; fc[i] = 0; }
  res.first_fail = ff;
  res.fail_count = (u64*)fc;
}

extern "C" int emu_check_evm_x(const uint64_t* steps, uint64_t n_steps, const uint64_t* bytecode, uint64_t n_bytecode,
                               const uint64_t* rw, uint64_t n_rw, const uint8_t* rw_flags, const uint64_t* fixed,
                               uint64_t n_fixed, const uint64_t* copy, uint64_t n_copy, const uint64_t* keccak,
                               uint64_t n_keccak, uint64_t row_begin, uint64_t row_end, uint64_t row_base, uint32_t flags,
                               const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count);
static const u64* g_emu_tx = nullptr;
static const u64* g_emu_block = nullptr;
static u64 g_emu_n_tx = 0, g_emu_n_block = 0;
static const unsigned char *g_emu_tx_flags = nullptr, *g_emu_block_flags = nullptr;
static const u64* g_emu_wd = nullptr;
static u64 g_emu_n_wd = 0;
// value type flags of the tx / block tables and the withdrawal table of the NEXT emu_check_evm_x call
extern "C" void emu_set_evm_block_tables(const uint8_t* tx_flags, const uint8_t* block_flags, const uint64_t* wd, uint64_t n_wd) {
  g_emu_tx_flags = tx_flags;
  g_emu_block_flags = block_flags;
  g_emu_wd = (const u64*)wd;
  g_emu_n_wd = n_wd;
}
static const u64* g_emu_exp = nullptr;
static u64 g_emu_n_exp = 0;
// exp table (11 cells) of the NEXT emu_check_evm_x call
extern "C" void emu_set_evm_exp_table(const uint64_t* exp, uint64_t n_exp) {
  g_emu_exp = (const u64*)exp;
  g_emu_n_exp = n_exp;
}
static const u64* g_emu_aux = nullptr;
static u64 g_emu_n_aux = 0;
// step-aux side table (step row, lo, hi) of the NEXT emu_check_evm_x call
extern "C" void emu_set_evm_step_aux(const uint64_t* aux, uint64_t n_aux) {
  g_emu_aux = (const u64*)aux;
  g_emu_n_aux = n_aux;
}
extern "C" void emu_set_evm_context_tables(const uint64_t* tx, uint64_t n_tx, const uint64_t* block, uint64_t n_block) {
  g_emu_tx = (const u64*)tx;
  g_emu_n_tx = n_tx;
  g_emu_block = (const u64*)block;
  g_emu_n_block = n_block;
}
extern "C" int emu_check_evm(const uint64_t* steps, uint64_t n_steps, const uint64_t* bytecode, uint64_t n_bytecode,
                             const uint64_t* rw, uint64_t n_rw, const uint64_t* fixed, uint64_t n_fixed,
                             uint64_t row_begin, uint64_t row_end, uint64_t row_base, uint32_t flags,
                             const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  return emu_check_evm_x(steps, n_steps, bytecode, n_bytecode, rw, n_rw, nullptr, fixed, n_fixed, nullptr, 0, nullptr, 0,
                         row_begin, row_end, row_base, flags, challenge, first_fail, fail_count);
}
extern "C" int emu_check_evm_x(const uint64_t* steps, uint64_t n_steps, const uint64_t* bytecode, uint64_t n_bytecode,
                               const uint64_t* rw, uint64_t n_rw, const uint8_t* rw_flags, const uint64_t* fixed,
                               uint64_t n_fixed, const uint64_t* copy, uint64_t n_copy, const uint64_t* keccak,
                               uint64_t n_keccak, uint64_t row_begin, uint64_t row_end, uint64_t row_base, uint32_t flags,
                               const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 k5[5] = {0, 1, 2, 3, 4}, k4[4] = {0, 1, 2, 3};
  IndexStore s1, s2;
  EvmTables t;
  static const unsigned char kFromCode[6] = {16, 16, 1, 4, 1, 4};
  t.bytecode = build_index((const u64*)bytecode, n_bytecode, 6, k5, 5, ch, s1, true, kFromCode);
  t.rw = build_index((const u64*)rw, n_rw, 14, k5, 5, ch, s2);
  // the fixed table is the same array call after call: keep its index and bitmap
  struct FixedCache { const uint64_t* p = nullptr; uint64_t n = 0, sum = 0; Fr ch; IndexStore slots; IndexDev ix; std::vector<u32> bitmap; };
  static FixedCache fxc;
  u64 fx_sum = 0;
  for (u64 k = 0; k < 257 && n_fixed; k++) {
    const u64 r = (n_fixed - 1) * k / 256;
    for (u32 c = 0; c < 4; c++) fx_sum = fx_sum * 0x9E3779B97F4A7C15ull + fixed[((u64)c * n_fixed + r) * 4];
  }
  if (!(fxc.p == fixed && fxc.n == n_fixed && fxc.sum == fx_sum && fr_eq(fxc.ch, ch))) {
    fxc.ix = build_index((const u64*)fixed, n_fixed, 4, k4, 4, ch, fxc.slots, false);
    fxc.bitmap.assign(ZK_RESP_BITMAP_WORDS, 0);
    for (u64 r = 0; r < n_fixed; r++) resp_bitmap_row(fxc.ix.tab, fxc.bitmap.data(), r);
    fxc.p = fixed; fxc.n = n_fixed; fxc.sum = fx_sum; fxc.ch = ch;
  }
  t.fixed = fxc.ix;
  t.rw.tab.flags = rw_flags;
  const u32 ck[11] = {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12}, kk[3] = {0, 1, 2};
  IndexStore s4, s5;
  t.copy = build_index((const u64*)copy, n_copy, 14, ck, 11, ch, s4);
  t.keccak = build_index((const u64*)keccak, n_keccak, 5, kk, 3, ch, s5);
  // tx / block tables of the ORIGIN / GASPRICE / BlockCtx gadgets (set by emu_set_evm_context_tables)
  const u32 tk[3] = {0, 1, 2}, bk[2] = {0, 1};
  IndexStore s6, s7;
  t.tx = build_index(g_emu_tx, g_emu_n_tx, 5, tk, 3, ch, s6);
  t.block = build_index(g_emu_block, g_emu_n_block, 4, bk, 2, ch, s7);
  t.tx.tab.flags = g_emu_tx_flags;
  t.block.tab.flags = g_emu_block_flags;
  const u32 ek[9] = {0, 1, 2, 3, 4, 5, 6, 7, 8};
  IndexStore s11;
  t.exp = build_index(g_emu_exp, g_emu_n_exp, 11, ek, 9, ch, s11);
  g_emu_exp = nullptr;
  g_emu_n_exp = 0;
  const u32 ak[1] = {0};
  IndexStore s12;
  t.aux = build_index(g_emu_aux, g_emu_n_aux, 3, ak, 1, ch, s12);
  g_emu_aux = nullptr;
  g_emu_n_aux = 0;
  const u32 wk[1] = {0};
  IndexStore s8, s9;
  IndexDev wd_ix = build_index(g_emu_wd, g_emu_n_wd, 4, wk, 1, ch, s8);
  t.wd = wd_ix.tab;
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)steps, n_steps, 13, nullptr);
  // as api.cu:check_evm, the indexes and constants of es_needs only for the states of the checked steps; otherwise an
  // index without rows (every lookup there is unsat) and zeroed block stats, so that a missing needs bit fails here too
  unsigned needs = 0;
  for (u64 i = row_begin; i < row_end; i++) {
    const Fr cs = wcell(w, S_STATE, i);
    if (fr_fits64(cs) && cs.l[0] < ZK_ES_COUNT) needs |= es_needs((int)cs.l[0]);
  }
  t.rw_rwc = build_index((const u64*)rw, needs & RW_BY_COUNTER ? n_rw : 0, 14, wk, 1, ch, s9);
  if (needs & RW_BY_COUNTER) t.rw_rwc.tab = t.rw.tab;  // same storage choice as t.rw (same matrix)
  IndexStore s10;
  t.bytecode4 = build_index((const u64*)bytecode, needs & BYTECODE_PAIR ? n_bytecode : 0, 6, k4, 4, ch, s10);  // evm_err.cuh
  if (needs & BYTECODE_PAIR) t.bytecode4.tab = t.bytecode.tab;
  g_emu_tx = g_emu_block = nullptr;
  g_emu_n_tx = g_emu_n_block = 0;
  g_emu_tx_flags = g_emu_block_flags = nullptr;
  g_emu_wd = nullptr;
  g_emu_n_wd = 0;
  PosState p_bc, p_rw;
  if (g_emu_positional) {
    add_positional(t.bytecode, ZK_POS_RUNS, p_bc);
    add_positional(t.rw, ZK_POS_DENSE, p_rw);
  }
  g_emu_pos_ok = (pos_enabled(t.bytecode) ? 1 : 0) | (pos_enabled(t.rw) ? 2 : 0);
  t.resp_bitmap = fxc.bitmap.data();
  BlockStats stats;  // k_evm_block_stats, serially
  memset(&stats, 0, sizeof(stats));
  if (needs & BLOCK_STATS) {
    for (u64 r = 0; r < t.tx.tab.n_rows; r++) block_stats_tx_row(t.tx, (u32)r, &stats);
    for (u64 r = 0; r < t.wd.n_rows; r++) block_stats_wd_row(t.wd, (u32)r, &stats);
    if (pos_enabled(t.rw) && t.rw.pos_kind == ZK_POS_DENSE) stats.max_rws = (u32)t.rw.tab.n_rows;
    else
      for (u64 r = 0; r < t.rw.tab.n_rows; r++) stats.max_rws += first_of_kind_ix(t.rw_rwc, (u32)r) ? 1 : 0;
  }
  t.stats = &stats;
  ResultDev res;
  init_result(res, first_fail, fail_count, EV_N_CONSTRAINTS);
  Fr stack_pre[2];
  stack_key_pre(t.rw, stack_pre);
  // api.cu:evm_narrow — the narrow instances of the hot kernels run when the storage has these properties
  auto narrow_col = [](const unsigned char* base, const u64* off, const unsigned char* width, u32 c) {
    if (width[c] >= 1 && width[c] <= 8) return true;
    if (width[c] != 0) return false;
    const u64* cell = (const u64*)(base + off[c]);
    return (cell[1] | cell[2] | cell[3]) == 0;
  };
  bool narrow = g_emu_packed && both_positional(t);
  for (u32 c = 0; c < 13 && narrow; c++)
    if (c != 5 && c != 6) narrow = narrow_col(w.base, w.off, w.width, c);
  for (u32 c = 0; c < 5 && narrow; c++) narrow = narrow_col(t.rw.tab.base, t.rw.tab.off, t.rw.tab.width, c);
  for (u32 c = 0; c < 6 && narrow; c++) narrow = t.bytecode.tab.width[c] == kFromCode[c];
  g_emu_narrow_runs += narrow;
  for (u64 i = row_begin; i < row_end; i++) {
    StepCtx s{w, t, res, i, i + 1, row_base + i, true, t.resp_bitmap, 1u, stack_pre, nullptr, -1, narrow ? 1 : 0};
    verify_step(s, flags);
  }
  return 0;
}

extern "C" int emu_check_bytecode(const uint64_t* cols, uint64_t n_rows, const uint64_t* push, uint64_t n_push,
                                  const uint64_t* keccak, uint64_t n_keccak, const uint64_t r[4],
                                  uint64_t row_begin, uint64_t row_end, uint32_t flags,
                                  const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 pk[2] = {0, 1}, kk[5] = {0, 1, 2, 3, 4};
  IndexStore s1, s2;
  IndexDev push_ix = build_index((const u64*)push, n_push, 2, pk, 2, ch, s1);
  IndexDev kec_ix = build_index((const u64*)keccak, n_keccak, 5, kk, 5, ch, s2);
  PosState p_push;  // api.cu check_bytecode: the push table is served by position when it is dense from its first row
  if (g_emu_positional) add_positional(push_ix, ZK_POS_DENSE, p_push);
  g_emu_pos_ok = pos_enabled(push_ix) ? 1 : 0;
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)cols, n_rows, 12, nullptr);
  CheckRange rg{row_begin, row_end, 0, flags};
  ResultDev res;
  init_result(res, first_fail, fail_count, BC_N_CONSTRAINTS);
  const Fr r_mont = fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}});
  for (u64 i = row_begin; i < row_end; i++) check_bytecode_row<L_ANY>(w, rg, push_ix, nullptr, kec_ix, r_mont, res, i);
  return 0;
}

extern "C" int emu_check_copy(const uint64_t* rows, uint64_t n_rows, const uint8_t* row_flags, const uint64_t* rw,
                              uint64_t n_rw, const uint8_t* rw_flags, const uint64_t* bytecode, uint64_t n_bytecode,
                              const uint64_t* tx, uint64_t n_tx, const uint8_t* tx_flags, const uint64_t r[4],
                              uint64_t row_begin, uint64_t row_end, uint32_t flags, const uint64_t challenge[4],
                              uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 k5[5] = {0, 1, 2, 3, 4}, k3[3] = {0, 1, 2};
  IndexStore s1, s2, s3;
  CopyTables t;
  t.rw = build_index((const u64*)rw, n_rw, 14, k5, 5, ch, s1);
  t.rw.tab.flags = rw_flags;
  t.bytecode = build_index((const u64*)bytecode, n_bytecode, 6, k5, 5, ch, s2);
  t.tx = build_index((const u64*)tx, n_tx, 5, k3, 3, ch, s3);
  t.tx.tab.flags = tx_flags;
  PosState p_bc, p_rw;
  if (g_emu_positional) {
    add_positional(t.bytecode, ZK_POS_RUNS, p_bc);
    add_positional(t.rw, ZK_POS_DENSE, p_rw);
  }
  g_emu_pos_ok = (pos_enabled(t.bytecode) ? 1 : 0) | (pos_enabled(t.rw) ? 2 : 0);
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)rows, n_rows, 20, row_flags);
  CheckRange rg{row_begin, row_end, 0, flags};
  ResultDev res;
  init_result(res, first_fail, fail_count, CP_N_CONSTRAINTS);
  const Fr r_mont = fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}});
  for (u64 i = row_begin; i < row_end; i++) check_copy_rows<L_ANY>(w, rg, t, r_mont, res, i, true, 1u);
  return 0;
}

extern "C" int emu_check_state(const uint64_t* rows, uint64_t n_rows, const uint8_t* flags, const uint64_t* mpt,
                               uint64_t n_mpt, uint64_t row_begin, uint64_t row_end, uint32_t cflags,
                               const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 k12[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
  IndexStore s1;
  IndexDev ix = build_index((const u64*)mpt, n_mpt, 12, k12, 12, ch, s1);
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)rows, n_rows, 57, flags);
  CheckRange rg{row_begin, row_end, 0, cflags};
  ResultDev res;
  init_result(res, first_fail, fail_count, ST_N_CONSTRAINTS);
  for (u64 i = row_begin; i < row_end; i++) check_state_row_dev<L_ANY>(w, rg, ix, res, i, true, 1u);
  return 0;
}

extern "C" int emu_check_exp(const uint64_t* rows, uint64_t n_rows, uint64_t row_begin, uint64_t row_end, uint32_t cflags,
                             uint32_t* first_fail, uint64_t* fail_count) {
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)rows, n_rows, 21, nullptr);
  CheckRange rg{row_begin, row_end, 0, cflags};
  ResultDev res;
  init_result(res, first_fail, fail_count, XP_N_CONSTRAINTS);
  for (u64 i = row_begin; i < row_end; i++) check_exp_row<L_ANY>(w, rg, res, i);
  return 0;
}

extern "C" int emu_check_pi(const uint64_t* rows, uint64_t n_rows, const uint64_t* keccak, uint64_t n_keccak,
                            const uint64_t* gas, uint64_t n_gas, const uint64_t keccak_rand[4], const uint64_t byte_base[4],
                            const uint64_t circuit_len[4], uint64_t row_begin, uint64_t row_end, uint32_t cflags,
                            const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 kk[5] = {0, 1, 2, 3, 4}, gk[3] = {0, 1, 2};
  IndexStore s1, s2;
  IndexDev kix = build_index((const u64*)keccak, n_keccak, 5, kk, 5, ch, s1);
  IndexDev gix = build_index((const u64*)gas, n_gas, 3, gk, 3, ch, s2);
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)rows, n_rows, 28, nullptr);
  ResultDev res;
  init_result(res, first_fail, fail_count, PI_N_CONSTRAINTS);
  PiParams pp{fr_to_mont(Fr{{keccak_rand[0], keccak_rand[1], keccak_rand[2], keccak_rand[3]}}),
              fr_to_mont(Fr{{byte_base[0], byte_base[1], byte_base[2], byte_base[3]}}),
              Fr{{circuit_len[0], circuit_len[1], circuit_len[2], circuit_len[3]}}};
  CheckRange rg{row_begin, row_end, 0, cflags};
  for (u64 i = row_begin; i < row_end; i++) check_pi_row<L_ANY>(w, rg, kix, gix, pp, res, i);
  return 0;
}

// ---- witness assignment (assign.cu): the per-thread bodies run serially, the narrow result is widened to canonical
static size_t emu_up32(size_t x) { return (x + 31) / 32 * 32; }
static void widen(const unsigned char* base, const u64* off, const unsigned char* width, u32 n_cols, u64 n_rows, uint64_t* out) {
  for (u32 c = 0; c < n_cols; c++)
    for (u64 r = 0; r < n_rows; r++) {
      const Fr v = ld_col(base + off[c], width[c], r);
      memcpy(out + ((size_t)c * n_rows + r) * 4, v.l, 32);
    }
}
static std::vector<u64> emu_chunks(const u64* seg, u64 n) {
  std::vector<u64> c(n + 1, 0);
  for (u64 k = 0; k < n; k++) c[k + 1] = c[k] + (seg[k + 1] - seg[k] + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK;
  return c;
}
extern "C" int emu_assign_bytecode(uint32_t k, uint64_t n_contracts, const uint8_t* code, const uint8_t* bits,
                                   const uint64_t* offsets, const uint64_t* hashes, const uint64_t r[4], uint64_t* out) {
  const u64 n_rows = 1ull << k, total = offsets[n_contracts];
  std::vector<u64> chunks = emu_chunks((const u64*)offsets, n_contracts);
  BytecodeAssign a;
  a.s = SegHorner{code, (const u64*)offsets, chunks.data(), n_contracts, chunks[n_contracts], fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}})};
  a.bits = bits;
  a.hashes = (const u64*)hashes;
  a.n_rows = n_rows;
  a.n_table_rows = total + n_contracts;
  size_t bytes = 0;
  for (int c = 0; c < 12; c++) {
    a.off[c] = bytes;
    bytes += emu_up32((size_t)kBytecodeAssignWidths[c] * n_rows);
  }
  std::vector<unsigned char> buf(bytes + 32, 0xAB);
  a.base = buf.data();
  std::vector<Fr> cv(a.s.n_chunks + 1);
  for (u64 c = 0; c < a.s.n_chunks; c++) seg_local(a.s, cv.data(), c);
  for (u64 q = 0; q < n_contracts; q++) seg_carry(a.s, cv.data(), nullptr, q);
  for (u64 rr = 0; rr < n_rows; rr++) assign_bytecode_row(a, rr);
  for (u64 c = 0; c < a.s.n_chunks; c++) assign_bytecode_rlc(a, cv.data(), c);
  widen(buf.data(), a.off, kBytecodeAssignWidths, 12, n_rows, out);
  return 0;
}
extern "C" int emu_assign_state(uint64_t n_rows, const uint64_t* ops /* [15][n][4] */, uint64_t* out /* [57][n][4] */) {
  StateAssign a;
  a.base = (const unsigned char*)ops;
  a.off_addr = 4 * n_rows * 32, a.off_klo = 6 * n_rows * 32, a.off_khi = 7 * n_rows * 32;
  a.w_addr = a.w_klo = a.w_khi = 32;
  const size_t ls = emu_up32(2 * n_rows), bs = emu_up32(n_rows);
  std::vector<unsigned char> buf(10 * ls + 32 * bs + 32, 0xAB);
  a.limbs = buf.data();
  a.kbytes = buf.data() + 10 * ls;
  a.n_rows = n_rows, a.limb_stride = ls, a.byte_stride = bs;
  for (u64 r = 0; r < n_rows; r++) assign_state_row(a, r);
  for (int c = 0; c < 8; c++) memcpy(out + (size_t)c * n_rows * 4, ops + (size_t)c * n_rows * 4, n_rows * 32);
  for (int c = 8; c < 15; c++) memcpy(out + (size_t)(42 + c) * n_rows * 4, ops + (size_t)c * n_rows * 4, n_rows * 32);
  for (int q = 0; q < 10; q++)
    for (u64 r = 0; r < n_rows; r++) {
      const Fr v = ld_col(a.limbs + q * ls, 2, r);
      memcpy(out + ((size_t)(8 + q) * n_rows + r) * 4, v.l, 32);
    }
  for (int q = 0; q < 32; q++)
    for (u64 r = 0; r < n_rows; r++) {
      const Fr v = ld_col(a.kbytes + q * bs, 1, r);
      memcpy(out + ((size_t)(18 + q) * n_rows + r) * 4, v.l, 32);
    }
  return 0;
}
extern "C" int emu_assign_copy(uint64_t n_events, const uint64_t* events, const uint8_t* data, const uint8_t* bits,
                               const uint64_t r[4], uint64_t* out /* [20][n][4] */, uint8_t* flags_out) {
  std::vector<u64> seg(n_events + 1, 0);
  for (u64 e = 0; e < n_events; e++) seg[e + 1] = seg[e] + events[16 * e + 5];
  const u64 total = seg[n_events], n_rows = 2 * total;
  std::vector<u64> chunks = emu_chunks(seg.data(), n_events);
  CopyAssign a;
  a.s = SegHorner{data, seg.data(), chunks.data(), n_events, chunks[n_events], fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}})};
  a.ev = (const CopyEvent*)events;
  a.bits = bits;
  size_t bytes = 0;
  for (int c = 0; c < 20; c++) {
    a.off[c] = bytes;
    bytes += emu_up32((size_t)kCopyAssignWidths[c] * n_rows);
  }
  std::vector<unsigned char> buf(bytes + 32, 0xAB);
  a.base = buf.data();
  a.flags = flags_out;
  a.n_rows = n_rows;
  std::vector<Fr> cv(a.s.n_chunks + 1), tot(n_events + 1);
  for (u64 c = 0; c < a.s.n_chunks; c++) seg_local(a.s, cv.data(), c);
  for (u64 q = 0; q < n_events; q++) seg_carry(a.s, cv.data(), tot.data(), q);
  for (u64 c = 0; c < a.s.n_chunks; c++) assign_copy_chunk(a, cv.data(), tot.data(), c);
  widen(buf.data(), a.off, kCopyAssignWidths, 20, n_rows, out);
  return 0;
}

// 256-bit integer division of the MOD witness assignment (evm.cu:div256), for tests/test_emu_parity.py
extern "C" void emu_div256(const uint64_t* n, const uint64_t* d, uint64_t* q) {
  u64 qq[4];
  div256((const u64*)n, (const u64*)d, qq);
  for (int k = 0; k < 4; k++) q[k] = qq[k];
}

extern "C" int emu_check_tx(const uint64_t* rows, uint64_t n_rows, const uint8_t* flags, const uint64_t* keccak,
                            uint64_t n_keccak, const uint64_t r[4], uint64_t row_begin, uint64_t row_end,
                            const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 kk[5] = {0, 1, 2, 3, 4};
  IndexStore s1;
  IndexDev kix = build_index((const u64*)keccak, n_keccak, 5, kk, 5, ch, s1);
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)rows, n_rows, 14, flags);
  ResultDev res;
  init_result(res, first_fail, fail_count, TX_N_CONSTRAINTS);
  const Fr r_mont = fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}});
  CheckRange rg{row_begin, row_end, 0, 0};
  for (u64 i = row_begin; i < row_end; i++) check_tx_row(w, rg, kix, r_mont, res, i);
  return 0;
}

extern "C" int emu_check_sig(const uint64_t* rows, uint64_t n_rows, const uint8_t* flags, const uint64_t* keccak,
                             uint64_t n_keccak, const uint64_t r[4], uint64_t row_begin, uint64_t row_end,
                             const uint64_t challenge[4], uint32_t* first_fail, uint64_t* fail_count) {
  const Fr ch{{challenge[0], challenge[1], challenge[2], challenge[3]}};
  const u32 kk[5] = {0, 1, 2, 3, 4};
  IndexStore s1;
  IndexDev kix = build_index((const u64*)keccak, n_keccak, 5, kk, 5, ch, s1);
  Store ws;
  WitnessDev w = make_witness(ws, (const u64*)rows, n_rows, 21, flags);
  ResultDev res;
  init_result(res, first_fail, fail_count, SG_N_CONSTRAINTS);
  const Fr r_mont = fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}});
  CheckRange rg{row_begin, row_end, 0, 0};
  for (u64 i = row_begin; i < row_end; i++) check_sig_row(w, rg, kix, r_mont, res, i);
  return 0;
}

extern "C" int emu_n_evm_constraints() { return EV_N_CONSTRAINTS; }

// Keccak-256 of the device header (csrc/keccak.cuh), for tests/test_emu_parity.py
extern "C" void emu_keccak256(const uint8_t* msg, uint64_t len, uint8_t out[32]) {
  u64 d[4];
  keccak256(msg, len, d);
  memcpy(out, d, 32);
}
extern "C" void emu_keccak256_word(const uint8_t* msg, uint64_t len, uint64_t lo[2], uint64_t hi[2]) {
  u64 d[4], l[2], h[2];
  keccak256(msg, len, d);
  keccak_digest_to_word(d, l, h);
  lo[0] = l[0]; lo[1] = l[1]; hi[0] = h[0]; hi[1] = h[1];
}

// the keccak table's input_rlc as k_keccak256 folds it (128 chunks + pairwise tree), canonical result
extern "C" void emu_keccak_rlc(const uint8_t* msg, uint64_t len, const uint64_t r[4], uint64_t out[4]) {
  Fr r_mont = fr_to_mont(Fr{{r[0], r[1], r[2], r[3]}});
  Fr val[128], pw[128];
  const u64 per = (len + 127) / 128;
  for (u64 t = 0; t < 128; t++) {
    const u64 lo = std::min<u64>(len, t * per), hi = std::min<u64>(len, lo + per);
    rlc_chunk(msg, lo, hi, r_mont, val[t], pw[t]);
  }
  for (int stride = 1; stride < 128; stride <<= 1)
    for (int t = 0; t < 128; t += 2 * stride) rlc_combine(val[t], pw[t], val[t + stride], pw[t + stride]);
  for (int k = 0; k < 4; k++) out[k] = val[0].l[k];
}
