// tests/emu/zk_emu_tables.cu — TEST INFRASTRUCTURE: runs the tx-table and copy-table builders of csrc/assign.cu (the
// same __host__ __device__ bodies k_assign_tx_zeros / k_assign_tx_rows and k_copy_table_count / k_copy_table_write call,
// and the host validation of zk_assign_tx_table) serially on the CPU, so the tables can be diffed against the host
// mirror without a GPU.  The zero-byte count, which the device adds up with warp ballots, is a serial loop here over
// the same byte-to-tx search.  Never shipped, never used by the product; built by tests/emu_tables_lib.py with a
// host-only compilation.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../zkevm-specs_b200/csrc/assign.cu"

using namespace zk;

static size_t up32(size_t x) { return (x + 31) / 32 * 32; }
// narrow columns -> canonical uint64[n_cols][n_rows][4]
static void widen(const unsigned char* base, const u64* off, const unsigned char* width, u32 n_cols, u64 n_rows, uint64_t* out) {
  for (u32 c = 0; c < n_cols; c++)
    for (u64 r = 0; r < n_rows; r++) {
      const Fr v = ld_col(base + off[c], width[c], r);
      memcpy(out + ((size_t)c * n_rows + r) * 4, v.l, 32);
    }
}
static size_t layout(const unsigned char* widths, u32 n_cols, u64 n_rows, u64* off) {
  size_t bytes = 0;
  for (u32 c = 0; c < n_cols; c++) {
    off[c] = bytes;
    bytes += up32((size_t)widths[c] * n_rows);
  }
  return bytes;
}

// the row count zk_assign_tx_table would give, or -1 where it rejects the input; widths_out [5] (may be NULL)
extern "C" int64_t emu_tx_table_rows(uint64_t n_txs, const uint64_t* rec, const uint64_t* cd_off, uint8_t* widths_out) {
  u64 n_rows;
  unsigned char w[5];
  if (tx_table_plan(n_txs, (const u64*)rec, (const u64*)cd_off, &n_rows, w)) return -1;
  if (widths_out) memcpy(widths_out, w, 5);
  return (int64_t)n_rows;
}

// zk_assign_tx_table on the CPU: out [5][n_rows][4], flags_out [n_rows]; -1 where the device call rejects the input or
// n_rows is not the table's row count
extern "C" int emu_assign_tx_table(uint64_t n_txs, const uint64_t* rec, const uint8_t* cd, const uint64_t* cd_off,
                                   uint64_t n_rows, uint64_t* out, uint8_t* flags_out) {
  u64 want;
  TxTableAssign a;
  if (tx_table_plan(n_txs, (const u64*)rec, (const u64*)cd_off, &want, a.width) || want != n_rows) return -1;
  std::vector<unsigned long long> zeros(n_txs, 0);
  a.rec = (const u64*)rec;
  a.cd = cd;
  a.cd_off = (const u64*)cd_off;
  a.zeros = zeros.data();
  a.n_txs = n_txs, a.n_rows = n_rows, a.n_cd = n_txs ? cd_off[n_txs] : 0;
  const size_t bytes = layout(a.width, 5, n_rows, a.off);
  std::vector<unsigned char> buf(bytes + 32, 0xAB), flags(n_rows + 1, 0xAB);  // 0xAB: a cell left unwritten shows
  a.base = buf.data();
  a.flags = flags.data();
  for (u64 j = 0; j < a.n_cd; j++)
    if (cd[j] == 0) zeros[tx_of_byte(a, j)]++;
  for (u64 r = 0; r < n_rows; r++) assign_tx_row(a, r);
  widen(buf.data(), a.off, a.width, 5, n_rows, out);
  memcpy(flags_out, flags.data(), n_rows);
  return 0;
}

// zk_assign_copy_table on the CPU over a canonical copy circuit [20][n][4]: returns the table's row count with out
// [14][n_out_max][4] filled (in circuit order), -2 for "Not enough rows in copy circuit", -3 for "Invalid copy circuit",
// -1 if the table has more than n_out_max rows
extern "C" int64_t emu_assign_copy_table(uint64_t n, const uint64_t* circuit, uint64_t n_out_max, uint64_t* out) {
  CopyTableAssign a;
  a.w.base = (const unsigned char*)circuit;
  a.w.n_rows = n;
  a.w.flags = nullptr;
  for (u32 c = 0; c < ZK_MAX_COLS; c++) a.w.off[c] = (u64)c * n * 32, a.w.width[c] = 32;
  u64 fail = ~0ull, count = 0;
  for (u64 i = 0; i < n; i++)
    if (copy_row_is_first(a, i)) {
      count++;
      if (copy_row_fails(a, i)) fail = std::min(fail, i);
    }
  if (fail != ~0ull) return fail + 1 == n ? -2 : -3;
  if (count > n_out_max) return -1;
  for (int c = 0; c < 14; c++) a.width[c] = c == 0 ? 1 : 32;
  const size_t bytes = layout(a.width, 14, count, a.off);
  std::vector<unsigned char> buf(bytes + 32, 0xAB);
  a.base = buf.data();
  u64 pos = 0;
  for (u64 i = 0; i < n; i++)
    if (copy_row_is_first(a, i)) copy_table_row(a, i, pos++);
  widen(buf.data(), a.off, a.width, 14, count, out);
  return (int64_t)count;
}
