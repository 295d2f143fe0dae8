// tests/emu/zk_emu_exp.cu — TEST INFRASTRUCTURE: runs the exp-circuit builder of csrc/assign.cu (the same
// __host__ __device__ bodies k_assign_exp_chain and k_assign_exp_rows call) serially on the CPU, so the rows and the exp
// table can be diffed against the host mirror without a GPU.  Never shipped, never used by the product; built by
// tests/emu_exp_lib.py with a host-only compilation.
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

// ExpCircuit.add_event per event + padding to n_rows_min, and its exp table: the caller sizes out [21][n_rows][4] and
// table_out [11][n_table][4] (returns -1 if those sizes are not the ones the bodies produce)
extern "C" int emu_assign_exp(uint64_t n_events, const uint64_t* events, uint64_t n_rows_min, uint64_t n_rows, uint64_t n_table,
                              uint64_t* out, uint64_t* table_out) {
  std::vector<u64> row_off(n_events + 1, 0);
  for (u64 e = 0; e < n_events; e++) row_off[e + 1] = row_off[e] + exp_event_rows((const u64*)events + 12 * e + 4);
  const u64 n_used = row_off[n_events];
  if (n_rows != std::max<u64>(n_used, n_rows_min) || n_table != n_used + (n_rows > n_used ? 1 : 0)) return -1;
  ExpAssign a;
  a.ev = (const u64*)events;
  a.row_off = row_off.data();
  a.n_events = n_events, a.n_used = n_used, a.n_rows = n_rows;
  size_t bytes = 0, tbytes = 0;
  for (int c = 0; c < 21; c++) {
    a.off[c] = bytes;
    bytes += up32((size_t)kExpAssignWidths[c] * n_rows);
  }
  for (int c = 0; c < 11; c++) {
    a.toff[c] = tbytes;
    tbytes += up32((size_t)kExpTableWidths[c] * n_table);
  }
  std::vector<unsigned char> buf(bytes + 32, 0xAB), tbuf(tbytes + 32, 0xAB);  // 0xAB: a cell left unwritten shows
  a.base = buf.data();
  a.tbase = tbuf.data();
  for (u64 k = 0; k < n_events; k++) assign_exp_chain(a, k);
  for (u64 r = 0; r < n_rows; r++) assign_exp_row(a, r);
  widen(buf.data(), a.off, kExpAssignWidths, 21, n_rows, out);
  widen(tbuf.data(), a.toff, kExpTableWidths, 11, n_table, table_out);
  return 0;
}
