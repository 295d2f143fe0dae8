// tests/emu/zk_emu_state_mpt.cu — TEST INFRASTRUCTURE: runs zk_assign_state_circuit_mpt's builders of csrc/assign.cu
// (the host validation, and the same __host__ __device__ bodies k_state_mpt_insert / _first / _compact / _rows /
// _table and k_assign_state_derive call) serially on the CPU, so the rows and the MPT table can be diffed against the
// host mirror and the reference without a GPU.  The two count scans are a serial exclusive prefix here, stored in the
// two-level (block carry + chunk carry) form k_assign_pi_scan leaves.  Never shipped, never used by the product; built
// by tests/emu_state_mpt_lib.py with a host-only compilation.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../zkevm-specs_b200/csrc/assign.cu"

using namespace zk;

static size_t up32(size_t x) { return (x + 31) / 32 * 32; }

// the home slot of a key (address, field_tag, key lo, key hi: 4 limbs each) in the hash table of n operations
extern "C" uint64_t emu_state_mpt_home_slot(const uint64_t* key16, uint64_t n) {
  Fr k[4];
  for (int c = 0; c < 4; c++) memcpy(k[c].l, key16 + 4 * c, 32);
  return state_mpt_hash(k) & (state_mpt_slots(n) - 1);
}

// the count scan of k_assign_pi_scan / k_assign_pi_scan_top in its two-level form, computed serially
static void count_scan(const unsigned char* fl, u64 n, unsigned mask, std::vector<u64>& x, std::vector<u64>& top) {
  const u64 n_chunks = (n + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK;
  x.assign(n_chunks + 1, 0);
  top.assign(n_chunks / PI_SCAN_BLOCK_CHUNKS + 2, 0);
  u64 run = 0;
  for (u64 c = 0; c < n_chunks; c++) {
    if (c % PI_SCAN_BLOCK_CHUNKS == 0) top[c / PI_SCAN_BLOCK_CHUNKS] = run;
    x[c] = run - top[c / PI_SCAN_BLOCK_CHUNKS];
    for (u64 j = c * ZK_SEG_CHUNK; j < std::min<u64>(n, (c + 1) * ZK_SEG_CHUNK); j++) run += (fl[j] & mask) != 0;
  }
}

// zk_assign_state_circuit_mpt on the CPU over canonical operation cells ops[13][n][4] and flags[n] (may be NULL).
// Returns 0 with rows_out [57][n][4] and mpt_out [12][n][4] (the first *n_upd rows) filled; -1 where the host
// validation rejects the input; -2 (the mirror's KeyError) or -3 (its AssertionError) with *fail_op = the op.
extern "C" int emu_assign_state_mpt(uint64_t n, const uint64_t* ops, const uint8_t* flags, uint64_t* rows_out,
                                    uint64_t* mpt_out, uint64_t* n_upd, uint64_t* fail_op) {
  u64 off13[13];
  uint8_t w13[13];
  for (int c = 0; c < 13; c++) off13[c] = (u64)c * n * 32, w13[c] = 32;
  const size_t ops_bytes = 13 * n * 32;
  if (state_ops_error(n, 13, ops, ops_bytes ? ops_bytes : 32 * 13, (const uint64_t*)off13, w13)) return -1;
  const u64 cap = state_mpt_slots(n);
  std::vector<u64> slots(cap, SM_EMPTY);
  std::vector<u32> key_min(cap, ~0u), rank_at(cap, ~0u), slot_of(n + 1), upd_op(n + 1), mpt_op(n + 1);
  std::vector<unsigned char> fl(n + 1, 0);
  StateMpt a;
  a.base = (const unsigned char*)ops;
  for (int c = 0; c < 13; c++) a.off[c] = off13[c], a.w[c] = 32;
  a.flags = flags;
  a.n = n;
  a.slots = slots.data();
  a.key_min = key_min.data();
  a.rank_at = rank_at.data();
  a.mask = cap - 1;
  a.slot_of = slot_of.data();
  a.fl = fl.data();
  a.upd_op = upd_op.data();
  a.mpt_op = mpt_op.data();
  for (u64 i = 0; i < n; i++) state_mpt_insert(a, i);
  u64 fail = ~0ull, n_u = 0, n_m = 0;
  for (u64 i = 0; i < n; i++) {
    unsigned why;
    const unsigned f = state_mpt_first(a, i, &why);
    if (why && fail == ~0ull) fail = (i << 2) | why;
    n_u += (f >> 1) & 1;
    n_m += f & 1;
  }
  if (fail != ~0ull) {
    *fail_op = fail >> 2;
    return (fail & 3) == SM_FAIL_FIELD_TAG ? -2 : -3;
  }
  std::vector<u64> xu, tu, xm, tm;
  count_scan(fl.data(), n, 2, xu, tu);
  count_scan(fl.data(), n, 1, xm, tm);
  a.x_upd = xu.data(), a.top_upd = tu.data(), a.x_mpt = xm.data(), a.top_mpt = tm.data();
  a.n_upd = n_u, a.n_mpt = n_m;
  std::vector<u64> root(n + 1, 0xABABABABABABABABull);  // a row left unwritten shows
  a.root = (unsigned char*)root.data();
  const unsigned char tw[12] = {32, 1, 32, 32, 8, 1, 8, 1, 16, 16, 16, 16};  // the widths the device uses for 32-byte inputs
  size_t tbytes = 0;
  for (int c = 0; c < 12; c++) a.toff[c] = tbytes, a.twidth[c] = tw[c], tbytes += up32((size_t)tw[c] * n_u);
  std::vector<unsigned char> tbuf(tbytes + 32, 0xAB);
  a.tbase = tbuf.data();
  for (u64 i = 0; i < n; i++) state_mpt_compact(a, i);
  for (u64 k = 0; k < n; k++) state_mpt_row_root(a, k);
  for (u64 u = 0; u < n_u; u++) state_mpt_table_row(a, u);
  // op2row of every row
  std::vector<unsigned short> limbs(10 * (n + 1));
  std::vector<unsigned char> kbytes(32 * (n + 1));
  StateAssign s;
  s.base = (const unsigned char*)ops;
  s.off_addr = off13[SO_ADDR], s.off_klo = off13[SO_KLO], s.off_khi = off13[SO_KHI];
  s.w_addr = s.w_klo = s.w_khi = 32;
  s.limbs = (unsigned char*)limbs.data();
  s.kbytes = kbytes.data();
  s.n_rows = n, s.limb_stride = 2 * n, s.byte_stride = n;
  for (u64 r = 0; r < n; r++) assign_state_row(s, r);
  // the 57 cells: ops 0..7, limbs, key bytes, value / initial value, root lo, root hi (0), selector
  const int src13[57 - 42] = {0, 1, 2, 3, 4, 5, 6, 7, SO_VLO, SO_VHI, SO_ILO, SO_IHI, -1, -2, SO_SEL};
  for (u64 r = 0; r < n; r++) {
    for (int c = 0; c < 57; c++) {
      u64 v[4] = {0, 0, 0, 0};
      if (c >= 8 && c < 18) v[0] = limbs[(c - 8) * n + r];
      else if (c >= 18 && c < 50) v[0] = kbytes[(c - 18) * n + r];
      else {
        const int s13 = src13[c < 8 ? c : c - 42];
        if (s13 >= 0) memcpy(v, ops + ((size_t)s13 * n + r) * 4, 32);
        else if (s13 == -1) v[0] = root[r];
      }
      memcpy(rows_out + ((size_t)c * n + r) * 4, v, 32);
    }
  }
  for (int c = 0; c < 12; c++)
    for (u64 u = 0; u < n_u; u++) {
      const Fr v = ld_col(tbuf.data() + a.toff[c], a.twidth[c], u);
      memcpy(mpt_out + ((size_t)c * n_u + u) * 4, v.l, 32);
    }
  *n_upd = n_u;
  return 0;
}
