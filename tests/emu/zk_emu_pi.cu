// tests/emu/zk_emu_pi.cu — TEST INFRASTRUCTURE: runs the public-inputs builder of csrc/assign.cu (the same __host__
// __device__ bodies the k_assign_pi_* kernels call, and the host validation of zk_assign_pi_circuit) serially on the
// CPU, so the rows and the two tables can be diffed against the host mirror without a GPU.  The two scans, which the
// device runs as block-level scans, are run here as serial loops with the same chunk values, carries and layout.
// Never shipped, never used by the product; built by tests/emu_pi_lib.py with a host-only compilation.
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
// what k_assign_pi_scan + k_assign_pi_scan_top leave: x[c] carried into chunk c from its block, top[b] into block b
template <class S>
static void scan_serial(const S& s, std::vector<typename S::T>& x, std::vector<typename S::T>& top) {
  const u64 n_chunks = (s.n + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK, n_blocks = (n_chunks + PI_SCAN_BLOCK_CHUNKS - 1) / PI_SCAN_BLOCK_CHUNKS;
  x.assign(n_chunks, s.id());
  top.assign(n_blocks + 1, s.id());
  for (u64 b = 0; b < n_blocks; b++) {
    typename S::T carry = s.id();
    for (u64 c = b * PI_SCAN_BLOCK_CHUNKS; c < std::min(n_chunks, (b + 1) * PI_SCAN_BLOCK_CHUNKS); c++) {
      x[c] = carry;
      carry = S::op(carry, s.fold(c * ZK_SEG_CHUNK, std::min<u64>((c + 1) * ZK_SEG_CHUNK, s.n)));
    }
    top[b] = carry;
  }
  typename S::T carry = s.id();
  for (u64 b = 0; b < n_blocks; b++) {
    const typename S::T t = top[b];
    top[b] = carry;
    carry = S::op(carry, t);
  }
}

// fr_inv of a canonical cell (limbs in v[4]) into out[4]
extern "C" void emu_fr_inv(const uint64_t* v, uint64_t* out) {
  const Fr r = fr_inv(Fr{{v[0], v[1], v[2], v[3]}});
  memcpy(out, r.l, 32);
}

// zk_assign_pi_circuit on the CPU: out [28][n][4], keccak_out [5][2][4], gas_out [3][n_gas][4] with n_gas = 1 + the
// CallDataLength fields' sum, word_out [4] (the digest Word).  r_keccak / r_base: the two challenges, canonical.
// Returns -1 where the device call rejects the input, or if n_gas is not the table's row count.
extern "C" int emu_assign_pi(uint64_t max_txs, uint64_t max_cd, uint64_t max_wd, const uint8_t* raw, uint64_t n,
                             const uint64_t* r_keccak, const uint64_t* r_base, uint64_t* out, uint64_t* keccak_out,
                             uint64_t n_gas, uint64_t* gas_out, uint64_t* word_out) {
  if (pi_shape_error(max_txs, max_cd, max_wd, n)) return -1;
  std::vector<u64> cd_off(max_txs + 1);
  if (pi_calldata_offsets(max_txs, max_cd, raw, cd_off.data())) return -1;
  const u64 n_inv = std::max<u64>(256, max_txs + 1);
  std::vector<unsigned char> seq(n);
  std::vector<Fr> inv(n_inv);
  std::vector<RlcPair> kx, ktop;
  std::vector<u64> gx, gtop;
  u64 dig[8];
  PiAssign a;
  a.F = raw;
  a.seq = seq.data();
  a.cd_off = cd_off.data();
  a.inv = inv.data();
  a.dig = dig;
  a.n = n, a.max_txs = max_txs, a.max_cd = max_cd, a.max_wd = max_wd, a.n_inv = n_inv;
  a.rand_mont = fr_to_mont(Fr{{r_keccak[0], r_keccak[1], r_keccak[2], r_keccak[3]}});
  a.base_mont = fr_to_mont(Fr{{r_base[0], r_base[1], r_base[2], r_base[3]}});
  const size_t bytes = layout(kPiAssignWidths, 28, n, a.off), kbytes = layout(kPiKeccakWidths, 5, 2, a.koff);
  if (n_gas != 1 + cd_off[max_txs]) return -1;
  const size_t gbytes = layout(kPiGasWidths, 3, n_gas, a.goff);
  // 0xAB: a cell left unwritten shows
  std::vector<unsigned char> buf(bytes + 32, 0xAB), kbuf(kbytes + 32, 0xAB), gbuf(gbytes + 32, 0xAB);
  a.base = buf.data();
  a.kbase = kbuf.data();
  a.gbase = gbuf.data();
  for (u64 r = 0; r < n; r++) assign_pi_seq(a, r);
  for (u64 k = 0; k < n_inv; k++) assign_pi_inv(a, k);
  keccak256(a.seq, n, a.dig);
  scan_serial(PiKrlcScan{a.seq, n, a.rand_mont}, kx, ktop);
  a.kx = kx.data();
  a.ktop = ktop.data();
  for (u64 c = 0; c < (n + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK; c++) assign_pi_krlc(a, c);
  scan_serial(PiGasScan{raw + PI_TX0 + PI_SLOT_BYTES * max_txs, max_cd}, gx, gtop);
  a.gx = gx.data();
  a.gtop = gtop.data();
  for (u64 c = 0; c < (max_cd + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK; c++) assign_pi_calldata(a, c);
  for (u64 r = 0; r < n; r++) assign_pi_row(a, r);
  assign_pi_finish(a);
  widen(buf.data(), a.off, kPiAssignWidths, 28, n, out);
  widen(kbuf.data(), a.koff, kPiKeccakWidths, 5, 2, keccak_out);
  widen(gbuf.data(), a.goff, kPiGasWidths, 3, n_gas, gas_out);
  memcpy(word_out, dig + 4, 32);
  return 0;
}
