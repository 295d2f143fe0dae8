// assign.cu — witness assignment on the device (SURVEY.md 8(f)-3): the row builders the reference runs as
// Python object loops, fed from the compact data they expand.
//
//   assign_bytecode_circuit  src/zkevm_specs/bytecode_circuit.py:104-167   raw code bytes -> 12-cell rows
//   op2row / assign_state_circuit  src/zkevm_specs/state_circuit.py:827-889  15 operation cells -> 57-cell rows
//                            + _mock_mpt_updates (state_circuit.py:903-933): 13 operation cells -> the same rows with
//                            their roots, and the MPT table
//   CopyCircuit.copy         src/zkevm_specs/evm_circuit/typing.py:1010-1147 copy events + bytes -> 20-cell rows
//   ExpCircuit.add_event     src/zkevm_specs/evm_circuit/typing.py:880-994  (base, exponent, id) -> 21-cell rows
//                            + the exp table (Tables._convert_exp_circuit_to_table, table.py:654-671)
//   public_data2witness      src/zkevm_specs/pi_circuit.py:839-1073  raw public-input bytes -> 28-cell rows, one per byte
//                            + the keccak table and the calldata gas table its lookups read
//
// The two sequential pieces — value_rlc of a contract and rlc_acc of a copy event, both Horner chains
// acc = acc * r + byte — run as a chunked segmented scan: one thread folds a 32-byte chunk
// (k_seg_local), one thread per segment chains the chunk values with r^32 (k_seg_carry), then one
// thread per chunk replays its bytes from the carried-in value and writes the running value of each row.
// Everything else of a row is a closed form of (segment, position).  Rows are written as narrow columns
// (fr.cuh:ld_col widths), so a check after an assignment reads 80-150 B per row instead of 384-1,824.
// Included by api.cu (it uses the context).
#include "circuit.cuh"
#include "keccak.cuh"
#include "words.cuh"

namespace zk {

#define ZK_SEG_CHUNK 32
struct SegHorner {
  const unsigned char* bytes;  // the segments' bytes, concatenated
  const u64* seg_off;          // [n_seg + 1] byte offsets
  const u64* chunk_off;        // [n_seg + 1] first chunk of each segment (ceil(len / 32) chunks each)
  u64 n_seg, n_chunks;
  Fr r_mont;  // the challenge in Montgomery form
};

ZK_HD u64 seg_of_chunk(const SegHorner& s, u64 c) {  // the largest k with chunk_off[k] <= c
  u64 lo = 0, hi = s.n_seg;
  while (hi - lo > 1) {
    const u64 mid = (lo + hi) >> 1;
    if (s.chunk_off[mid] <= c) lo = mid;
    else hi = mid;
  }
  return lo;
}
ZK_HD void st_narrow(unsigned char* col, u32 width, u64 row, u64 v) {
  if (width == 1) col[row] = (unsigned char)v;
  else if (width == 2) ((unsigned short*)col)[row] = (unsigned short)v;
  else if (width == 4) ((u32*)col)[row] = (u32)v;
  else ((u64*)col)[row] = v;
}
ZK_HD void st_u128(unsigned char* col, u64 row, u64 lo, u64 hi) {
  ((u64*)col)[2 * row] = lo;
  ((u64*)col)[2 * row + 1] = hi;
}
ZK_HD void st_fr(unsigned char* col, u64 row, const Fr& v) {
  u64* p = (u64*)col + 4 * row;
  p[0] = v.l[0];
  p[1] = v.l[1];
  p[2] = v.l[2];
  p[3] = v.l[3];
}

ZK_HD u64 zk_min64(u64 a, u64 b) { return a < b ? a : b; }
// the per-thread bodies are __host__ __device__ so that tests/emu can run them serially on the CPU
ZK_HD void seg_local(const SegHorner& s, Fr* chunk_val, u64 c) {
  const u64 k = seg_of_chunk(s, c);
  const u64 b0 = s.seg_off[k] + (c - s.chunk_off[k]) * ZK_SEG_CHUNK;
  const u64 b1 = zk_min64(b0 + ZK_SEG_CHUNK, s.seg_off[k + 1]);
  Fr acc = fr_u64(0);
  for (u64 j = b0; j < b1; j++) acc = fr_add(fr_montmul(acc, s.r_mont), fr_u64(s.bytes[j]));
  chunk_val[c] = acc;
}
// chunk_val[c] becomes the value carried INTO chunk c; seg_total[k] the Horner value of the whole segment
ZK_HD void seg_carry(const SegHorner& s, Fr* chunk_val, Fr* seg_total, u64 k) {
  Fr rp = s.r_mont;  // r^32, Montgomery form
  for (int q = 0; q < 5; q++) rp = fr_montmul(rp, rp);
  const u64 c0 = s.chunk_off[k], c1 = s.chunk_off[k + 1], len = s.seg_off[k + 1] - s.seg_off[k];
  Fr carry = fr_u64(0);
  for (u64 c = c0; c < c1; c++) {
    const Fr v = chunk_val[c];
    chunk_val[c] = carry;
    const u64 left = len - (c - c0) * ZK_SEG_CHUNK;
    if (left >= ZK_SEG_CHUNK) {
      carry = fr_montmul(carry, rp);
    } else {
      for (u64 q = 0; q < left; q++) carry = fr_montmul(carry, s.r_mont);
    }
    carry = fr_add(carry, v);
  }
  if (seg_total) seg_total[k] = carry;
}

// ---------------------------------------------------------------- bytecode circuit
struct BytecodeAssign {
  SegHorner s;              // segments = contracts
  const unsigned char* bits;  // is_code bit per code byte (Bytecode.table_assignments, typing.py:390-427)
  const u64* hashes;        // [n_seg][4]: code hash lo (2 limbs), hi (2 limbs)
  u64 n_rows;               // 2^k
  u64 n_table_rows;         // total bytes + contracts (what the table would hold), may exceed n_rows
  unsigned char* base;
  u64 off[12];
};
static const unsigned char kBytecodeAssignWidths[12] = {1, 1, 16, 16, 1, 4, 4, 1, 1, 32, 4, 1};
enum { A_QFIRST, A_QLAST, A_HASH_LO, A_HASH_HI, A_TAG, A_INDEX, A_VALUE, A_ISCODE, A_PDL, A_RLC, A_LEN, A_PDS };

// value_rlc of the Byte rows: replay each chunk from its carried-in value
ZK_HD void assign_bytecode_rlc(const BytecodeAssign& a, const Fr* chunk_val, u64 c) {
  const SegHorner& s = a.s;
  const u64 k = seg_of_chunk(s, c);
  const u64 b0 = s.seg_off[k] + (c - s.chunk_off[k]) * ZK_SEG_CHUNK;
  const u64 b1 = zk_min64(b0 + ZK_SEG_CHUNK, s.seg_off[k + 1]);
  Fr acc = chunk_val[c];
  for (u64 j = b0; j < b1; j++) {
    acc = fr_add(fr_montmul(acc, s.r_mont), fr_u64(s.bytes[j]));
    const u64 row = j + k + 1;  // k Header rows of earlier contracts + this one's
    if (row < a.n_rows) st_fr(a.base + a.off[A_RLC], row, acc);
  }
}
// every other cell (and value_rlc = 0 of Header / padding rows): one thread per row
ZK_HD void assign_bytecode_row(const BytecodeAssign& a, u64 r) {
  const SegHorner& s = a.s;
  {
    u64 hl0, hl1, hh0, hh1, tag = 1, index = 0, value = 0, is_code = 0, pdl = 0, len = 0, pds = 0;
    bool byte_row = false;
    if (r < a.n_table_rows) {
      u64 lo = 0, hi = s.n_seg;  // largest k with seg_off[k] + k <= r
      while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if (s.seg_off[mid] + mid <= r) lo = mid;
        else hi = mid;
      }
      const u64 k = lo, start = s.seg_off[k], local = r - (start + k);
      len = s.seg_off[k + 1] - start;
      hl0 = a.hashes[4 * k], hl1 = a.hashes[4 * k + 1], hh0 = a.hashes[4 * k + 2], hh1 = a.hashes[4 * k + 3];
      if (local == 0) {
        value = len;
      } else {
        byte_row = true;
        const u64 j = start + local - 1;
        tag = 2;
        index = local - 1;
        value = s.bytes[j];
        is_code = (a.bits[j >> 3] >> (j & 7)) & 1;
        pds = (value >= 0x60 && value <= 0x7f) ? value - 0x5f : 0;  // get_push_size
        if (!is_code) {  // data byte of the PUSH at the nearest code byte p before it: left = size - (j - p - 1)
          u64 p = j;
          while (p > start) {
            p--;
            if ((a.bits[p >> 3] >> (p & 7)) & 1) break;
          }
          const u64 pv = s.bytes[p];
          const u64 psz = (pv >= 0x60 && pv <= 0x7f) ? pv - 0x5f : 0;
          pdl = psz - (j - p - 1);
        }
      }
    } else {  // padding: (EMPTY_HASH, Header, 0 ...)   bytecode_circuit.py:150-165
      hl0 = 0x7bfad8045d85a470ull, hl1 = 0xe500b653ca82273bull, hh0 = 0x927e7db2dcc703c0ull, hh1 = 0xc5d2460186f7233cull;
    }
    a.base[a.off[A_QFIRST] + r] = r == 0;
    a.base[a.off[A_QLAST] + r] = r == a.n_rows - 1;
    st_u128(a.base + a.off[A_HASH_LO], r, hl0, hl1);
    st_u128(a.base + a.off[A_HASH_HI], r, hh0, hh1);
    a.base[a.off[A_TAG] + r] = (unsigned char)tag;
    ((u32*)(a.base + a.off[A_INDEX]))[r] = (u32)index;
    ((u32*)(a.base + a.off[A_VALUE]))[r] = (u32)value;
    a.base[a.off[A_ISCODE] + r] = (unsigned char)is_code;
    a.base[a.off[A_PDL] + r] = (unsigned char)pdl;
    ((u32*)(a.base + a.off[A_LEN]))[r] = (u32)len;
    a.base[a.off[A_PDS] + r] = (unsigned char)pds;
    if (!byte_row) st_fr(a.base + a.off[A_RLC], r, fr_u64(0));
  }
}

// ---------------------------------------------------------------- state circuit
// op2row: address -> 10 little-endian 16-bit limbs (cells 8..17), storage key -> 32 little-endian bytes
// (cells 18..49); the other 15 cells of a row are the operation's own and stay where they were uploaded.
struct StateAssign {
  const unsigned char* base;  // the uploaded operation columns
  u64 off_addr, off_klo, off_khi;
  unsigned char w_addr, w_klo, w_khi;
  unsigned char* limbs;  // [10] columns of u16
  unsigned char* kbytes;  // [32] columns of u8
  u64 n_rows, limb_stride, byte_stride;
};
ZK_HD void assign_state_row(const StateAssign& a, u64 r) {
  {
    const Fr addr = ld_col(a.base + a.off_addr, a.w_addr, r);
    const Fr klo = ld_col(a.base + a.off_klo, a.w_klo, r), khi = ld_col(a.base + a.off_khi, a.w_khi, r);
#pragma unroll
    for (int q = 0; q < 10; q++)
      ((unsigned short*)(a.limbs + q * a.limb_stride))[r] = (unsigned short)(addr.l[q >> 2] >> (16 * (q & 3)));
#pragma unroll
    for (int q = 0; q < 32; q++) {
      const Fr& h = q < 16 ? klo : khi;
      (a.kbytes + q * a.byte_stride)[r] = (unsigned char)(h.l[(q & 15) >> 3] >> (8 * (q & 7)));
    }
  }
}

// ---------------------------------------------------------------- copy circuit
// one event = CopyCircuit.copy(r, rw_dict, src_id, src_tag, dst_id, dst_tag, src_addr, src_addr_end, dst_addr,
// copy_length, src_data, log_id): 2 rows per byte (read row, write row)
struct CopyEvent {  // 16 u64 per event, host layout of zk_assign_copy_circuit
  u64 src_tag, dst_tag /* low byte: CopyDataTypeTag; bit 8: the id is a Word */, src_addr, src_addr_end, dst_addr, length, log_id, rw_counter;
  u64 src_id[4];  // lo (2 limbs), hi (2 limbs)
  u64 dst_id[4];
};
struct CopyAssign {
  SegHorner s;  // segments = events, bytes = the copied values (0 where the source is out of bounds)
  const CopyEvent* ev;
  const unsigned char* bits;  // is_code bit per byte (events that touch bytecode), may be null
  unsigned char* base;
  unsigned char* flags;  // [n_rows] row flags: bit 0 = the id cell is a Word
  u64 off[20];
  u64 n_rows;
};
static const unsigned char kCopyAssignWidths[20] = {1, 1, 1, 16, 16, 1, 8, 8, 8, 32, 32, 1, 1, 8, 8, 1, 1, 1, 1, 1};
#define CPT_BYTECODE 1
#define CPT_MEMORY 2
#define CPT_TXCALLDATA 3
#define CPT_TXLOG 4
#define CPT_RLCACC 5
#define TXLOG_DATA 3

ZK_HD void assign_copy_chunk(const CopyAssign& a, const Fr* chunk_val, const Fr* seg_total, u64 c) {
  const SegHorner& s = a.s;
  const u64 k = seg_of_chunk(s, c);
  CopyEvent e = a.ev[k];
  const unsigned char src_word = (e.src_tag >> 8) & 1, dst_word = (e.dst_tag >> 8) & 1;  // the id is a Word (row flag bit 0)
  e.src_tag &= 0xFF;
  e.dst_tag &= 0xFF;
  const u64 b0 = s.seg_off[k] + (c - s.chunk_off[k]) * ZK_SEG_CHUNK;
  const u64 b1 = zk_min64(b0 + ZK_SEG_CHUNK, s.seg_off[k + 1]);
  const bool to_rlc = e.dst_tag == CPT_RLCACC, src_mem = e.src_tag == CPT_MEMORY;
  const bool dst_rw = e.dst_tag == CPT_MEMORY || e.dst_tag == CPT_TXLOG;
  const bool has_code = e.src_tag == CPT_BYTECODE || e.dst_tag == CPT_BYTECODE;
  const u64 n_real = e.src_addr_end > e.src_addr ? zk_min64(e.length, e.src_addr_end - e.src_addr) : 0;
  const u64 rw_total = (src_mem ? n_real : 0) + (dst_rw ? e.length : 0);
  const Fr total = to_rlc ? seg_total[k] : fr_u64(0);
  const u64 dst_shift = e.dst_tag == CPT_TXLOG ? ((u64)TXLOG_DATA << 32) + (e.log_id << 48) : 0;
  Fr acc = chunk_val[c];
  unsigned char* B = a.base;
  for (u64 j = b0; j < b1; j++) {
    const u64 i = j - s.seg_off[k];
    const bool pad = i >= n_real;
    const u64 value = pad ? 0 : s.bytes[j];
    const u64 is_code = (has_code && !pad && a.bits) ? (a.bits[j >> 3] >> (j & 7)) & 1 : 0;
    acc = fr_add(fr_montmul(acc, s.r_mont), fr_u64(value));
    const u64 reads_before = src_mem ? zk_min64(i, n_real) : 0, writes_before = dst_rw ? i : 0;
    const u64 rd = 2 * j, wr = 2 * j + 1;
    // read row (typing.py:1043-1058)
    u64 rwc = reads_before + writes_before;
    B[a.off[0] + rd] = 1;
    B[a.off[1] + rd] = i == 0;
    B[a.off[2] + rd] = 0;
    st_u128(B + a.off[3], rd, e.src_id[0], e.src_id[1]);
    st_u128(B + a.off[4], rd, e.src_id[2], e.src_id[3]);
    B[a.off[5] + rd] = (unsigned char)e.src_tag;
    ((u64*)(B + a.off[6]))[rd] = e.src_addr + i;
    ((u64*)(B + a.off[7]))[rd] = e.src_addr_end;
    ((u64*)(B + a.off[8]))[rd] = e.length - i;
    st_fr(B + a.off[9], rd, fr_u64(value));
    st_fr(B + a.off[10], rd, total);
    B[a.off[11] + rd] = (unsigned char)is_code;
    B[a.off[12] + rd] = pad;
    ((u64*)(B + a.off[13]))[rd] = e.rw_counter + rwc;
    ((u64*)(B + a.off[14]))[rd] = rw_total - rwc;
    B[a.off[15] + rd] = e.src_tag == CPT_MEMORY;
    B[a.off[16] + rd] = e.src_tag == CPT_BYTECODE;
    B[a.off[17] + rd] = e.src_tag == CPT_TXCALLDATA;
    B[a.off[18] + rd] = e.src_tag == CPT_TXLOG;
    B[a.off[19] + rd] = e.src_tag == CPT_RLCACC;
    a.flags[rd] = src_word;
    // write row (typing.py:1060-1076)
    rwc = (src_mem ? zk_min64(i + 1, n_real) : 0) + writes_before;
    B[a.off[0] + wr] = 0;
    B[a.off[1] + wr] = 0;
    B[a.off[2] + wr] = i == e.length - 1;
    st_u128(B + a.off[3], wr, e.dst_id[0], e.dst_id[1]);
    st_u128(B + a.off[4], wr, e.dst_id[2], e.dst_id[3]);
    B[a.off[5] + wr] = (unsigned char)e.dst_tag;
    ((u64*)(B + a.off[6]))[wr] = e.dst_addr + i + dst_shift;
    ((u64*)(B + a.off[7]))[wr] = 0;
    ((u64*)(B + a.off[8]))[wr] = 0;
    st_fr(B + a.off[9], wr, to_rlc ? acc : fr_u64(value));
    st_fr(B + a.off[10], wr, total);
    B[a.off[11] + wr] = (unsigned char)is_code;
    B[a.off[12] + wr] = 0;
    ((u64*)(B + a.off[13]))[wr] = e.rw_counter + rwc;
    ((u64*)(B + a.off[14]))[wr] = rw_total - rwc;
    B[a.off[15] + wr] = e.dst_tag == CPT_MEMORY;
    B[a.off[16] + wr] = e.dst_tag == CPT_BYTECODE;
    B[a.off[17] + wr] = e.dst_tag == CPT_TXCALLDATA;
    B[a.off[18] + wr] = e.dst_tag == CPT_TXLOG;
    B[a.off[19] + wr] = e.dst_tag == CPT_RLCACC;
    a.flags[wr] = dst_word;
  }
}

// ---------------------------------------------------------------- exponentiation circuit
// one event = ExpCircuit.add_event(base, exponent, identifier): n = (bitlen(x) - 1) + (popcount(x) - 1) rows for an
// exponent x >= 2 (none for 0 and 1), row 0 the final product.  Counted from the top, e_0 = x and e_{k+1} = e_k - 1
// (e_k odd) or e_k / 2; d_k = base^e_k mod 2^256, a_k = d_{k+1} (a_{n-1} = base), b_k = base (e_k odd) or a_k.
// Only d is a chain: k_assign_exp_chain runs square-and-multiply per event and writes d of each row it produces;
// every other cell is a closed form of (x, k, base, identifier, d_k, d_{k+1}).  Walking x from its least significant
// bit, bit j < bitlen(x) - 1 contributes an odd row e = x >> j when it is set, then an even row e = (x >> j) & ~1, so
// j + popcount(x mod 2^j) rows precede bit j's rows.
struct ExpAssign {
  const u64* ev;       // [n_events][12]: base, exponent, identifier (4 little-endian limbs each)
  const u64* row_off;  // [n_events + 1] first row of each event
  u64 n_events, n_used, n_rows;  // event rows, circuit rows (n_used + fill_dummy_events padding)
  unsigned char* base;  // the circuit's narrow columns
  u64 off[21];
  unsigned char* tbase;  // the exp table's narrow columns: n_used rows, + the padding row once if n_rows > n_used
  u64 toff[11];
};
static const unsigned char kExpAssignWidths[21] = {1, 1, 32, 1, 16, 16, 16, 16, 16, 16, 16, 16, 16, 16, 1, 1, 16, 16, 16, 16, 1};
static const unsigned char kExpTableWidths[11] = {1, 32, 1, 8, 8, 8, 8, 16, 16, 16, 16};
enum { E_USABLE, E_STEP, E_ID, E_LAST, E_BASE, E_EXPO = 6, E_EXPN = 8, E_A = 10, E_B = 12, E_C = 14, E_D = 16, E_Q = 18, E_R = 20 };

ZK_HD int zk_popc64(u64 x) {
#ifdef __CUDA_ARCH__
  return __popcll(x);
#else
  return __builtin_popcountll(x);
#endif
}
ZK_HD int zk_bitlen64(u64 x) {
#ifdef __CUDA_ARCH__
  return 64 - __clzll((long long)x);
#else
  return x ? 64 - __builtin_clzll(x) : 0;
#endif
}
ZK_HD int exp_bitlen(const u64 x[4]) {
  return x[3] ? 192 + zk_bitlen64(x[3]) : x[2] ? 128 + zk_bitlen64(x[2]) : x[1] ? 64 + zk_bitlen64(x[1]) : zk_bitlen64(x[0]);
}
// rows of one event (the host sizes the circuit with it)
ZK_HD u64 exp_event_rows(const u64 x[4]) {
  const int len = exp_bitlen(x);
  if (len < 2) return 0;
  return (u64)(len - 1) + (u64)(zk_popc64(x[0]) + zk_popc64(x[1]) + zk_popc64(x[2]) + zk_popc64(x[3]) - 1);
}
// limb i of x (0 beyond the top), without indexing x by a run-time value (which would put it in local memory)
ZK_HD u64 limb_at(const u64 x[4], int i) { return i == 0 ? x[0] : i == 1 ? x[1] : i == 2 ? x[2] : i == 3 ? x[3] : 0; }
// popcount(x mod 2^j), 0 <= j <= 256
ZK_HD int popc_below(const u64 x[4], int j) {
  int n = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int b = j - 64 * i;
    const u64 m = b >= 64 ? ~0ull : (b <= 0 ? 0ull : (1ull << b) - 1);
    n += zk_popc64(x[i] & m);
  }
  return n;
}

// d of every row of event k: forward step f (from the top bit down) produces row n - 1 - f
ZK_HD void assign_exp_chain(const ExpAssign& a, u64 k) {
  const u64* e = a.ev + 12 * k;
  const u64 b[4] = {e[0], e[1], e[2], e[3]}, x[4] = {e[4], e[5], e[6], e[7]};
  const u64 r0 = a.row_off[k], n = a.row_off[k + 1] - r0;
  if (n == 0) return;
  unsigned char* dlo = a.base + a.off[E_D];
  unsigned char* dhi = a.base + a.off[E_D + 1];
  u64 acc[4] = {b[0], b[1], b[2], b[3]};
  u64 row = r0 + n;
  for (int j = exp_bitlen(x) - 2; j >= 0; j--) {
    mul256_lo(acc, acc, acc);  // square: e = 2 e
    row--;
    st_u128(dlo, row, acc[0], acc[1]);
    st_u128(dhi, row, acc[2], acc[3]);
    if ((limb_at(x, j >> 6) >> (j & 63)) & 1) {  // multiply: e = e + 1
      mul256_lo(acc, b, acc);
      row--;
      st_u128(dlo, row, acc[0], acc[1]);
      st_u128(dhi, row, acc[2], acc[3]);
    }
  }
}

// every other cell of circuit row r, and table row r (+ the padding row at n_used)
ZK_HD void assign_exp_row(const ExpAssign& a, u64 r) {
  unsigned char* B = a.base;
  u64 b[4] = {1, 0, 0, 0}, ex[4] = {1, 0, 0, 0}, id[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0}, d[4] = {1, 0, 0, 0}, m[4];
  u64 odd = 1;
  bool step = false, last = false;
  if (r < a.n_used) {
    u64 lo = 0, hi = a.n_events;  // the largest k with row_off[k] <= r: the event (with rows) that holds row r
    while (hi - lo > 1) {
      const u64 mid = (lo + hi) >> 1;
      if (a.row_off[mid] <= r) lo = mid;
      else hi = mid;
    }
    const u64* e = a.ev + 12 * lo;
    const u64 x[4] = {e[4], e[5], e[6], e[7]};
    b[0] = e[0], b[1] = e[1], b[2] = e[2], b[3] = e[3];
    id[0] = e[8], id[1] = e[9], id[2] = e[10], id[3] = e[11];
    const u64 k = r - a.row_off[lo];
    last = r + 1 == a.row_off[lo + 1];
    step = true;
    // the bit j whose rows hold row k: the largest j < bitlen(x) - 1 with j + popcount(x mod 2^j) <= k
    int jl = 0, jh = exp_bitlen(x) - 1;
    while (jh - jl > 1) {
      const int mid = (jl + jh) >> 1;
      if ((u64)(mid + popc_below(x, mid)) <= k) jl = mid;
      else jh = mid;
    }
    const int sh = jl >> 6, bt = jl & 63;
#pragma unroll
    for (int i = 0; i < 4; i++) {  // e = x >> j
      const u64 l0 = limb_at(x, i + sh), l1 = limb_at(x, i + sh + 1);
      ex[i] = bt ? (l0 >> bt) | (l1 << (64 - bt)) : l0;
    }
    odd = (ex[0] & 1) && k == (u64)(jl + popc_below(x, jl));
    ex[0] &= odd ? ~0ull : ~1ull;
#pragma unroll
    for (int i = 0; i < 4; i++) q[i] = (ex[i] >> 1) | (i < 3 ? ex[i + 1] << 63 : 0);
    const u64* dl = (const u64*)(B + a.off[E_D]);
    const u64* dh = (const u64*)(B + a.off[E_D + 1]);
    d[0] = dl[2 * r], d[1] = dl[2 * r + 1], d[2] = dh[2 * r], d[3] = dh[2 * r + 1];
    if (last) {
      m[0] = b[0], m[1] = b[1], m[2] = b[2], m[3] = b[3];
    } else {
      m[0] = dl[2 * r + 2], m[1] = dl[2 * r + 3], m[2] = dh[2 * r + 2], m[3] = dh[2 * r + 3];
    }
  } else {  // fill_dummy_events: (1, 0, 0, 0, base 1, exponent 1, exponentiation 1, a 1, b 1, c 0, d 1, q 0, r 1)
    m[0] = 1, m[1] = m[2] = m[3] = 0;
    st_u128(B + a.off[E_D], r, 1, 0);
    st_u128(B + a.off[E_D + 1], r, 0, 0);
  }
  u64 bb[4];  // b = base (odd) or a, chosen cell by cell: a pointer to either array would put both in local memory
#pragma unroll
  for (int i = 0; i < 4; i++) bb[i] = odd ? b[i] : m[i];
  B[a.off[E_USABLE] + r] = 1;
  B[a.off[E_STEP] + r] = step;
  st_fr(B + a.off[E_ID], r, Fr{{id[0], id[1], id[2], id[3]}});
  B[a.off[E_LAST] + r] = last;
  st_u128(B + a.off[E_BASE], r, b[0], b[1]);
  st_u128(B + a.off[E_BASE + 1], r, b[2], b[3]);
  st_u128(B + a.off[E_EXPO], r, ex[0], ex[1]);
  st_u128(B + a.off[E_EXPO + 1], r, ex[2], ex[3]);
  st_u128(B + a.off[E_EXPN], r, d[0], d[1]);
  st_u128(B + a.off[E_EXPN + 1], r, d[2], d[3]);
  st_u128(B + a.off[E_A], r, m[0], m[1]);
  st_u128(B + a.off[E_A + 1], r, m[2], m[3]);
  st_u128(B + a.off[E_B], r, bb[0], bb[1]);
  st_u128(B + a.off[E_B + 1], r, bb[2], bb[3]);
  B[a.off[E_C] + r] = 0;
  B[a.off[E_C + 1] + r] = 0;
  st_u128(B + a.off[E_Q], r, q[0], q[1]);
  st_u128(B + a.off[E_Q + 1], r, q[2], q[3]);
  B[a.off[E_R] + r] = (unsigned char)odd;
  // the table row (Tables._convert_exp_circuit_to_table: is_step = 1 on every row, padding included): one per event
  // row, and the padding row once, at n_used
  if (r <= a.n_used) {
    unsigned char* T = a.tbase;
    T[a.toff[0] + r] = 1;
    st_fr(T + a.toff[1], r, Fr{{id[0], id[1], id[2], id[3]}});
    T[a.toff[2] + r] = last;
#pragma unroll
    for (int i = 0; i < 4; i++) ((u64*)(T + a.toff[3 + i]))[r] = b[i];
    st_u128(T + a.toff[7], r, ex[0], ex[1]);
    st_u128(T + a.toff[8], r, ex[2], ex[3]);
    st_u128(T + a.toff[9], r, d[0], d[1]);
    st_u128(T + a.toff[10], r, d[2], d[3]);
  }
}

// ---------------------------------------------------------------- public-inputs circuit
// public_data2witness (pi_circuit.py:839-1073) from the raw public-input stream F = b"".join(rpi_byte_values): one row
// per byte.  The values (block fields, tx-table fields, calldata bytes, withdrawal fields) lie back to back in F at
// offsets that are a closed form of MAX_TXS, MAX_CALLDATA_BYTES and MAX_WITHDRAWALS (pi_value_of).  Row r lies in the
// value whose forward range [s, s + len) holds r and carries F[2s + len - 1 - r]: each value's bytes reversed.  The
// reference processes the values from last to first, each value's bytes first to last; that order `seq` is row n-1
// down to row 0, and the digest is keccak256(seq).  rpi_bytes_keccakrlc is one Horner chain over all of seq: chunks of
// 32 bytes fold to (value, r^32) pairs (rlc_chunk), the pairs are scanned in two levels (a block of 256 threads over 4
// chunks each, then one block over the block totals), and each chunk replays its bytes from its carried-in value.  The
// per-tx calldata gas sums use the same scan over integers.  Everything else of a row is a closed form of the row and
// the few bytes it names.
#define PI_BLOCK_BYTES 8437ull  // N_BYTES_ONE + N_BYTES_BLOCK + N_BYTES_EXTRA_VALUE: the block section + 3 Words
#define PI_TX0 8454ull          // the first tx slot, after the empty tx row's (tx_id 8, index 8, value 1)
#define PI_SLOT_BYTES 336ull    // one tx slot: 10 fields of (tx_id 8, index 8, value lo, [value hi 16])
#define PI_WD_BYTES 56ull       // one withdrawal: id 8, validator_id 8, address lo 16, hi 16, amount 8
#define PI_CDL_OFF 256ull       // the CallDataLength value inside a slot (field 7's lo)
#define PI_TX_LEN 10ull
#define PI_TAG_CALLDATA 13  // TxContextFieldTag.CallData
#define PI_CDL_TAG 8        // TxContextFieldTag.CallDataLength
#define PI_SCAN_GROUP 4               // chunks per thread of k_assign_pi_scan
#define PI_SCAN_BLOCK_CHUNKS 1024ull  // chunks per block of k_assign_pi_scan (256 threads)
// the 28 cells of ZK_CIRCUIT_PI (pi.cu P_*), and the narrow width of each: flags, bytes and tags 1 B, counters and ids
// 8 B, Word halves 16 B, accumulators, inverses and the tx value lo (a 160-bit address is a Value) 32 B
enum { PA_QLAST, PA_QTX, PA_QCD, PA_QCD_START, PA_QKECCAK, PA_QVSTART, PA_TXID_INV, PA_VLO_INV, PA_DIFF_INV, PA_GAS,
       PA_FINAL, PA_QWD, PA_BYTES, PA_KRLC, PA_VLC, PA_DIG_LO, PA_DIG_HI, PA_QEN, PA_TXID, PA_TAG, PA_INDEX, PA_VLO, PA_VHI,
       PA_WD_ID, PA_WD_VAL, PA_WD_ALO, PA_WD_AHI, PA_WD_AMT };
static const unsigned char kPiAssignWidths[28] = {1, 1, 1, 1, 1, 1, 32, 32, 32, 8, 1, 1, 1, 32,
                                                  32, 16, 16, 1, 8, 1, 8, 32, 16, 8, 8, 16, 16, 8};
static const unsigned char kPiKeccakWidths[5] = {1, 32, 8, 16, 16};  // is_enabled, input_rlc, input_len, output lo, hi
static const unsigned char kPiGasWidths[3] = {8, 1, 8};              // tx_id, is_final, gas_cost_acc

struct RlcPair {
  Fr v, p;  // Horner value (canonical), r^len (Montgomery form)
};
ZK_HD RlcPair rlc_pair_op(const RlcPair& l, const RlcPair& r) {
  RlcPair o = l;
  rlc_combine(o.v, o.p, r.v, r.p);
  return o;
}
// the two scans: fold(lo, hi) is the monoid value of items [lo, hi), op combines left and right
struct PiKrlcScan {
  typedef RlcPair T;
  const unsigned char* seq;
  u64 n;
  Fr r_mont;
  ZK_HD T id() const { return RlcPair{fr_u64(0), fr_to_mont(fr_u64(1))}; }
  ZK_HD T fold(u64 lo, u64 hi) const {
    RlcPair o;
    rlc_chunk(seq, lo, hi, r_mont, o.v, o.p);
    return o;
  }
  static ZK_HD T op(const T& l, const T& r) { return rlc_pair_op(l, r); }
};
ZK_HD u64 pi_cd_cost(u64 b) { return b ? 16 : 4; }  // GAS_COST_TX_CALL_DATA_PER_(NON_)ZERO_BYTE
struct PiGasScan {
  typedef u64 T;
  const unsigned char* cd;  // the calldata bytes
  u64 n;
  ZK_HD T id() const { return 0; }
  ZK_HD T fold(u64 lo, u64 hi) const {
    u64 g = 0;
    for (u64 j = lo; j < hi; j++) g += pi_cd_cost(cd[j]);
    return g;
  }
  static ZK_HD T op(const T& l, const T& r) { return l + r; }
};

struct PiAssign {
  const unsigned char* F;  // the forward stream, n bytes
  unsigned char* seq;      // processing order: seq[n - 1 - r] = the byte of row r
  const u64* cd_off;       // [max_txs + 1] prefix sums of the CallDataLength fields
  Fr* inv;                 // [n_inv] 1/k (inv[0] = 0), n_inv = max(256, max_txs + 1)
  RlcPair* kx;             // per 32-byte chunk of seq: the Horner pair carried in from its block's earlier chunks
  RlcPair* ktop;           // per block of PI_SCAN_BLOCK_CHUNKS chunks: the pair carried in from earlier blocks
  u64* gx;                 // the same two arrays of the calldata gas scan
  u64* gtop;
  u64* dig;                // [4] keccak256(seq) as little-endian lanes, then [4] the digest Word (lo 2 limbs, hi 2 limbs)
  u64 n, max_txs, max_cd, max_wd, n_inv;
  Fr rand_mont, base_mont;  // ZK_CHALLENGE_PI_KECCAK, ZK_CHALLENGE_PI_BYTE_BASE in Montgomery form
  unsigned char* base;      // the circuit's narrow columns
  u64 off[28];
  unsigned char* kbase;  // the keccak table: 2 rows
  u64 koff[5];
  unsigned char* gbase;  // the calldata gas table: the zero row + one row per used calldata byte
  u64 goff[3];
};

// tx field f of a slot: its value lo is 20 bytes (from, to: 160-bit Values), 16 (Word lo) or 8; Words add a 16-byte hi
ZK_HD bool pi_field_word(u64 f) { return f == 2 || f == 6 || f == 9; }
ZK_HD u64 pi_field_lo(u64 f) { return (f == 3 || f == 4) ? 20 : pi_field_word(f) ? 16 : 8; }
ZK_HD u64 pi_field_len(u64 f) { return 16 + pi_field_lo(f) + (pi_field_word(f) ? 16 : 0); }
ZK_HD u64 pi_field_off(u64 f) {
  u64 o = 0;
  for (u64 g = 0; g < f; g++) o += pi_field_len(g);
  return o;
}
// the first ten values of the block section (0, coinbase, gas_limit, number, time, prev_randao lo, hi, base_fee lo, hi,
// chain_id); 16-byte Word halves follow from byte 117
ZK_HD u64 pi_head_len(u64 i) { return i == 0 ? 1 : i == 1 ? 20 : (i >= 5 && i <= 8) ? 16 : 8; }

// the value [s, s + len) of the forward stream that holds byte r
ZK_HD void pi_value_of(const PiAssign& a, u64 r, u64& s, u64& len) {
  const u64 c0 = PI_TX0 + PI_SLOT_BYTES * a.max_txs, w0 = c0 + a.max_cd;
  if (r < 117) {
    u64 o = 0, i = 0;
    while (o + pi_head_len(i) <= r) o += pi_head_len(i++);
    s = o, len = pi_head_len(i);
  } else if (r < PI_BLOCK_BYTES) {
    s = r - (r - 117) % 16, len = 16;
  } else if (r < PI_TX0) {  // the empty tx row: tx_id 8, index 8, value 1
    s = r < PI_BLOCK_BYTES + 8 ? PI_BLOCK_BYTES : r < PI_BLOCK_BYTES + 16 ? PI_BLOCK_BYTES + 8 : PI_BLOCK_BYTES + 16;
    len = r < PI_BLOCK_BYTES + 16 ? 8 : 1;
  } else if (r < c0) {
    u64 b = r - (r - PI_TX0) % PI_SLOT_BYTES, f = 0;
    while (b + pi_field_len(f) <= r) b += pi_field_len(f++);
    const u64 q = r - b, lo = pi_field_lo(f);
    if (q < 16) s = b + (q & 8), len = 8;  // tx_id, index
    else if (q < 16 + lo) s = b + 16, len = lo;
    else s = b + 16 + lo, len = 16;
  } else if (r < w0) {
    s = r, len = 1;
  } else {
    const u64 o = (r - w0) % PI_WD_BYTES, b = r - o;
    if (o < 16) s = b + (o & 8), len = 8;
    else if (o < 48) s = b + (o & ~15ull), len = 16;  // address lo, hi
    else s = b + 48, len = 8;
  }
}
ZK_HD u64 pi_byte(const PiAssign& a, u64 r) {
  u64 s, len;
  pi_value_of(a, r, s, len);
  return a.F[2 * s + len - 1 - r];
}
// nb <= 20 big-endian bytes as an integer (< 2^160)
ZK_HD Fr pi_be(const unsigned char* p, u64 nb) {
  u64 l0 = 0, l1 = 0, l2 = 0;
  for (u64 i = 0; i < nb; i++) {
    const u64 k = nb - 1 - i, v = (u64)p[i] << (8 * (k & 7));
    if (k < 8) l0 |= v;
    else if (k < 16) l1 |= v;
    else l2 |= v;
  }
  return Fr{{l0, l1, l2, 0}};
}
// 1/k for |k| < n_inv, from the staged table
ZK_HD Fr pi_inv_small(const PiAssign& a, u64 k, bool neg) {
  const Fr v = a.inv[k];
  return neg ? fr_sub(fr_u64(0), v) : v;
}
// the largest slot j < max_txs with cd_off[j] <= k: the tx whose calldata holds byte k (when k < cd_off[max_txs])
ZK_HD u64 pi_slot_of(const PiAssign& a, u64 k) {
  u64 lo = 0, hi = a.max_txs;
  while (hi - lo > 1) {
    const u64 mid = (lo + hi) >> 1;
    if (a.cd_off[mid] <= k) lo = mid;
    else hi = mid;
  }
  return lo;
}
// the gas of calldata bytes [0, x), x < max_cd, from the scan
ZK_HD u64 pi_gas_before(const PiAssign& a, u64 x) {
  const u64 c = x / ZK_SEG_CHUNK, c0 = PI_TX0 + PI_SLOT_BYTES * a.max_txs;
  u64 g = a.gtop[c / PI_SCAN_BLOCK_CHUNKS] + a.gx[c];
  for (u64 j = c * ZK_SEG_CHUNK; j < x; j++) g += pi_cd_cost(a.F[c0 + j]);
  return g;
}

ZK_HD void assign_pi_seq(const PiAssign& a, u64 r) { a.seq[a.n - 1 - r] = (unsigned char)pi_byte(a, r); }
ZK_HD void assign_pi_inv(const PiAssign& a, u64 k) { a.inv[k] = fr_inv(fr_u64(k)); }

// rpi_bytes_keccakrlc of the rows of 32-byte chunk c of seq (rows n-1-t for t in the chunk), from its carried-in value
ZK_HD void assign_pi_krlc(const PiAssign& a, u64 c) {
  const u64 t0 = c * ZK_SEG_CHUNK, t1 = zk_min64(t0 + ZK_SEG_CHUNK, a.n);
  Fr acc = rlc_pair_op(a.ktop[c / PI_SCAN_BLOCK_CHUNKS], a.kx[c]).v;
  for (u64 t = t0; t < t1; t++) {
    acc = fr_add_u64(fr_montmul(acc, a.rand_mont), a.seq[t]);
    st_fr(a.base + a.off[PA_KRLC], a.n - 1 - t, acc);
  }
}

// the tx-table cells of the calldata rows 10 * max_txs + 1 + k for the bytes k of 32-byte chunk c of the calldata, and
// their gas-table rows 1 + k.  Byte k belongs to the tx slot j with cd_off[j] <= k < cd_off[j + 1]; bytes from
// cd_off[max_txs] on are padding (tx_id, index, gas, is_final all 0), whose gas row would repeat the zero row: the table
// holds the zero row and the used bytes' rows only, the reference's set without copies.  (A lookup counts identical rows
// once by walking them, so ~n copies of the zero row cost each lookup of it ~n probes.)
ZK_HD void assign_pi_calldata(const PiAssign& a, u64 c) {
  const u64 k0 = c * ZK_SEG_CHUNK, k1 = zk_min64(k0 + ZK_SEG_CHUNK, a.max_cd), total = a.cd_off[a.max_txs];
  const u64 row0 = PI_TX_LEN * a.max_txs + 1, c0 = PI_TX0 + PI_SLOT_BYTES * a.max_txs;
  u64 j = pi_slot_of(a, k0);
  u64 g = k0 < total ? pi_gas_before(a, k0) - pi_gas_before(a, a.cd_off[j]) : 0;  // gas of this tx's bytes before k0
  unsigned char* B = a.base;
  unsigned char* T = a.gbase;
  for (u64 k = k0; k < k1; k++) {
    while (j + 1 < a.max_txs && a.cd_off[j + 1] <= k) j++, g = 0;  // a new tx starts at k
    const u64 b = a.F[c0 + k];
    const bool used = k < total;
    g += pi_cd_cost(b);
    const u64 tx_id = used ? j + 1 : 0, idx = used ? k - a.cd_off[j] : 0, gas = used ? g : 0;
    const bool fin = used && k + 1 == a.cd_off[j + 1];
    u64 nxt = 0;  // the next row's tx_id (0 after the last calldata row)
    if (k + 1 < total) {
      u64 jn = j;
      while (jn + 1 < a.max_txs && a.cd_off[jn + 1] <= k + 1) jn++;
      nxt = jn + 1;
    }
    const u64 r = row0 + k;
    B[a.off[PA_QTX] + r] = 0;
    B[a.off[PA_QCD] + r] = 1;
    B[a.off[PA_QCD_START] + r] = k == 0;
    st_fr(B + a.off[PA_TXID_INV], r, a.inv[tx_id]);
    st_fr(B + a.off[PA_VLO_INV], r, a.inv[b]);
    st_fr(B + a.off[PA_DIFF_INV], r, nxt >= tx_id ? pi_inv_small(a, nxt - tx_id, false) : pi_inv_small(a, tx_id - nxt, true));
    ((u64*)(B + a.off[PA_GAS]))[r] = gas;
    B[a.off[PA_FINAL] + r] = fin;
    ((u64*)(B + a.off[PA_TXID]))[r] = tx_id;
    B[a.off[PA_TAG] + r] = PI_TAG_CALLDATA;
    ((u64*)(B + a.off[PA_INDEX]))[r] = idx;
    st_fr(B + a.off[PA_VLO], r, fr_u64(b));
    st_u128(B + a.off[PA_VHI], r, 0, 0);
    if (used) {
      ((u64*)(T + a.goff[0]))[1 + k] = tx_id;
      T[a.goff[1] + 1 + k] = fin;
      ((u64*)(T + a.goff[2]))[1 + k] = gas;
    }
  }
}

// every cell of row r but rpi_bytes_keccakrlc, the calldata rows' tx-table cells and row 0's digest
ZK_HD void assign_pi_row(const PiAssign& a, u64 r) {
  unsigned char* B = a.base;
  const unsigned char* F = a.F;
  u64 s, len;
  pi_value_of(a, r, s, len);
  const u64 last = 2 * s + len - 1 - r;  // the forward position of this row's byte
  Fr lc = fr_u64(0);  // rpi_value_lc: Horner over the value's bytes from its first one to this row's
  for (u64 j = s; j <= last; j++) lc = fr_add_u64(fr_montmul(lc, a.base_mont), F[j]);
  B[a.off[PA_QLAST] + r] = r == a.n - 1;
  B[a.off[PA_QKECCAK] + r] = r == 0;
  B[a.off[PA_QVSTART] + r] = r == s + len - 1;
  B[a.off[PA_BYTES] + r] = F[last];
  st_fr(B + a.off[PA_VLC], r, lc);
  st_u128(B + a.off[PA_DIG_LO], r, 0, 0);
  st_u128(B + a.off[PA_DIG_HI], r, 0, 0);
  B[a.off[PA_QEN] + r] = 1;
  const u64 n_tx = PI_TX_LEN * a.max_txs + 1, n_cd = n_tx + a.max_cd;
  if (r < n_tx || r >= n_cd) {  // a tx-table row (the empty row 0, then slot (r - 1) / 10, field (r - 1) % 10), or none
    u64 tx_id = 0, idx = 0, tag = 0, h0 = 0, h1 = 0;
    Fr lo = fr_u64(0), tag_inv = fr_u64(0), lo_inv = fr_u64(0);
    if (r < n_tx) {
      u64 b = PI_BLOCK_BYTES, w = 1;
      bool word = false;
      if (r) {
        const u64 f = (r - 1) % PI_TX_LEN;
        b = PI_TX0 + PI_SLOT_BYTES * ((r - 1) / PI_TX_LEN) + pi_field_off(f);
        w = pi_field_lo(f);
        word = pi_field_word(f);
        tag = f + 1;  // i % TX_LEN or TX_LEN
      }
      tx_id = pi_be(F + b, 8).l[0];
      idx = pi_be(F + b + 8, 8).l[0];
      lo = pi_be(F + b + 16, w);
      if (word) {
        const Fr h = pi_be(F + b + 16 + w, 16);
        h0 = h.l[0], h1 = h.l[1];
      }
      tag_inv = tag >= PI_CDL_TAG ? pi_inv_small(a, tag - PI_CDL_TAG, false) : pi_inv_small(a, PI_CDL_TAG - tag, true);
      lo_inv = fr_inv(lo);
    }
    B[a.off[PA_QTX] + r] = r < n_tx;
    B[a.off[PA_QCD] + r] = 0;
    B[a.off[PA_QCD_START] + r] = 0;
    st_fr(B + a.off[PA_TXID_INV], r, tag_inv);
    st_fr(B + a.off[PA_VLO_INV], r, lo_inv);
    st_fr(B + a.off[PA_DIFF_INV], r, fr_u64(0));
    ((u64*)(B + a.off[PA_GAS]))[r] = 0;
    B[a.off[PA_FINAL] + r] = 0;
    ((u64*)(B + a.off[PA_TXID]))[r] = tx_id;
    B[a.off[PA_TAG] + r] = (unsigned char)tag;
    ((u64*)(B + a.off[PA_INDEX]))[r] = idx;
    st_fr(B + a.off[PA_VLO], r, lo);
    st_u128(B + a.off[PA_VHI], r, h0, h1);
  }
  u64 wd[7] = {0, 0, 0, 0, 0, 0, 0};  // id, validator_id, address lo (2 limbs), hi (2 limbs), amount
  const bool is_wd = r >= n_cd && r - n_cd < a.max_wd;
  if (is_wd) {
    const unsigned char* p = F + PI_TX0 + PI_SLOT_BYTES * a.max_txs + a.max_cd + PI_WD_BYTES * (r - n_cd);
    const Fr lo = pi_be(p + 16, 16), hi = pi_be(p + 32, 16);
    wd[0] = pi_be(p, 8).l[0], wd[1] = pi_be(p + 8, 8).l[0], wd[2] = lo.l[0], wd[3] = lo.l[1], wd[4] = hi.l[0], wd[5] = hi.l[1];
    wd[6] = pi_be(p + 48, 8).l[0];
  }
  B[a.off[PA_QWD] + r] = is_wd;
  ((u64*)(B + a.off[PA_WD_ID]))[r] = wd[0];
  ((u64*)(B + a.off[PA_WD_VAL]))[r] = wd[1];
  st_u128(B + a.off[PA_WD_ALO], r, wd[2], wd[3]);
  st_u128(B + a.off[PA_WD_AHI], r, wd[4], wd[5]);
  ((u64*)(B + a.off[PA_WD_AMT]))[r] = wd[6];
  if (r == 0) {  // the gas table's zero row
    unsigned char* T = a.gbase;
    ((u64*)(T + a.goff[0]))[0] = 0;
    T[a.goff[1]] = 0;
    ((u64*)(T + a.goff[2]))[0] = 0;
  }
}

// after the sponge and the keccak RLC: row 0's digest cells, the keccak table (0, 0, 0, 0, 0), (1, krlc[0], n, digest
// lo, hi), and the digest Word at dig[4..8].  The reference's Word(keccak256(seq)) reads the 32 digest bytes
// little-endian (lo = bytes 0..15), so its limbs are the sponge's first four lanes as they are.
ZK_HD void assign_pi_finish(const PiAssign& a) {
  const u64 lo[2] = {a.dig[0], a.dig[1]}, hi[2] = {a.dig[2], a.dig[3]};
  unsigned char* B = a.base;
  st_u128(B + a.off[PA_DIG_LO], 0, lo[0], lo[1]);
  st_u128(B + a.off[PA_DIG_HI], 0, hi[0], hi[1]);
  unsigned char* K = a.kbase;
  const Fr rlc = ld_col(B + a.off[PA_KRLC], 32, 0);
  K[a.koff[0]] = 0;
  K[a.koff[0] + 1] = 1;
  st_fr(K + a.koff[1], 0, fr_u64(0));
  st_fr(K + a.koff[1], 1, rlc);
  ((u64*)(K + a.koff[2]))[0] = 0;
  ((u64*)(K + a.koff[2]))[1] = a.n;
  st_u128(K + a.koff[3], 0, 0, 0);
  st_u128(K + a.koff[3], 1, lo[0], lo[1]);
  st_u128(K + a.koff[4], 0, 0, 0);
  st_u128(K + a.koff[4], 1, hi[0], hi[1]);
  a.dig[4] = lo[0], a.dig[5] = lo[1], a.dig[6] = hi[0], a.dig[7] = hi[1];
}

// host validation of zk_assign_pi_circuit (and of the CPU emulation): nullptr if the stream's length, the maxima and
// the CallDataLength fields are acceptable, with cd_off[max_txs + 1] filled; the reason otherwise
static const char* pi_shape_error(u64 max_txs, u64 max_cd, u64 max_wd, u64 n_bytes) {
  if (max_txs == 0) return "public inputs: MAX_TXS must be at least 1 (the reference asserts a tx)";
  if (max_wd == 0) return "public inputs: MAX_WITHDRAWALS must be at least 1 (the reference asserts a withdrawal)";
  if (max_txs >= (1ull << 31) || max_cd >= (1ull << 31) || max_wd >= (1ull << 31))
    return "public inputs: too many rows (row ids are below 2^31 - 1)";
  if (n_bytes != PI_TX0 + PI_SLOT_BYTES * max_txs + max_cd + PI_WD_BYTES * max_wd)
    return "public inputs: the stream's length is not the circuit_len of the three maxima";
  if (n_bytes >= 0x7FFFFFFFull) return "public inputs: too many rows (row ids are below 2^31 - 1)";
  return nullptr;
}
static const char* pi_calldata_offsets(u64 max_txs, u64 max_cd, const unsigned char* raw, u64* cd_off) {
  cd_off[0] = 0;
  for (u64 j = 0; j < max_txs; j++) {
    const u64 len = pi_be(raw + PI_TX0 + PI_SLOT_BYTES * j + PI_CDL_OFF, 8).l[0];
    if (len > max_cd - cd_off[j]) return "public inputs: the CallDataLength fields sum to more than MAX_CALLDATA_BYTES";
    cd_off[j + 1] = cd_off[j] + len;
  }
  return nullptr;
}

// ---------------------------------------------------------------- tx table
// Transaction.table_assignments (evm_circuit/typing.py:209-281) per tx, in tx order: the 12 fixed rows (tags 1..12,
// call_data_index_or_zero 0), then one (id, CallData, i, byte, 0) row per call-data byte.  Tx k owns rows
// [12 k + cd_off[k], 12 (k + 1) + cd_off[k + 1]).  A record is 11 cells of 4 little-endian limbs: id, nonce, gas,
// gas_price, caller_address, callee_address, is_create, value, tx_invalid, access_list_gas_cost, tx_sign_hash; the
// Word cells (gas_price, caller, callee, value) are 256-bit integers split into (lo, hi) here, the others values.
// CallDataLength comes from the offsets, CallDataGasCost = 16 len - 12 zeros from the zero-byte counts.
#define TX_REC_CELLS 11
#define TX_FIXED_ROWS 12
#define TX_TAG_CALLDATA 13
enum { TXR_ID, TXR_NONCE, TXR_GAS, TXR_GAS_PRICE, TXR_CALLER, TXR_CALLEE, TXR_IS_CREATE, TXR_VALUE, TXR_INVALID, TXR_ALGC,
       TXR_SIGN_HASH };
struct TxTableAssign {
  const u64* rec;            // [n_txs][11][4]
  const unsigned char* cd;   // call data of every tx, back to back
  const u64* cd_off;         // [n_txs + 1]
  unsigned long long* zeros;  // [n_txs] zero bytes of each tx's call data (k_assign_tx_zeros)
  u64 n_txs, n_rows, n_cd;
  unsigned char* base;  // the table's narrow columns: tx_id, tag, index, value lo, value hi
  u64 off[5];
  unsigned char width[5];
  unsigned char* flags;  // [n_rows] bit 0: the value is a Word
};

// tag -> the record cell it takes (-1: CallDataLength / CallDataGasCost, from the call data), and whether it is a Word
ZK_HD int tx_tag_cell(u64 tag) {
  return tag <= 7 ? (int)tag : tag == 8 || tag == 9 ? -1 : (int)tag - 2;
}
ZK_HD bool tx_tag_word(u64 tag) { return tag == 3 || tag == 4 || tag == 5 || tag == 7; }
ZK_HD void st_width(unsigned char* col, u32 width, u64 row, const Fr& v) {
  if (width == 32) st_fr(col, row, v);
  else if (width == 16) st_u128(col, row, v.l[0], v.l[1]);
  else st_narrow(col, width, row, v.l[0]);
}
// the tx whose call data holds byte j (j < n_cd): the largest k < n_txs with cd_off[k] <= j
ZK_HD u64 tx_of_byte(const TxTableAssign& a, u64 j) {
  u64 lo = 0, hi = a.n_txs;
  while (hi - lo > 1) {
    const u64 mid = (lo + hi) >> 1;
    if (a.cd_off[mid] <= j) lo = mid;
    else hi = mid;
  }
  return lo;
}
ZK_HD void assign_tx_row(const TxTableAssign& a, u64 r) {
  u64 lo = 0, hi = a.n_txs;  // the largest k with 12 k + cd_off[k] <= r: the tx that holds row r
  while (hi - lo > 1) {
    const u64 mid = (lo + hi) >> 1;
    if (TX_FIXED_ROWS * mid + a.cd_off[mid] <= r) lo = mid;
    else hi = mid;
  }
  const u64 k = lo, local = r - (TX_FIXED_ROWS * k + a.cd_off[k]);
  const u64* rec = a.rec + 4 * TX_REC_CELLS * k;
  u64 tag = TX_TAG_CALLDATA, index = 0;
  Fr vlo = fr_u64(0), vhi = fr_u64(0);
  bool word = false;
  if (local < TX_FIXED_ROWS) {
    tag = local + 1;
    const u64 len = a.cd_off[k + 1] - a.cd_off[k];
    const int cell = tx_tag_cell(tag);
    word = tx_tag_word(tag);
    if (cell < 0) {
      vlo = fr_u64(tag == 8 ? len : 16 * len - 12 * (u64)a.zeros[k]);
    } else {
      const u64* c = rec + 4 * cell;
      vlo = Fr{{c[0], c[1], word ? 0 : c[2], word ? 0 : c[3]}};
      if (word) vhi = Fr{{c[2], c[3], 0, 0}};
    }
  } else {
    index = local - TX_FIXED_ROWS;
    vlo = fr_u64(a.cd[a.cd_off[k] + index]);
  }
  st_width(a.base + a.off[0], a.width[0], r, Fr{{rec[0], rec[1], rec[2], rec[3]}});
  a.base[a.off[1] + r] = (unsigned char)tag;
  st_narrow(a.base + a.off[2], a.width[2], r, index);
  st_width(a.base + a.off[3], a.width[3], r, vlo);
  st_width(a.base + a.off[4], a.width[4], r, vhi);
  a.flags[r] = word;
}

// the width (1, 2, 4, 8, 16 or 32 bytes) that holds a 4-limb value
static unsigned char tx_cell_width(const u64* v) {
  if (v[2] | v[3]) return 32;
  if (v[1]) return 16;
  return v[0] < (1ull << 8) ? 1 : v[0] < (1ull << 16) ? 2 : v[0] < (1ull << 32) ? 4 : 8;
}
static bool tx_fr_canonical(const u64* v) { return fr_lt(Fr{{v[0], v[1], v[2], v[3]}}, Fr{{ZK_P0, ZK_P1, ZK_P2, ZK_P3}}); }
// host validation and column widths of zk_assign_tx_table (and of the CPU emulation): nullptr with *n_rows and
// width[5] filled, the reason otherwise.  The widths come from the record maxima and from bounds of the derived
// cells (CallDataLength <= the longest call data, CallDataGasCost <= 16 times it), as the packer measures ranges.
static const char* tx_table_plan(u64 n_txs, const u64* rec, const u64* cd_off, u64* n_rows, unsigned char* width) {
  if (cd_off[0] != 0) return "tx table: call_data_offsets[0] must be 0";
  u64 max_len = 0;
  width[0] = 1, width[1] = 1, width[2] = 1, width[3] = 1, width[4] = 1;
  for (u64 k = 0; k < n_txs; k++) {
    if (cd_off[k + 1] < cd_off[k]) return "tx table: call_data_offsets must be non-decreasing";
    max_len = std::max<u64>(max_len, cd_off[k + 1] - cd_off[k]);
    for (int c = 0; c < TX_REC_CELLS; c++) {
      const u64* v = rec + 4 * (TX_REC_CELLS * k + c);
      const bool word = c == TXR_GAS_PRICE || c == TXR_CALLER || c == TXR_CALLEE || c == TXR_VALUE;
      if (!word && !tx_fr_canonical(v)) return "tx table: a value cell is not canonical (>= p)";
      if (c == TXR_ID) {
        width[0] = std::max(width[0], tx_cell_width(v));
      } else if (word) {
        const u64 lo[4] = {v[0], v[1], 0, 0}, hi[4] = {v[2], v[3], 0, 0};
        width[3] = std::max(width[3], tx_cell_width(lo));
        width[4] = std::max(width[4], tx_cell_width(hi));
      } else {
        width[3] = std::max(width[3], tx_cell_width(v));
      }
    }
    if (TX_FIXED_ROWS * (k + 1) + cd_off[k + 1] >= 0x7FFFFFFFull) return "tx table: too many rows (table rows are below 2^31 - 1)";
  }
  const u64 bound[4] = {16 * max_len, 0, 0, 0}, idx[4] = {max_len, 0, 0, 0};  // CallDataGasCost, CallDataLength
  width[3] = std::max(width[3], tx_cell_width(bound));
  width[2] = std::max(width[2], tx_cell_width(idx));
  *n_rows = TX_FIXED_ROWS * n_txs + cd_off[n_txs];
  return nullptr;
}

// ---------------------------------------------------------------- copy table
// Tables._convert_copy_circuit_to_table (evm_circuit/table.py:627-652) over the resident copy circuit: every row i whose
// is_first equals 1 gives one row, in circuit order, of (is_first, id lo, hi, tag, addr, src_addr_end, bytes_left,
// rlc_acc, rw_counter, rwc_inc_left) of row i and (id lo, hi, tag, addr) of row i + 1 as the destination's.  A stream
// compaction: k_copy_table_count counts each tile's rows and raises the reference's two asserts as the smallest
// failing row, the host scans the tile counts (k_assign_pi_scan_top) and k_copy_table_write writes each tile's rows
// from its offset.
#define CT_TILE 1024  // circuit rows per block of the two copy-table kernels (256 threads, 4 rows each)
// the circuit column each table column comes from (table columns 4, 5, 6 and 9 from row i + 1)
static const unsigned char kCopyTableSrc[14] = {1, 3, 4, 5, 3, 4, 5, 6, 7, 6, 8, 10, 13, 14};
struct CopyTableAssign {
  WitnessDev w;  // the resident copy circuit, any storage form
  u64* tile_count;  // [n_tiles] is_first rows of each tile, then (after the scan) the rows before each tile
  unsigned long long* fail;  // [0] the smallest row that fails an assert (~0: none), [1] is_first rows in all
  unsigned char* base;       // the table's narrow columns
  u64 off[14];
  unsigned char width[14];
};
// a count: as the PI scan's monoid over `flags`, fold(lo, hi) counts the items in [lo, hi) with a bit of `mask` set
// (k_assign_pi_scan); the copy table scans its tile counts with k_assign_pi_scan_top only, which never folds
struct CountScan {
  typedef u64 T;
  const unsigned char* flags;
  u64 n;
  unsigned mask;
  ZK_HD T id() const { return 0; }
  ZK_HD T fold(u64 lo, u64 hi) const {
    u64 c = 0;
    for (u64 j = lo; j < hi; j++) c += (flags[j] & mask) != 0;
    return c;
  }
  static ZK_HD T op(const T& l, const T& r) { return l + r; }
};
ZK_HD bool fr_is_one(const Fr& v) { return v.l[0] == 1 && !(v.l[1] | v.l[2] | v.l[3]); }
ZK_HD bool copy_row_is_first(const CopyTableAssign& a, u64 i) { return i < a.w.n_rows && fr_is_one(wcell(a.w, 1, i)); }
// an is_first row the reference's conversion asserts on: the last row ("Not enough rows in copy circuit"), or a next
// row whose q_step is not 0 ("Invalid copy circuit")
ZK_HD bool copy_row_fails(const CopyTableAssign& a, u64 i) {
  if (i + 1 == a.w.n_rows) return true;
  const Fr q = wcell(a.w, 0, i + 1);
  return (q.l[0] | q.l[1] | q.l[2] | q.l[3]) != 0;
}
ZK_HD void copy_table_row(const CopyTableAssign& a, u64 i, u64 pos) {
  unsigned char* B = a.base;
  st_width(B + a.off[0], a.width[0], pos, wcell(a.w, 1, i));
  st_width(B + a.off[1], a.width[1], pos, wcell(a.w, 3, i));
  st_width(B + a.off[2], a.width[2], pos, wcell(a.w, 4, i));
  st_width(B + a.off[3], a.width[3], pos, wcell(a.w, 5, i));
  st_width(B + a.off[4], a.width[4], pos, wcell(a.w, 3, i + 1));
  st_width(B + a.off[5], a.width[5], pos, wcell(a.w, 4, i + 1));
  st_width(B + a.off[6], a.width[6], pos, wcell(a.w, 5, i + 1));
  st_width(B + a.off[7], a.width[7], pos, wcell(a.w, 6, i));
  st_width(B + a.off[8], a.width[8], pos, wcell(a.w, 7, i));
  st_width(B + a.off[9], a.width[9], pos, wcell(a.w, 6, i + 1));
  st_width(B + a.off[10], a.width[10], pos, wcell(a.w, 8, i));
  st_width(B + a.off[11], a.width[11], pos, wcell(a.w, 10, i));
  st_width(B + a.off[12], a.width[12], pos, wcell(a.w, 13, i));
  st_width(B + a.off[13], a.width[13], pos, wcell(a.w, 14, i));
}

// ---------------------------------------------------------------- state circuit roots + MPT table
// _mock_mpt_updates (state_circuit.py:903-933) walks the operations once, keeping the first touch of each MPT key
// (address, field_tag, storage_key lo, hi) of an Account or Storage op; update u (first-touch order) moves the root
// from 3 + 5u to 3 + 5(u + 1).  assign_state_circuit (:861-889) gives row k root_prev of the update of the first MPT op
// after k, or the final root 3 + 5U.  Here: an open-addressing hash table over the MPT ops keeps the smallest op
// index per key (an op is a first touch when it is its key's minimum), count scans over the first-touch and MPT-op
// flags rank the updates and list the MPT ops in order, and every row and table row is then a closed form.
#define SM_EMPTY 0xFFFFFFFFFFFFFFFFull  // a slot is (hash32 << 32) | op index of the op that claimed it
#define SM_TAG_STORAGE 4
#define SM_TAG_ACCOUNT 6
#define SM_PROOF_STORAGE_MOD 6
#define SM_FAIL_FIELD_TAG 1  // a first-touch Account op's field tag is not 1..4 (the mirror's KeyError)
#define SM_FAIL_WORD 2       // a first-touch op's Word value or initial value is >= 2^256 (Word() asserts)
// the 13 operation cells (zk_assign_state_circuit_mpt): the 15 of zk_assign_state_circuit without the root
enum { SO_RWC, SO_WRITE, SO_TAG, SO_ID, SO_ADDR, SO_FIELD, SO_KLO, SO_KHI, SO_VLO, SO_VHI, SO_ILO, SO_IHI, SO_SEL };
struct StateMpt {
  const unsigned char* base;  // the staged operation columns
  u64 off[13];
  unsigned char w[13];
  const unsigned char* flags;  // row flags (bit 0: value is a Word, bit 1: initial value is a Word), may be null
  u64 n;
  u64* slots;     // [mask + 1], SM_EMPTY = free
  u32* key_min;   // [mask + 1] the smallest op index of the key that claimed the slot
  u32* rank_at;   // [mask + 1] the update rank of that key
  u64 mask;
  u32* slot_of;   // [n] the slot of op i's key, ~0: not an MPT op
  unsigned char* fl;  // [n] bit 0: an MPT op, bit 1: a first touch
  unsigned long long* stat;  // [0] the first failing op ((i << 2) | SM_FAIL_*, ~0: none), [1] updates, [2] MPT ops
  const u64 *x_upd, *top_upd, *x_mpt, *top_mpt;  // the two count scans (k_assign_pi_scan)
  u32* upd_op;  // [U] the op of update u
  u32* mpt_op;  // [MPT ops] the MPT ops in order
  u64 n_upd, n_mpt;
  unsigned char* root;  // the state matrix's root lo column, 8 bytes per row
  unsigned char* tbase;  // the MPT table's narrow columns
  u64 toff[12];
  unsigned char twidth[12];
};
ZK_HD Fr sm_cell(const StateMpt& a, int c, u64 i) { return ld_col(a.base + a.off[c], a.w[c], i); }
ZK_HD bool sm_is(const Fr& v, u64 x) { return v.l[0] == x && !(v.l[1] | v.l[2] | v.l[3]); }
// the key hash: a multiply-xor over the 16 limbs of the 4 key cells, then a 64-bit finaliser; unkeyed, so the slot
// of a key is a function of the key and the capacity alone (tests build colliding keys from it)
ZK_HD u64 state_mpt_hash(const Fr (&k)[4]) {
  u64 h = 0x243F6A8885A308D3ull;
#pragma unroll
  for (int c = 0; c < 4; c++)
#pragma unroll
    for (int q = 0; q < 4; q++) h = (h ^ k[c].l[q]) * 0x9E3779B97F4A7C15ull + (u64)(4 * c + q);
  h ^= h >> 32;
  h *= 0xD6E8FEB86659FD93ull;
  h ^= h >> 32;
  return h;
}
// op i's MPT key, false if it is not an Account or Storage op
ZK_HD bool state_mpt_key(const StateMpt& a, u64 i, Fr (&k)[4]) {
  const Fr tag = sm_cell(a, SO_TAG, i);
  if (!sm_is(tag, SM_TAG_STORAGE) && !sm_is(tag, SM_TAG_ACCOUNT)) return false;
  k[0] = sm_cell(a, SO_ADDR, i);
  k[1] = sm_cell(a, SO_FIELD, i);
  k[2] = sm_cell(a, SO_KLO, i);
  k[3] = sm_cell(a, SO_KHI, i);
  return true;
}
// claim or find the slot of op i's key and lower the key's minimum to i
ZK_HD void state_mpt_insert(const StateMpt& a, u64 i) {
  Fr k[4];
  if (!state_mpt_key(a, i, k)) {
    a.slot_of[i] = ~0u;
    a.fl[i] = 0;
    return;
  }
  const u64 h = state_mpt_hash(k), entry = (h & 0xFFFFFFFF00000000ull) | i;
  u64 b = h & a.mask;
  for (;;) {
    const u64 old = atomic_cas_u64(&a.slots[b], SM_EMPTY, entry);
    if (old == SM_EMPTY) break;
    if ((old >> 32) == (entry >> 32)) {  // same fingerprint: compare the full key with the claimer's
      Fr o[4];
      state_mpt_key(a, (u32)old, o);
      if (fr_eq(o[0], k[0]) && fr_eq(o[1], k[1]) && fr_eq(o[2], k[2]) && fr_eq(o[3], k[3])) break;
    }
    b = (b + 1) & a.mask;
  }
  a.slot_of[i] = (u32)b;
  atomic_min_u32(&a.key_min[b], (u32)i);
  a.fl[i] = 1;
}
// a Word's integer lo + hi 2^128 as 4 limbs; false if it is >= 2^256
ZK_HD bool sm_word_int(const Fr& lo, const Fr& hi, u64 (&v)[4]) {
  v[0] = lo.l[0], v[1] = lo.l[1];
  v[2] = lo.l[2] + hi.l[0];
  const u64 c2 = v[2] < hi.l[0];
  const u64 s3 = lo.l[3] + hi.l[1];
  v[3] = s3 + c2;
  const bool carry = s3 < hi.l[1] || v[3] < c2;
  return !(carry || hi.l[2] || hi.l[3]);
}
// Word(op.value.int_value()) of a value cell pair: a field value is lo itself, a Word lo + hi 2^128
ZK_HD bool sm_value(const StateMpt& a, u64 i, int c_lo, bool word, u64 (&v)[4]) {
  const Fr lo = sm_cell(a, c_lo, i);
  if (!word) {
    v[0] = lo.l[0], v[1] = lo.l[1], v[2] = lo.l[2], v[3] = lo.l[3];
    return true;
  }
  return sm_word_int(lo, sm_cell(a, c_lo + 1, i), v);
}
ZK_HD unsigned sm_flags(const StateMpt& a, u64 i) { return a.flags ? a.flags[i] : 0; }
// after every insert: mark op i's first touch, and the reason (SM_FAIL_*) the mirror's loop would stop at it, or 0
ZK_HD unsigned state_mpt_first(const StateMpt& a, u64 i, unsigned* fail) {
  *fail = 0;
  const u32 s = a.slot_of[i];
  if (s == ~0u) return 0;
  const bool first = a.key_min[s] == (u32)i;
  a.fl[i] = first ? 3 : 1;
  if (first) {
    const Fr ft = sm_cell(a, SO_FIELD, i);
    const unsigned f = sm_flags(a, i);
    u64 v[4];
    if (sm_is(sm_cell(a, SO_TAG, i), SM_TAG_ACCOUNT) && (ft.l[1] | ft.l[2] | ft.l[3] || ft.l[0] < 1 || ft.l[0] > 4)) *fail = SM_FAIL_FIELD_TAG;
    else if (!sm_value(a, i, SO_VLO, f & 1, v) || !sm_value(a, i, SO_ILO, f & 2, v)) *fail = SM_FAIL_WORD;
  }
  return a.fl[i];
}
// the items before j (< n) with a bit of `mask` set, from a count scan
ZK_HD u64 sm_count_before(const u64* x, const u64* top, const unsigned char* fl, unsigned mask, u64 j) {
  const u64 c = j / ZK_SEG_CHUNK;
  u64 v = top[c / PI_SCAN_BLOCK_CHUNKS] + x[c];
  for (u64 t = c * ZK_SEG_CHUNK; t < j; t++) v += (fl[t] & mask) != 0;
  return v;
}
// op i's place in the ordered MPT-op list and, for a first touch, its update rank
ZK_HD void state_mpt_compact(const StateMpt& a, u64 i) {
  const unsigned f = a.fl[i];
  if (f & 1) a.mpt_op[sm_count_before(a.x_mpt, a.top_mpt, a.fl, 1, i)] = (u32)i;
  if (f & 2) {
    const u64 r = sm_count_before(a.x_upd, a.top_upd, a.fl, 2, i);
    a.upd_op[r] = (u32)i;
    a.rank_at[a.slot_of[i]] = (u32)r;
  }
}
// row k's root lo: root_prev of the first MPT op after k, or the final root
ZK_HD void state_mpt_row_root(const StateMpt& a, u64 k) {
  u64 root = 3 + 5 * a.n_upd;
  if (k + 1 < a.n) {
    const u64 j = sm_count_before(a.x_mpt, a.top_mpt, a.fl, 1, k + 1);
    if (j < a.n_mpt) root = 3 + 5 * (u64)a.rank_at[a.slot_of[a.mpt_op[j]]];
  }
  ((u64*)a.root)[k] = root;
}
// MPT table row u from the op of update u: address, proof type, key lo, hi, root, 0, root_prev, 0, value lo, hi,
// value_prev lo, hi, the two values re-split into 128-bit halves
ZK_HD void state_mpt_table_row(const StateMpt& a, u64 u) {
  const u64 i = a.upd_op[u];
  const unsigned f = sm_flags(a, i);
  const Fr field = sm_cell(a, SO_FIELD, i);
  const u64 proof = sm_is(sm_cell(a, SO_TAG, i), SM_TAG_STORAGE) ? SM_PROOF_STORAGE_MOD : field.l[0];
  u64 v[4], p[4];
  sm_value(a, i, SO_VLO, f & 1, v);
  sm_value(a, i, SO_ILO, f & 2, p);
  unsigned char* T = a.tbase;
  st_width(T + a.toff[0], a.twidth[0], u, sm_cell(a, SO_ADDR, i));
  T[a.toff[1] + u] = (unsigned char)proof;
  st_width(T + a.toff[2], a.twidth[2], u, sm_cell(a, SO_KLO, i));
  st_width(T + a.toff[3], a.twidth[3], u, sm_cell(a, SO_KHI, i));
  ((u64*)(T + a.toff[4]))[u] = 3 + 5 * (u + 1);
  T[a.toff[5] + u] = 0;
  ((u64*)(T + a.toff[6]))[u] = 3 + 5 * u;
  T[a.toff[7] + u] = 0;
  st_u128(T + a.toff[8], u, v[0], v[1]);
  st_u128(T + a.toff[9], u, v[2], v[3]);
  st_u128(T + a.toff[10], u, p[0], p[1]);
  st_u128(T + a.toff[11], u, p[2], p[3]);
}

// host validation of the packed operation columns of zk_assign_state_circuit (15) and zk_assign_state_circuit_mpt (13)
// (and of the CPU emulation): the row bound, the column format, and the address (column 4) within 160 bits
static const char* state_ops_error(uint64_t n_rows, int n_cols, const void* packed_ops, uint64_t total_bytes,
                                   const uint64_t* col_offsets, const uint8_t* col_widths) {
  if (n_rows >= 0xFFFFFFFFull) return "too many rows (row ids are uint32)";
  if (!col_offsets || !col_widths) return "the state circuit needs offsets and widths of the operation columns";
  for (int c = 0; c < n_cols; c++) {
    const unsigned w = col_widths[c];
    if (!(w == 0 || w == 1 || w == 2 || w == 4 || w == 8 || w == 16 || w == 32)) return "packed column width must be 0, 1, 2, 4, 8, 16 or 32";
    if (col_offsets[c] % 32 || col_offsets[c] + (w ? (size_t)w * n_rows : 32) > total_bytes)
      return "packed column offset misaligned or outside the buffer";
  }
  if (col_widths[4] == 32) {  // op.address.to_bytes(20, "little") raises OverflowError beyond 160 bits (state_circuit.py:832)
    const u64* a = (const u64*)((const unsigned char*)packed_ops + col_offsets[4]);
    for (u64 r = 0; r < n_rows; r++)
      if ((a[4 * r + 2] >> 32) || a[4 * r + 3]) return "operation address does not fit 20 bytes (op2row raises OverflowError)";
  }
  return nullptr;
}
// the hash table of zk_assign_state_circuit_mpt: a power of two >= 2 n slots (at most half full), at least 64
static u64 state_mpt_slots(u64 n) {
  u64 cap = 64;
  while (cap < 2 * n) cap <<= 1;
  return cap;
}

#ifdef __CUDACC__
__global__ void __launch_bounds__(256) k_seg_local(SegHorner s, Fr* chunk_val) {
  const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < s.n_chunks) seg_local(s, chunk_val, c);
}
__global__ void __launch_bounds__(128) k_seg_carry(SegHorner s, Fr* chunk_val, Fr* seg_total) {
  const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < s.n_seg) seg_carry(s, chunk_val, seg_total, k);
}
__global__ void __launch_bounds__(256) k_assign_bytecode_rlc(const __grid_constant__ BytecodeAssign a, const Fr* chunk_val) {
  const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < a.s.n_chunks) assign_bytecode_rlc(a, chunk_val, c);
}
__global__ void __launch_bounds__(256) k_assign_bytecode_rows(const __grid_constant__ BytecodeAssign a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += stride) assign_bytecode_row(a, r);
}
__global__ void __launch_bounds__(256) k_assign_state_derive(const __grid_constant__ StateAssign a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += stride) assign_state_row(a, r);
}
__global__ void __launch_bounds__(256) k_assign_copy_rows(const __grid_constant__ CopyAssign a, const Fr* chunk_val, const Fr* seg_total) {
  const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < a.s.n_chunks) assign_copy_chunk(a, chunk_val, seg_total, c);
}
__global__ void __launch_bounds__(128) k_assign_exp_chain(const __grid_constant__ ExpAssign a) {
  const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < a.n_events) assign_exp_chain(a, k);
}
// persistent grid (api.cu grid_persistent): threads walk the rows with a grid stride
__global__ void __launch_bounds__(256) k_assign_exp_rows(const __grid_constant__ ExpAssign a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += stride) assign_exp_row(a, r);
}

// ---- public-inputs circuit
__global__ void __launch_bounds__(256) k_assign_pi_seq(const __grid_constant__ PiAssign a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += stride) assign_pi_seq(a, r);
}
__global__ void __launch_bounds__(256) k_assign_pi_inv(const __grid_constant__ PiAssign a) {
  const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < a.n_inv) assign_pi_inv(a, k);
}
// the digest: one thread runs the sponge over all of seq (about n / 136 permutations)
__global__ void __launch_bounds__(32) k_assign_pi_sponge(const __grid_constant__ PiAssign a) {
  if (threadIdx.x == 0) keccak256(a.seq, a.n, a.dig);
}
// exclusive scan of the values of a block (Hillis-Steele in shared memory); sh[blockDim.x - 1] is left holding the
// block's combined value
template <class S>
__device__ __forceinline__ typename S::T pi_block_excl(const S& s, typename S::T x, typename S::T* sh) {
  sh[threadIdx.x] = x;
  __syncthreads();
  for (u32 d = 1; d < blockDim.x; d <<= 1) {
    const typename S::T y = threadIdx.x >= d ? S::op(sh[threadIdx.x - d], sh[threadIdx.x]) : sh[threadIdx.x];
    __syncthreads();
    sh[threadIdx.x] = y;
    __syncthreads();
  }
  return threadIdx.x ? sh[threadIdx.x - 1] : s.id();
}
// level 1: each thread folds PI_SCAN_GROUP 32-byte chunks; x[c] = the value carried into chunk c from the earlier chunks
// of its block, top[b] = block b's total
template <class S>
__global__ void __launch_bounds__(256) k_assign_pi_scan(const __grid_constant__ S s, typename S::T* x, typename S::T* top) {
  __shared__ typename S::T sh[256];
  const u64 n_chunks = (s.n + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK;
  const u64 c0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) * PI_SCAN_GROUP;
  const typename S::T v = c0 < n_chunks ? s.fold(c0 * ZK_SEG_CHUNK, zk_min64((c0 + PI_SCAN_GROUP) * ZK_SEG_CHUNK, s.n)) : s.id();
  typename S::T carry = pi_block_excl(s, v, sh);
  if (threadIdx.x == 0) top[blockIdx.x] = sh[blockDim.x - 1];
  for (u64 c = c0; c < c0 + PI_SCAN_GROUP && c < n_chunks; c++) {
    x[c] = carry;
    carry = S::op(carry, s.fold(c * ZK_SEG_CHUNK, zk_min64((c + 1) * ZK_SEG_CHUNK, s.n)));
  }
}
// level 2, one block: top[b] becomes the value carried into block b (each thread walks a contiguous run of totals)
template <class S>
__global__ void __launch_bounds__(256) k_assign_pi_scan_top(const __grid_constant__ S s, u64 n_blocks, typename S::T* top) {
  __shared__ typename S::T sh[256];
  const u64 per = (n_blocks + blockDim.x - 1) / blockDim.x;
  const u64 b0 = zk_min64(threadIdx.x * per, n_blocks), b1 = zk_min64(b0 + per, n_blocks);
  typename S::T v = s.id();
  for (u64 b = b0; b < b1; b++) v = S::op(v, top[b]);
  typename S::T carry = pi_block_excl(s, v, sh);
  for (u64 b = b0; b < b1; b++) {
    const typename S::T t = top[b];
    top[b] = carry;
    carry = S::op(carry, t);
  }
}
__global__ void __launch_bounds__(256) k_assign_pi_krlc(const __grid_constant__ PiAssign a) {
  const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < (a.n + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK) assign_pi_krlc(a, c);
}
__global__ void __launch_bounds__(256) k_assign_pi_calldata(const __grid_constant__ PiAssign a) {
  const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < (a.max_cd + ZK_SEG_CHUNK - 1) / ZK_SEG_CHUNK) assign_pi_calldata(a, c);
}
__global__ void __launch_bounds__(256) k_assign_pi_rows(const __grid_constant__ PiAssign a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += stride) assign_pi_row(a, r);
}
__global__ void __launch_bounds__(32) k_assign_pi_finish(const __grid_constant__ PiAssign a) {
  if (threadIdx.x == 0) assign_pi_finish(a);
}

// ---- tx table
// zero call-data bytes per tx, one thread per byte on a persistent grid: the lanes of a warp that hold bytes of the same
// tx add their zero bytes with one atomic, so a tx of 2^20 bytes costs 2^15 atomics, not one thread walking it
__global__ void __launch_bounds__(256) k_assign_tx_zeros(const __grid_constant__ TxTableAssign a) {
  const u32 lane = threadIdx.x & 31;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; w < a.n_cd; w += stride) {  // warp-uniform
    const u64 j = w + lane;
    const bool in = j < a.n_cd;
    const u64 k = in ? tx_of_byte(a, j) : ~0ull;
    const u32 zero = __ballot_sync(~0u, in && a.cd[j] == 0);
    const u32 same = __match_any_sync(~0u, k);
    if (in && lane == (u32)__ffs(same) - 1 && (zero & same)) atomicAdd(a.zeros + k, (unsigned long long)__popc(zero & same));
  }
}
__global__ void __launch_bounds__(256) k_assign_tx_rows(const __grid_constant__ TxTableAssign a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += stride) assign_tx_row(a, r);
}

// ---- copy table
// per tile of CT_TILE circuit rows: its is_first rows, the smallest row failing an assert, the total
__global__ void __launch_bounds__(256) k_copy_table_count(const __grid_constant__ CopyTableAssign a) {
  __shared__ u32 cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  u32 mine = 0;
#pragma unroll
  for (int q = 0; q < CT_TILE / 256; q++) {
    const u64 i = (u64)blockIdx.x * CT_TILE + q * 256 + threadIdx.x;
    if (copy_row_is_first(a, i)) {
      mine++;
      if (copy_row_fails(a, i)) atomicMin(a.fail, (unsigned long long)i);
    }
  }
  for (int o = 16; o; o >>= 1) mine += __shfl_down_sync(~0u, mine, o);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) {
    a.tile_count[blockIdx.x] = cnt;
    if (cnt) atomicAdd(a.fail + 1, (unsigned long long)cnt);
  }
}
// after the exclusive scan of the tile counts: each tile's is_first rows, in circuit order, from its offset
__global__ void __launch_bounds__(256) k_copy_table_write(const __grid_constant__ CopyTableAssign a) {
  __shared__ u32 warp_n[8];
  const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64 pos = a.tile_count[blockIdx.x];
  for (int q = 0; q < CT_TILE / 256; q++) {
    const u64 i = (u64)blockIdx.x * CT_TILE + q * 256 + threadIdx.x;
    const bool f = copy_row_is_first(a, i);
    const u32 b = __ballot_sync(~0u, f);
    if (lane == 0) warp_n[warp] = __popc(b);
    __syncthreads();
    u32 before = 0, total = 0;
#pragma unroll
    for (u32 v = 0; v < 8; v++) {
      const u32 n = warp_n[v];
      before += v < warp ? n : 0;
      total += n;
    }
    if (f) copy_table_row(a, i, pos + before + __popc(b & ((1u << lane) - 1)));
    pos += total;
    __syncthreads();
  }
}

// ---- state circuit roots + MPT table (persistent grids, grid stride)
__global__ void __launch_bounds__(256) k_state_mpt_insert(const __grid_constant__ StateMpt a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) state_mpt_insert(a, i);
}
// first touches, the first failing op (one atomic per failing op: a rejected input), and the two totals with one
// atomic per warp
__global__ void __launch_bounds__(256) k_state_mpt_first(const __grid_constant__ StateMpt a) {
  const u32 lane = threadIdx.x & 31;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; w < a.n; w += stride) {  // warp-uniform
    const u64 i = w + lane;
    unsigned f = 0, fail = 0;
    if (i < a.n) f = state_mpt_first(a, i, &fail);
    if (fail) atomicMin(a.stat, (unsigned long long)((i << 2) | fail));
    const u32 upd = __ballot_sync(~0u, f & 2), mpt = __ballot_sync(~0u, f & 1);
    if (lane == 0) {
      if (upd) atomicAdd(a.stat + 1, (unsigned long long)__popc(upd));
      if (mpt) atomicAdd(a.stat + 2, (unsigned long long)__popc(mpt));
    }
  }
}
__global__ void __launch_bounds__(256) k_state_mpt_compact(const __grid_constant__ StateMpt a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) state_mpt_compact(a, i);
}
__global__ void __launch_bounds__(256) k_state_mpt_rows(const __grid_constant__ StateMpt a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < a.n; k += stride) state_mpt_row_root(a, k);
}
__global__ void __launch_bounds__(256) k_state_mpt_table(const __grid_constant__ StateMpt a) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 u = (u64)blockIdx.x * blockDim.x + threadIdx.x; u < a.n_upd; u += stride) state_mpt_table_row(a, u);
}
#endif

}  // namespace zk
