// words.cuh — 256-bit words as (lo, hi) 128-bit field cells and the mul_add_words gate.
//
// Device-side counterpart of Word (src/zkevm_specs/util/arithmetic.py:99-168) and of
// mul_add_words (util/arithmetic.py:245-276, evm_circuit/instruction.py:599-632), shared by the
// MUL/DIV/MOD gate program (evm.cu), the exp circuit (exp.cu) and its row builder (assign.cu).
#pragma once
#include "fr.cuh"

namespace zk {

// 2^-128 in Montgomery form (= 2^128): montmul(x, this) == x / 2^128 mod p
#define ZK_MONT_INV2_128 Fr{{0x0ull, 0x0ull, 0x1ull, 0x0ull}}

struct Word2 {
  Fr lo, hi;
};
ZK_HD bool word_in_domain(const Word2& w) { return fr_fits128(w.lo) && fr_fits128(w.hi); }
ZK_HD bool word_eq(const Word2& a, const Word2& b) {
  return fr_eq(a.lo, b.lo) && fr_eq(a.hi, b.hi);
}

// exact small unsigned integers (< 2^196) as Fr: sums of 64x64-bit limb products, optionally
// shifted left by one limb (the "* 2^64" of mul_add_words)
ZK_HD void acc_add_mul(Fr& acc, u64 a, u64 b, int shift_limbs) {
  const unsigned __int128 v = (unsigned __int128)a * b;
  u64 c = 0;
  const u64 lo = (u64)v, hi = (u64)(v >> 64);
  if (shift_limbs == 0) {
    acc.l[0] = adc64(acc.l[0], lo, c);
    acc.l[1] = adc64(acc.l[1], hi, c);
    acc.l[2] = adc64(acc.l[2], 0, c);
    acc.l[3] += c;
  } else {
    acc.l[1] = adc64(acc.l[1], lo, c);
    acc.l[2] = adc64(acc.l[2], hi, c);
    acc.l[3] += c;
  }
}

// mul_add_words(a, b, c, d): t0..t3 from 64-bit limbs, carries = (...) / 2^128 IN THE FIELD, overflow
// term.  Requires a, b in the 128-bit-halves domain (to_64s); c, d are arbitrary cells.  The two
// constrain_equal of the reference hold by construction of the carries; what can fail are the
// 9-byte range checks of the carries, left to the caller.
ZK_HD void mul_add_carries(const Word2& a, const Word2& b, const Word2& c, const Word2& d, Fr* carry_lo, Fr* carry_hi,
                           Fr* overflow) {
  const u64 a0 = a.lo.l[0], a1 = a.lo.l[1], a2 = a.hi.l[0], a3 = a.hi.l[1];
  const u64 b0 = b.lo.l[0], b1 = b.lo.l[1], b2 = b.hi.l[0], b3 = b.hi.l[1];
  Fr lo_part = fr_u64(0), hi_part = fr_u64(0), ovf = fr_u64(0);  // exact integers < 2^195 < p
  acc_add_mul(lo_part, a0, b0, 0);
  acc_add_mul(lo_part, a0, b1, 1);
  acc_add_mul(lo_part, a1, b0, 1);
  acc_add_mul(hi_part, a0, b2, 0);
  acc_add_mul(hi_part, a1, b1, 0);
  acc_add_mul(hi_part, a2, b0, 0);
  acc_add_mul(hi_part, a0, b3, 1);
  acc_add_mul(hi_part, a1, b2, 1);
  acc_add_mul(hi_part, a2, b1, 1);
  acc_add_mul(hi_part, a3, b0, 1);
  acc_add_mul(ovf, a1, b3, 0);
  acc_add_mul(ovf, a2, b2, 0);
  acc_add_mul(ovf, a3, b1, 0);
  acc_add_mul(ovf, a2, b3, 0);
  acc_add_mul(ovf, a3, b2, 0);
  acc_add_mul(ovf, a3, b3, 0);
  *carry_lo = fr_montmul(fr_sub(fr_add(lo_part, c.lo), d.lo), ZK_MONT_INV2_128);
  *carry_hi = fr_montmul(fr_sub(fr_add(fr_add(hi_part, c.hi), *carry_lo), d.hi), ZK_MONT_INV2_128);
  *overflow = fr_add(*carry_hi, ovf);
}
// range_check(x, 9): x.n fits 9 bytes
ZK_HD bool fits_9_bytes(const Fr& x) { return fr_fits128(x) && (x.l[1] >> 8) == 0; }

// low 256 bits of a * b (4 little-endian limbs): the MUL gate's fast form (evm.cu) and the exp circuit's
// square-and-multiply chain (assign.cu)
ZK_HD void mul256_lo(const u64 a[4], const u64 b[4], u64 o[4]) {
  u64 t[4] = {0, 0, 0, 0};
#pragma unroll
  for (int x = 0; x < 4; x++) {
    u64 c = 0;
#pragma unroll
    for (int y = 0; y + x < 4; y++) {
      unsigned __int128 v = (unsigned __int128)a[x] * b[y] + t[x + y] + c;
      t[x + y] = (u64)v;
      c = (u64)(v >> 64);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; k++) o[k] = t[k];
}

}  // namespace zk
