// fr.cuh — BN254 scalar-field cells on the device (sm_90a).
//
// Device-side counterpart of the reference's FQ (src/zkevm_specs/util/arithmetic.py:41-63,
// arithmetic in py_ecc.bn128.FQ).  A cell is 4 little-endian uint64 limbs holding the
// CANONICAL value (< p); witness matrices stay canonical in HBM because most reference
// checks compare the integer `.n` (ranges, `FQ == int`, `<`).  Montgomery form is used
// only inside true Fr x Fr products: montmul(a, bR) = a*b mod p, so keeping the constant
// operand (challenge powers, 2^-128, ...) in Montgomery form costs one multiply per product
// and no conversions.
#pragma once
#include <stdint.h>

namespace zk {

typedef unsigned long long u64;
typedef unsigned int u32;

struct Fr {
  u64 l[4];
};

#define ZK_P0 0x43e1f593f0000001ull
#define ZK_P1 0x2833e84879b97091ull
#define ZK_P2 0xb85045b68181585dull
#define ZK_P3 0x30644e72e131a029ull
#define ZK_N0 0xc2e1f593efffffffull  // -p^-1 mod 2^64
// R^2 mod p, R = 2^256
#define ZK_R2_0 0x1bb8e645ae216da7ull
#define ZK_R2_1 0x53fe3ab1e35c59e3ull
#define ZK_R2_2 0x8c49833d53bb8085ull
#define ZK_R2_3 0x0216d0b17f4e44a5ull
// 2^64 in Montgomery form (2^64 * 2^256 mod p)
#define ZK_MONT_TWO64 Fr{{0xb4c6edf97c5fb586ull, 0x708c8d50bfeb93beull, 0x9ffd1de404f7e0efull, 0x215b02ac9a392866ull}}

// A 32-byte cell is two independent 128-bit loads (LDG.E.128, the widest global load sm_90a has),
// issued back to back; a warp reading 32 consecutive rows of a column moves 1 KiB in two
// instructions.  .nc: witness/table cells are read-only.
// (The host branch exists only so that tests/emu can run the SAME gate programs on the CPU
// for local debugging before a GPU call; the product never executes it.)
#define ZK_HD __host__ __device__ __forceinline__
#define ZK_HD_NOINLINE __host__ __device__ __noinline__
ZK_HD Fr ld_cell(const u64* p) {
  Fr r;
#ifdef __CUDA_ARCH__
  asm volatile(
      "ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
      "ld.global.nc.v2.u64 {%2,%3}, [%4+16];"
      : "=l"(r.l[0]), "=l"(r.l[1]), "=l"(r.l[2]), "=l"(r.l[3])
      : "l"(p));
#else
  r.l[0] = p[0]; r.l[1] = p[1]; r.l[2] = p[2]; r.l[3] = p[3];
#endif
  return r;
}
// Columns are stored at their own width (include/zkcheck.h, "packed columns"): a column whose
// values all fit w bytes is kept as n_rows little-endian w-byte integers, w in {1,2,4,8,16,32};
// w = 0 is a constant column (one 32-byte cell).  Byte-, flag- and counter-valued columns are
// most of every table, so a warp reading 32 consecutive rows of such a column touches 1-8
// sectors instead of 32, and the stored tables shrink ~5x (the 17.8 M-row bytecode table of
// the bench: 3.4 GB -> 0.70 GB).  The branch is uniform: the width is a per-column constant.
// Device form is BRANCH-FREE (three predicated loads, one executes): with branches the compiler
// cannot batch a thread's independent cell loads ahead of the compares, and the gate programs are
// latency-bound on exactly that.  Widths <= 8 load the aligned 8-byte
// word that contains the value (a w-byte integer at a multiple of w never straddles one; columns
// start at multiples of 32 and are padded to 32) and shift/mask it out.
ZK_HD Fr ld_col(const unsigned char* p, u32 width, u64 row) {
  Fr r;
#ifdef __CUDA_ARCH__
  r.l[0] = r.l[1] = r.l[2] = r.l[3] = 0;
  const u32 lw = width ? width : 32u;  // constant column: stride 0, one 32-byte cell
  const u64 a = (u64)p + row * width;
  asm volatile(
      "{\n\t"
      ".reg .pred pa, pb, pc;\n\t"
      "setp.le.u32 pa, %5, 8;\n\t"
      "setp.eq.u32 pb, %5, 16;\n\t"
      "setp.eq.u32 pc, %5, 32;\n\t"
      "@pa ld.global.nc.u64 %0, [%6];\n\t"
      "@pb ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
      "@pc ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
      "@pc ld.global.nc.v2.u64 {%2,%3}, [%4+16];\n\t"
      "}"
      : "+l"(r.l[0]), "+l"(r.l[1]), "+l"(r.l[2]), "+l"(r.l[3])
      : "l"(a), "r"(lw), "l"(a & ~7ull));
  const bool narrow = lw <= 8;
  const u32 sh = narrow ? ((u32)a & 7u) * 8u : 0u;
  const u64 m = lw >= 8 ? ~0ull : ((1ull << (8u * lw)) - 1ull);
  r.l[0] = (r.l[0] >> sh) & m;
#else
  if (width == 32) return ld_cell((const u64*)p + row * 4);
  r.l[1] = r.l[2] = r.l[3] = 0;
  switch (width) {
    case 1: r.l[0] = p[row]; break;
    case 2: r.l[0] = ((const unsigned short*)p)[row]; break;
    case 4: r.l[0] = ((const u32*)p)[row]; break;
    case 8: r.l[0] = ((const u64*)p)[row]; break;
    case 16: r.l[0] = ((const u64*)p)[2 * row]; r.l[1] = ((const u64*)p)[2 * row + 1]; break;
    default: return ld_cell((const u64*)p);  // 0: constant column
  }
#endif
  return r;
}
// ld_col for a column the HOST has verified to be "narrow": stored in at most 8 bytes per row, or a constant below 2^64
// (api.cu: Matrix::narrow_mask).  One aligned 8-byte load, shift, mask — and limbs 1..3 are literal zeros, so the
// 4-limb compares / adds of the gate programs fold to one limb in kernels specialised for narrow step / key columns.
ZK_HD Fr ld_col_narrow(const unsigned char* p, u32 width, u64 row) {
  Fr r;
  r.l[1] = r.l[2] = r.l[3] = 0;
#ifdef __CUDA_ARCH__
  // rows of a resident matrix are below 2^32 (the sorted step lists and the table indexes hold 32-bit rows), so the
  // address is one 32 x 32 -> 64-bit multiply-add; width 0 = the constant cell itself (stride 0, mask of 8 bytes)
  const u64 a = (u64)p + (u64)(u32)row * width;
  const u64 v = __ldg((const u64*)(a & ~7ull));
  const u32 sh = ((u32)a & 7u) << 3;
  const u32 w8 = width ? width : 8u;
  r.l[0] = (v >> sh) & (~0ull >> (64u - 8u * w8));
#else
  switch (width) {
    case 1: r.l[0] = p[row]; break;
    case 2: r.l[0] = ((const unsigned short*)p)[row]; break;
    case 4: r.l[0] = ((const u32*)p)[row]; break;
    case 8: r.l[0] = ((const u64*)p)[row]; break;
    default: r.l[0] = ((const u64*)p)[0]; break;  // 0: constant column
  }
#endif
  return r;
}
// ld_col with the width known at compile time: one plain typed load (kernels that are
// specialised for a storage layout, e.g. k_pos_verify over the type-width bytecode table)
template <int W>
ZK_HD Fr ld_col_c(const unsigned char* p, u64 row) {
  Fr r;
  r.l[0] = r.l[1] = r.l[2] = r.l[3] = 0;
#ifdef __CUDA_ARCH__
  if constexpr (W == 32) return ld_cell((const u64*)p + row * 4);
  else if constexpr (W == 16) {
    const ulonglong2 v = __ldg((const ulonglong2*)p + row);
    r.l[0] = v.x;
    r.l[1] = v.y;
  } else if constexpr (W == 8) r.l[0] = __ldg((const u64*)p + row);
  else if constexpr (W == 4) r.l[0] = __ldg((const u32*)p + row);
  else if constexpr (W == 2) r.l[0] = __ldg((const unsigned short*)p + row);
  else if constexpr (W == 1) r.l[0] = __ldg(p + row);
  else return ld_cell((const u64*)p);
  return r;
#else
  return ld_col(p, (u32)W, row);
#endif
}
ZK_HD u32 ld_u32(const u32* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
ZK_HD u64 ld_u64(const u64* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
ZK_HD u64 ld_volatile_u64(const u64* p) { return *(const volatile u64*)p; }  // written earlier in the same stream
ZK_HD u64 atomic_cas_u64(u64* p, u64 expect, u64 val) {
#ifdef __CUDA_ARCH__
  return atomicCAS(p, expect, val);
#else
  const u64 old = *p;
  if (old == expect) *p = val;
  return old;
#endif
}
ZK_HD u32 atomic_add_u32(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
  return atomicAdd(p, v);
#else
  const u32 old = *p;
  *p += v;
  return old;
#endif
}
ZK_HD void atomic_min_u32(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
  atomicMin(p, v);
#else
  if (v < *p) *p = v;
#endif
}
ZK_HD void atomic_add_u64(u64* p, u64 v) {
#ifdef __CUDA_ARCH__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}

__host__ __device__ __forceinline__ Fr fr_u64(u64 v) { return Fr{{v, 0, 0, 0}}; }
__host__ __device__ __forceinline__ Fr fr_u128(u64 lo, u64 hi) { return Fr{{lo, hi, 0, 0}}; }
__host__ __device__ __forceinline__ bool fr_eq(const Fr& a, const Fr& b) {
  return ((a.l[0] ^ b.l[0]) | (a.l[1] ^ b.l[1]) | (a.l[2] ^ b.l[2]) | (a.l[3] ^ b.l[3])) == 0;
}
__host__ __device__ __forceinline__ bool fr_is_zero(const Fr& a) {
  return (a.l[0] | a.l[1] | a.l[2] | a.l[3]) == 0;
}
// FQ == int (py_ecc compares .n with the raw int)
__host__ __device__ __forceinline__ bool fr_eq_u64(const Fr& a, u64 v) {
  return a.l[0] == v && (a.l[1] | a.l[2] | a.l[3]) == 0;
}
// .n fits in 64 / 128 bits
__host__ __device__ __forceinline__ bool fr_fits64(const Fr& a) { return (a.l[1] | a.l[2] | a.l[3]) == 0; }
__host__ __device__ __forceinline__ bool fr_fits128(const Fr& a) { return (a.l[2] | a.l[3]) == 0; }
// integer compare of .n
__host__ __device__ __forceinline__ bool fr_lt(const Fr& a, const Fr& b) {
  if (a.l[3] != b.l[3]) return a.l[3] < b.l[3];
  if (a.l[2] != b.l[2]) return a.l[2] < b.l[2];
  if (a.l[1] != b.l[1]) return a.l[1] < b.l[1];
  return a.l[0] < b.l[0];
}

__host__ __device__ __forceinline__ u64 adc64(u64 a, u64 b, u64& c) {
  unsigned __int128 t = (unsigned __int128)a + b + c;
  c = (u64)(t >> 64);
  return (u64)t;
}
__host__ __device__ __forceinline__ u64 sbb64(u64 a, u64 b, u64& br) {
  unsigned __int128 t = (unsigned __int128)a - b - br;
  br = (u64)(t >> 64) & 1;
  return (u64)t;
}
// s - p if s >= p (s < 2^255)
__host__ __device__ __forceinline__ Fr fr_sub_p_if_ge(const Fr& s) {
  Fr d;
#ifdef __CUDA_ARCH__
  u64 br;
  asm("sub.cc.u64 %0, %5, %9;\n\t"
      "subc.cc.u64 %1, %6, %10;\n\t"
      "subc.cc.u64 %2, %7, %11;\n\t"
      "subc.cc.u64 %3, %8, %12;\n\t"
      "subc.u64 %4, 0, 0;"
      : "=l"(d.l[0]), "=l"(d.l[1]), "=l"(d.l[2]), "=l"(d.l[3]), "=l"(br)
      : "l"(s.l[0]), "l"(s.l[1]), "l"(s.l[2]), "l"(s.l[3]), "l"(ZK_P0), "l"(ZK_P1), "l"(ZK_P2), "l"(ZK_P3));
  return br ? s : d;
#else
  u64 br = 0;
  d.l[0] = sbb64(s.l[0], ZK_P0, br);
  d.l[1] = sbb64(s.l[1], ZK_P1, br);
  d.l[2] = sbb64(s.l[2], ZK_P2, br);
  d.l[3] = sbb64(s.l[3], ZK_P3, br);
  return br ? s : d;
#endif
}
// (a + b) mod p for canonical a, b  (a+b < 2p < 2^255: no carry out)
__host__ __device__ __forceinline__ Fr fr_add(const Fr& a, const Fr& b) {
  Fr s;
#ifdef __CUDA_ARCH__
  asm("add.cc.u64 %0, %4, %8;\n\t"
      "addc.cc.u64 %1, %5, %9;\n\t"
      "addc.cc.u64 %2, %6, %10;\n\t"
      "addc.u64 %3, %7, %11;"
      : "=l"(s.l[0]), "=l"(s.l[1]), "=l"(s.l[2]), "=l"(s.l[3])
      : "l"(a.l[0]), "l"(a.l[1]), "l"(a.l[2]), "l"(a.l[3]), "l"(b.l[0]), "l"(b.l[1]), "l"(b.l[2]), "l"(b.l[3]));
#else
  u64 c = 0;
  s.l[0] = adc64(a.l[0], b.l[0], c);
  s.l[1] = adc64(a.l[1], b.l[1], c);
  s.l[2] = adc64(a.l[2], b.l[2], c);
  s.l[3] = adc64(a.l[3], b.l[3], c);
#endif
  return fr_sub_p_if_ge(s);
}
__host__ __device__ __forceinline__ Fr fr_sub(const Fr& a, const Fr& b) {
  Fr d;
#ifdef __CUDA_ARCH__
  u64 br;
  asm("sub.cc.u64 %0, %5, %9;\n\t"
      "subc.cc.u64 %1, %6, %10;\n\t"
      "subc.cc.u64 %2, %7, %11;\n\t"
      "subc.cc.u64 %3, %8, %12;\n\t"
      "subc.u64 %4, 0, 0;"
      : "=l"(d.l[0]), "=l"(d.l[1]), "=l"(d.l[2]), "=l"(d.l[3]), "=l"(br)
      : "l"(a.l[0]), "l"(a.l[1]), "l"(a.l[2]), "l"(a.l[3]), "l"(b.l[0]), "l"(b.l[1]), "l"(b.l[2]), "l"(b.l[3]));
  // br is all-ones on borrow: add back p & br
  asm("add.cc.u64 %0, %0, %4;\n\t"
      "addc.cc.u64 %1, %1, %5;\n\t"
      "addc.cc.u64 %2, %2, %6;\n\t"
      "addc.u64 %3, %3, %7;"
      : "+l"(d.l[0]), "+l"(d.l[1]), "+l"(d.l[2]), "+l"(d.l[3])
      : "l"(ZK_P0 & br), "l"(ZK_P1 & br), "l"(ZK_P2 & br), "l"(ZK_P3 & br));
#else
  u64 br = 0;
  d.l[0] = sbb64(a.l[0], b.l[0], br);
  d.l[1] = sbb64(a.l[1], b.l[1], br);
  d.l[2] = sbb64(a.l[2], b.l[2], br);
  d.l[3] = sbb64(a.l[3], b.l[3], br);
  if (br) {
    u64 c = 0;
    d.l[0] = adc64(d.l[0], ZK_P0, c);
    d.l[1] = adc64(d.l[1], ZK_P1, c);
    d.l[2] = adc64(d.l[2], ZK_P2, c);
    d.l[3] = adc64(d.l[3], ZK_P3, c);
  }
#endif
  return d;
}
__host__ __device__ __forceinline__ Fr fr_add_u64(const Fr& a, u64 v) { return fr_add(a, fr_u64(v)); }
__host__ __device__ __forceinline__ Fr fr_sub_u64(const Fr& a, u64 v) { return fr_sub(a, fr_u64(v)); }

// Montgomery product a*b*2^-256 mod p (CIOS, 4x64-bit limbs; result canonical).
__host__ __device__ __forceinline__ Fr fr_montmul(const Fr& a, const Fr& b) {
  const u64 P[4] = {ZK_P0, ZK_P1, ZK_P2, ZK_P3};
  u64 t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const u64 bi = b.l[i];
    unsigned __int128 x;
    u64 c;
    x = (unsigned __int128)a.l[0] * bi + t0; t0 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)a.l[1] * bi + t1 + c; t1 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)a.l[2] * bi + t2 + c; t2 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)a.l[3] * bi + t3 + c; t3 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)t4 + c; t4 = (u64)x;
    u64 t5 = (u64)(x >> 64);
    const u64 m = t0 * ZK_N0;
    x = (unsigned __int128)m * P[0] + t0; c = (u64)(x >> 64);
    x = (unsigned __int128)m * P[1] + t1 + c; t0 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)m * P[2] + t2 + c; t1 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)m * P[3] + t3 + c; t2 = (u64)x; c = (u64)(x >> 64);
    x = (unsigned __int128)t4 + c; t3 = (u64)x; t4 = t5 + (u64)(x >> 64);
  }
  Fr r{{t0, t1, t2, t3}};
  // p < 2^254 and inputs < p  =>  result < 2p, t4 == 0
  return fr_sub_p_if_ge(r);
}
// One-limb Montgomery product: v * b * 2^-64 mod p for a 64-bit v (canonical result).  With
// b = C * 2^64 mod p this is v * C mod p at a quarter of the cost of fr_montmul — most lookup
// key cells (tags, counters, indices, addresses) fit one limb.
__host__ __device__ __forceinline__ Fr fr_montmul1(u64 v, const Fr& b) {
  unsigned __int128 x;
  u64 c, t0, t1, t2, t3, t4;
  x = (unsigned __int128)v * b.l[0]; t0 = (u64)x; c = (u64)(x >> 64);
  x = (unsigned __int128)v * b.l[1] + c; t1 = (u64)x; c = (u64)(x >> 64);
  x = (unsigned __int128)v * b.l[2] + c; t2 = (u64)x; c = (u64)(x >> 64);
  x = (unsigned __int128)v * b.l[3] + c; t3 = (u64)x; t4 = (u64)(x >> 64);
  const u64 m = t0 * ZK_N0;
  x = (unsigned __int128)m * ZK_P0 + t0; c = (u64)(x >> 64);
  x = (unsigned __int128)m * ZK_P1 + t1 + c; t0 = (u64)x; c = (u64)(x >> 64);
  x = (unsigned __int128)m * ZK_P2 + t2 + c; t1 = (u64)x; c = (u64)(x >> 64);
  x = (unsigned __int128)m * ZK_P3 + t3 + c; t2 = (u64)x; c = (u64)(x >> 64);
  t3 = t4 + c;  // (v*b + m*p) / 2^64 < 2p < 2^255
  return fr_sub_p_if_ge(Fr{{t0, t1, t2, t3}});
}
__host__ __device__ __forceinline__ Fr fr_to_mont(const Fr& a) {
  return fr_montmul(a, Fr{{ZK_R2_0, ZK_R2_1, ZK_R2_2, ZK_R2_3}});
}
// canonical product of two canonical cells
__host__ __device__ __forceinline__ Fr fr_mul(const Fr& a, const Fr& b) {
  return fr_montmul(fr_to_mont(a), b);
}
// a (canonical, fits 64 bits) times small constant-free u64, exact integer if it fits,
// else mod p: used for cheap "x * 256^k"-style terms
__host__ __device__ __forceinline__ Fr fr_shl_small(u64 v, int bits) {  // v * 2^bits, bits<192, as integer (< p guaranteed by caller)
  Fr r{{0, 0, 0, 0}};
  int w = bits >> 6, s = bits & 63;
  r.l[w] = v << s;
  if (s && w + 1 < 4) r.l[w + 1] = v >> (64 - s);
  return r;
}

}  // namespace zk
