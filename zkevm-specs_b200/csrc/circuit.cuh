// circuit.cuh — shared kernel-side plumbing: resident witness matrices and row addressing.
#pragma once
#include "lookup.cuh"

namespace zk {

#define ZK_MAX_COLS 64
struct WitnessDev {
  const unsigned char* base;   // column c: n_rows integers of width[c] bytes at base + off[c]
  u64 n_rows;                  // resident rows (incl. halos when sharded)
  const unsigned char* flags;  // optional per-row type flags
  u64 off[ZK_MAX_COLS];
  unsigned char width[ZK_MAX_COLS];  // 0 (constant column), 1, 2, 4, 8, 16 or 32 (fr.cuh:ld_col)
};

struct CheckRange {
  u64 row_begin, row_end;  // local rows to check
  u64 row_base;            // reported row = row_base + local
  u32 flags;               // ZK_FLAG_*
};

ZK_HD Fr wcell(const WitnessDev& w, u32 col, u64 row) {
  return ld_col(w.base + w.off[col], w.width[col], row);
}
// Storage layout a row-checker instance is compiled for.  L_CANON: every column holds canonical 32-byte
// cells (zk_upload_columns) — a cell load is one address add + two LDG.128; L_ANY: per-column widths
// (packed uploads) through the generic branch-free loader, ~20 more instructions per load.  The host
// picks the instance from the resident matrix's widths; results are identical.
enum { L_ANY = 0, L_CANON = 1 };
template <int LAYOUT>
ZK_HD Fr wcell_l(const WitnessDev& w, u32 col, u64 row) {
  if (LAYOUT == L_CANON) return ld_cell((const u64*)(w.base + w.off[col]) + row * 4);
  return ld_col(w.base + w.off[col], w.width[col], row);
}
template <int LAYOUT>
ZK_HD Fr tcell_l(const TableDev& t, u32 col, u64 row) {
  if (LAYOUT == L_CANON) return ld_cell((const u64*)(t.base + t.off[col]) + row * 4);
  return ld_col(t.base + t.off[col], t.width[col], row);
}
// rotation by +k / -k: wraps modulo n_rows when the whole circuit is resident, otherwise the
// caller supplied halo rows (include/zkcheck.h)
ZK_HD u64 rot_fwd(const WitnessDev& w, u64 row, u32 k, bool wrap) {
  u64 j = row + k;
  if (j >= w.n_rows) j = wrap ? j % w.n_rows : w.n_rows - 1;
  return j;
}
ZK_HD u64 rot_back(const WitnessDev& w, u64 row, bool wrap) {
  return row ? row - 1 : (wrap ? w.n_rows - 1 : 0);
}

#ifdef __CUDACC__
// (Two alternatives for the canonical row checkers were built and dropped: a 4-deep TMA tile pipeline with
// one 128-thread CTA per SM made the gate program itself the bound (few warps active, low issue rate);
// prefetch.global.L2 of the thread's next row cost more issue slots than it hid latency.)
// Stage a small read-only table into shared memory with ONE bulk asynchronous copy
// (cp.async.bulk, the 1-D TMA path: SASS UBLKCP) completing on an mbarrier.  Called by every
// thread of the block; returns when the bytes are visible to all of them.  `bytes` must be a
// multiple of 16 and both addresses 16-byte aligned.
__device__ __forceinline__ void stage_to_smem(void* smem_dst, const void* gmem_src, u32 bytes, u64* bar) {
  const u32 bar_a = (u32)__cvta_generic_to_shared(bar);
  const u32 dst_a = (u32)__cvta_generic_to_shared(smem_dst);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a),
        "l"(gmem_src), "r"(bytes), "r"(bar_a)
        : "memory");
  }
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "ZK_STAGE_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
      "@!p bra ZK_STAGE_WAIT;\n\t"
      "}" ::"r"(bar_a)
      : "memory");
}
#endif

}  // namespace zk
