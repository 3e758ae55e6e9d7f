// zq_common.cuh -- shared device helpers and descriptors for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

#define ZQ_FULL 0xffffffffu

// One compression unit (== one libzpaq::compressBlock call, Z:20255) as the kernels see it.
struct ZqUnit {
  u64 in_off;    // byte offset of the input in the device input arena
  u64 work_off;  // byte offset of this unit's sa | isa | lcp region in the per-wave work arena
  u64 lz_off;    // byte offset into the pre-pass stream buffer
  u64 model_off; // byte offset of this unit's component tables + VM memory in the model arena
  u64 coded_off; // byte offset of the arithmetic coder's output
  u32 n;         // input length
  u32 plan;      // index into the plan table
  u32 lz_cap;    // capacity reserved at lz_off
  u32 prefix_off, prefix_len;  // block prefix (tag .. segment header) in the blob
  u32 idx16;     // 1: sa/isa stored as u16 (n <= 65536), 0: u32
  u32 coded_cap; // capacity reserved at coded_off
  u32 want_pk;   // 1: the suffix sort also writes the packed rows the LZ77 scan kernels read (work region sized by zq_work_bytes_scan)
};

// Per (method, block size class) constants (== makeConfig's args, Z:19620-19628).
struct ZqPlan {
  int args[9];
  u32 payload_off, payload_len;  // selector + PCOMP bytes that precede the stream, in the blob
  u32 lz_level;                  // 0 none, 1 var-length codes, 2 byte codes, 3 BWT
  u32 use_sa;
  u32 e8e9;
  u32 modeled;                   // ncomp > 0
  u32 cm_plan;                   // index into the ZqCmPlan table when modeled
  u32 pad;
};

// per-unit work region: sa | isa (index width w = 2 or 4) | lcp (u16) | bwt (u8), each padded to 128 B
__host__ __device__ inline u64 zq_work_stride(u32 n, u32 w) { return (((u64)n + 1) * w + 127) & ~(u64)127; }
__host__ __device__ inline u64 zq_work_bytes(u32 n, u32 w) { return 2 * zq_work_stride(n, w) + zq_work_stride(n, 2) + zq_work_stride(n, 1); }

// The LZ77 scan pipeline (zq_lz77_scan.cuh) keeps three more arrays behind them: pk (one packed word per SA row:
// suffix start | LCP with the row above saturated at 255 | BWT byte; 4 bytes for 16-bit indices, 8 otherwise; padded so
// that whole 64-row groups can be bulk-copied), r0[n+1] and f[n][2].
__host__ __device__ inline u64 zq_align128(u64 x) { return (x + 127) & ~(u64)127; }
__host__ __device__ inline u64 zq_pk_bytes(u32 n, u32 w) { return zq_align128((((u64)n + 63) & ~(u64)63) * (w == 2 ? 4 : 8)); }
__host__ __device__ inline u64 zq_work_bytes_scan(u32 n, u32 w) {
  return zq_work_bytes(n, w) + zq_pk_bytes(n, w) + zq_align128(((u64)n + 1) * (w == 2 ? 4 : 8)) + zq_align128((u64)n * (w == 2 ? 8 : 16));
}

__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }
#ifdef ZQ_EMU   // host SIMT emulator build (tests/emu): no PTX, dynamic shared memory is a plain pointer
__device__ __forceinline__ u32 lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }
#define ZQ_DYN_SMEM(name) unsigned char* name = emu::dyn_smem
#else
__device__ __forceinline__ u32 lanemask_lt() {
  u32 m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}
#define ZQ_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif
// floor(log2(x))+1, 0 for 0 (== reference lg(), Z:19269)
__device__ __forceinline__ int zq_bitlen(u32 x) { return 32 - __clz(x); }

// ---- bulk async copies (TMA, cp.async.bulk) + mbarrier -------------------------------------------------------
// One elected thread arms the barrier with the byte count and issues the copies; everyone waits on the phase
// parity.  Addresses and sizes must be multiples of 16 bytes.  Under the host emulator the copy is a memcpy and
// the barrier a phase counter, so the kernels' control flow is identical.
#ifdef ZQ_EMU
struct ZqMbar { u32 phase; u32 pending; };
__device__ __forceinline__ void zq_mbar_init(ZqMbar* b, u32) { b->phase = 0; b->pending = 0; }
__device__ __forceinline__ void zq_mbar_expect_tx(ZqMbar* b, u32 bytes) { b->pending += bytes; if (b->pending == 0) ++b->phase; }
__device__ __forceinline__ void zq_bulk_g2s(void* dst, const void* src, u32 bytes, ZqMbar* b) {
  if (((uintptr_t)dst | (uintptr_t)src | bytes) & 15) { fprintf(stderr, "emu: misaligned bulk copy\n"); abort(); }
  memcpy(dst, src, bytes);
  b->pending -= bytes;
  if (b->pending == 0) ++b->phase;
}
__device__ __forceinline__ void zq_mbar_wait(ZqMbar* b, u32 parity) { while ((b->phase & 1u) == parity) emu::yield(); }
__device__ __forceinline__ bool zq_mbar_test(ZqMbar* b, u32 parity) { return (b->phase & 1u) != parity; }
__device__ __forceinline__ void zq_bulk_s2g(void* dst, const void* src, u32 bytes) {
  if (((uintptr_t)dst | (uintptr_t)src | bytes) & 15) { fprintf(stderr, "emu: misaligned bulk store\n"); abort(); }
  memcpy(dst, src, bytes);
}
__device__ __forceinline__ void zq_bulk_commit_wait() {}
__device__ __forceinline__ void zq_fence_async_smem() {}
#else
typedef u64 ZqMbar;
__device__ __forceinline__ u32 zq_smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void zq_mbar_init(ZqMbar* b, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(zq_smem_addr(b)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void zq_mbar_expect_tx(ZqMbar* b, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(zq_smem_addr(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void zq_bulk_g2s(void* dst, const void* src, u32 bytes, ZqMbar* b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(zq_smem_addr(dst)), "l"(src), "r"(bytes), "r"(zq_smem_addr(b)) : "memory");
}
__device__ __forceinline__ void zq_mbar_wait(ZqMbar* b, u32 parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "ZQ_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra ZQ_DONE;\n"
      "bra ZQ_WAIT;\n"
      "ZQ_DONE:\n"
      "}" ::"r"(zq_smem_addr(b)), "r"(parity) : "memory");
}
// has the phase with this parity completed?  (non-blocking: safe inside divergent code)
__device__ __forceinline__ bool zq_mbar_test(ZqMbar* b, u32 parity) {
  u32 ok;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}" : "=r"(ok) : "r"(zq_smem_addr(b)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void zq_bulk_s2g(void* dst, const void* src, u32 bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(zq_smem_addr(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void zq_bulk_commit_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (before a bulk store reads them)
__device__ __forceinline__ void zq_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif
