// zq_cm.cuh -- the ZPAQ context-mixing compressor (methods -m3/-m4/-m5 and any explicit model of
// <= 32 components): HCOMP virtual machine, component chain, logistic mixing and the binary
// arithmetic coder.  (A first engine -- one warp per block with the interpreter inline -- was 2-3x slower and is gone;
// its numbers are in profiles/README.md, r01_configs vs r01i.)
//
// Replaces (bit-exactly): ZPAQL::run0/execute Z:14232-14467, Predictor::predict0 Z:15041,
// update0 Z:15139, find Z:15254, train Z:13161, Encoder::encode/compress Z:15557-15589.
//
// Mapping.  Coding is a strict per-bit recurrence, so a block cannot be split along its bytes; what
// can be separated is the block's two machines:
//   * the CONTEXT machine (HCOMP, run once per byte) only ever looks at bytes that are already known
//     to the compressor, so in the encoder it runs AHEAD of the coder on its own warp and hands the
//     context hashes H[0..n) of each byte to the coder through a small shared-memory ring.  While it
//     is there it also prefetches, for the byte the coder will reach a few bytes later, the hash rows
//     / table lines every component is going to touch (their addresses depend on H and on the byte).
//   * the CODER warp: LANE i = COMPONENT i.  Per bit all lanes gather from their own tables at once
//     (hash row -> bit history -> adaptive probability; mixer weights are fetched in the same phase,
//     their row does not depend on the predictions); ISSE chains / MIX2 / SSE / AVG are resolved in
//     host-computed dependency levels with shuffles; each MIX is one multiply per input lane and one
//     REDUX add.  ICM/ISSE 16-byte hash rows are cached in shared memory for the four bits of a nibble.
// One (coder, context) warp pair per block; a CTA holds up to 12 pairs next to the 78 KB of
// model-independent tables (stretch, squash, dt, state table).  The decoder cannot run the context
// machine ahead (the byte is only known once decoded): there one warp does both, machine on lane 0.
// ncu of the first engine (profiles/r01h_cm_*): 2 800 (-m3) to 14 500 (-m5) dependent warp
// instructions per byte at IPC 0.1/warp, 30-60 % of them in the byte-code interpreter -- latency of
// the instruction stream, not memory, was the limit; hence the flat-switch interpreter on shared-memory
// byte code, the shared-memory row cache and the overlap of the two machines.
#pragma once
#include "zq_cm_types.h"
#include "zq_common.cuh"

namespace zqdev {

struct CmTablesDev {      // device mirror of zq::CmTables (same field order)
  int16_t stretch[32768];
  u16 squash[4096];
  int dt[1024];
  int dt2k[256];
  u8 ns[1024];
  u32 icm_init[256];
  u32 isse_init[512];
};
struct CmSmem {           // what the coder needs per bit
  int16_t stretch[32768];
  u16 squash[4096];
  int dt[1024];
  int dt2k[256];
  u8 ns[1024];
};

#define ZQ_CM_RING 8          // context vectors in flight between the two warps of a pair
#define ZQ_CM_CODE_CAP 1024   // HCOMP byte code staged to shared memory up to this size
#define ZQ_CM_HBUF 512        // H[] lives in shared memory up to 2^9 words (every built-in model)
struct CmUnitSmem {           // shared-memory working set of one block in flight
  u32 ring[ZQ_CM_RING][32];   // H[lane] after byte k, slot k % ZQ_CM_RING
  u8 rows[32][16];            // lane's current ICM/ISSE hash row
  u32 hbuf[ZQ_CM_HBUF];
  u8 code[ZQ_CM_CODE_CAP];
  volatile u32 produced, consumed;   // context vectors written / taken
  volatile int unit;
  u32 pad;
};

#ifdef ZQ_EMU
__device__ __forceinline__ void zq_pair_sync(u32 id) { emu::barrier((int)id, 64); }
__device__ __forceinline__ void zq_prefetch_l1(const void*) {}
__device__ __forceinline__ void zq_prefetch_l2(const void*) {}
#else
__device__ __forceinline__ void zq_pair_sync(u32 id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void zq_prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ void zq_prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#endif

// ---- model initialisation ------------------------------------------------------------------------
// One CTA writes one fill job (a table's initial values, Z:14968-15032) of one unit's model region.
__device__ __forceinline__ void cm_fill_job(const ZqCmFill f, const CmTablesDev* __restrict__ tab, u8* __restrict__ region) {
  u8* __restrict__ dst = region + f.off;
  const u64 nq = f.bytes >> 4;  // regions are 256 B aligned; tails shorter than 16 B are written bytewise
  uint4* __restrict__ d4 = (uint4*)dst;
  if (f.kind == ZQ_FILL_ZERO || f.kind == ZQ_FILL_U32 || f.kind == ZQ_FILL_U16 || f.kind == ZQ_FILL_MATCHBUF) {
    u32 v = f.kind == ZQ_FILL_U32 ? f.value : f.kind == ZQ_FILL_U16 ? (f.value | f.value << 16) : 0u;
    const uint4 q = make_uint4(v, v, v, v);
    for (u64 k = threadIdx.x; k < nq; k += blockDim.x) d4[k] = q;
    for (u64 k = (nq << 4) + threadIdx.x; k < f.bytes; k += blockDim.x) dst[k] = (u8)(v >> (8 * (k & 3)));
    if (f.kind == ZQ_FILL_MATCHBUF) { __syncthreads(); if (threadIdx.x == 0) dst[0] = 1; }
  } else if (f.kind == ZQ_FILL_SSE) {
    // cm[j] = squash((j&31)*64-992)<<17 | start : period of 32 entries = 8 uint4
    for (u64 k = threadIdx.x; k < nq; k += blockDim.x) {
      const u32 e = (u32)(k & 7) * 4;
      uint4 q;
      q.x = (u32)tab->squash[(e + 0) * 64 - 992 + 2048] << 17 | f.value;
      q.y = (u32)tab->squash[(e + 1) * 64 - 992 + 2048] << 17 | f.value;
      q.z = (u32)tab->squash[(e + 2) * 64 - 992 + 2048] << 17 | f.value;
      q.w = (u32)tab->squash[(e + 3) * 64 - 992 + 2048] << 17 | f.value;
      d4[k] = q;
    }
  } else {
    const u32* src = f.kind == ZQ_FILL_ICM ? tab->icm_init : tab->isse_init;
    u32* d = (u32*)dst;
    for (u32 k = threadIdx.x; k < f.bytes / 4; k += blockDim.x) d[k] = src[k];
  }
}

// grid.x = units in the wave * fill jobs of the largest plan
__global__ void __launch_bounds__(256)
k_cm_init(const ZqUnit* __restrict__ units, const ZqPlan* __restrict__ plans, const ZqCmPlan* __restrict__ cmplans,
          const ZqCmFill* __restrict__ fills, const int* __restrict__ todo, int ntodo, int maxjobs,
          const CmTablesDev* __restrict__ tab, u8* __restrict__ model_base) {
  const int t = blockIdx.x / maxjobs, j = blockIdx.x % maxjobs;
  if (t >= ntodo) return;
  const ZqUnit u = units[todo[t]];
  const ZqCmPlan& cp = cmplans[plans[u.plan].cm_plan];
  if (j >= (int)cp.fill_count) return;
  cm_fill_job(fills[cp.fill_first + j], tab, model_base + u.model_off);
}
// same, for explicit (model offset, plan) pairs (decoder)
__global__ void __launch_bounds__(256)
k_cm_init_pairs(const u64* __restrict__ model_off, const u32* __restrict__ plan_of, const ZqCmPlan* __restrict__ cmplans,
                const ZqCmFill* __restrict__ fills, int n, int maxjobs, const CmTablesDev* __restrict__ tab, u8* __restrict__ model_base) {
  const int t = blockIdx.x / maxjobs, j = blockIdx.x % maxjobs;
  if (t >= n) return;
  const ZqCmPlan& cp = cmplans[plan_of[t]];
  if (j >= (int)cp.fill_count) return;
  cm_fill_job(fills[cp.fill_first + j], tab, model_base + model_off[t]);
}

// ---- per-warp coder state ------------------------------------------------------------------------
struct CmCoder {
  u32 low, high;
  u8* out; u8* end; u32 overflow;
  __device__ __forceinline__ void init(u8* o, u32 cap) { low = 1; high = 0xffffffffu; out = o; end = o + cap; overflow = 0; }
  __device__ __forceinline__ void encode(int y, u32 p16) {   // Encoder::encode, Z:15557
    const u32 mid = low + (u32)(((u64)(high - low) * p16) >> 16);
    if (y) high = mid; else low = mid + 1;
    while ((high ^ low) < 0x1000000u) {
      if (out < end) { if (lane_id() == 0) *out = (u8)(high >> 24); } else overflow = 1;
      ++out;
      high = high << 8 | 255;
      low = low << 8;
      low += (low == 0);
    }
  }
};

// ---- ZPAQL machine -------------------------------------------------------------------------------
struct CmVm {   // registers live on the lane that owns the machine (lane 0)
  u32 a, b, c, d; int f;
  u8* m; u32* h; u32* r;
  u32 mmask, hmask;
  const u8* code; int len;
  int error;
};
struct VmOut { u8* out; u32 len, cap, error; };   // PCOMP's OUT sink (decoder)

// One run of the program (ZPAQL::run0, Z:14232) by ONE lane: a single switch over the opcode byte, the two-operand group
// (opcode >= 64: operation = op>>3, source = op&7) expanded case by case.  nvcc lowers it to a nine-level compare/branch
// tree over 25 KB of code: ncu (profiles/r01j) puts ~290 of the ~380 cycles per ZPAQL instruction there -- which is why
// the small models get their program translated and compiled instead (zq_jit.cpp).  (The template parameter VM of the
// kernels is kept for the emulator tests' signatures; every value runs this interpreter.)
#define ZQ_VM_X8(B, STMT)                                                  \
  case (B) + 0: { const u32 x = a; STMT; } break;                          \
  case (B) + 1: { const u32 x = b; STMT; } break;                          \
  case (B) + 2: { const u32 x = c; STMT; } break;                          \
  case (B) + 3: { const u32 x = d; STMT; } break;                          \
  case (B) + 4: { const u32 x = M[b & mm]; STMT; } break;                  \
  case (B) + 5: { const u32 x = M[c & mm]; STMT; } break;                  \
  case (B) + 6: { const u32 x = H[d & hm]; STMT; } break;                  \
  case (B) + 7: { const u32 x = P[pc++]; STMT; } break;
template <bool WITH_OUT>
__device__ void cm_vm_run_switch(CmVm& v, u32 input, VmOut* o) {
  const u8* P = v.code;
  u8* M = v.m; u32* H = v.h; u32* R = v.r;
  const u32 mm = v.mmask, hm = v.hmask;
  const int len = v.len;
  int pc = 0, stop = 0;
  int budget = 1 << 24;   // instructions per run: a program that loops forever (the reference would hang) ends as a ZPAQL error
  u32 a = input, b = v.b, c = v.c, d = v.d; int f = v.f;
  while (!stop) {
    if ((u32)pc >= (u32)len || --budget < 0) { stop = 2; break; }
    const u32 op = P[pc++];
    switch (op) {
      case 1: ++a; break; case 2: --a; break; case 3: a = ~a; break; case 4: a = 0; break;
      case 7: a = R[P[pc++]]; break;
      case 8: { const u32 t = a; a = b; b = t; } break;
      case 9: ++b; break; case 10: --b; break; case 11: b = ~b; break; case 12: b = 0; break;
      case 15: b = R[P[pc++]]; break;
      case 16: { const u32 t = a; a = c; c = t; } break;
      case 17: ++c; break; case 18: --c; break; case 19: c = ~c; break; case 20: c = 0; break;
      case 23: c = R[P[pc++]]; break;
      case 24: { const u32 t = a; a = d; d = t; } break;
      case 25: ++d; break; case 26: --d; break; case 27: d = ~d; break; case 28: d = 0; break;
      case 31: d = R[P[pc++]]; break;
      case 32: { const u32 t = M[b & mm]; M[b & mm] = (u8)a; a = (a & ~255u) | t; } break;
      case 33: M[b & mm] = (u8)(M[b & mm] + 1); break; case 34: M[b & mm] = (u8)(M[b & mm] - 1); break;
      case 35: M[b & mm] = (u8)~M[b & mm]; break; case 36: M[b & mm] = 0; break;
      case 39: if (f) pc += (int)((P[pc] + 128u) & 255u) - 127; else ++pc; break;
      case 40: { const u32 t = M[c & mm]; M[c & mm] = (u8)a; a = (a & ~255u) | t; } break;
      case 41: M[c & mm] = (u8)(M[c & mm] + 1); break; case 42: M[c & mm] = (u8)(M[c & mm] - 1); break;
      case 43: M[c & mm] = (u8)~M[c & mm]; break; case 44: M[c & mm] = 0; break;
      case 47: if (!f) pc += (int)((P[pc] + 128u) & 255u) - 127; else ++pc; break;
      case 48: { const u32 t = H[d & hm]; H[d & hm] = a; a = t; } break;
      case 49: H[d & hm] = H[d & hm] + 1; break; case 50: H[d & hm] = H[d & hm] - 1; break;
      case 51: H[d & hm] = ~H[d & hm]; break; case 52: H[d & hm] = 0; break;
      case 55: R[P[pc++]] = a; break;
      case 56: stop = 1; break;
      case 57:
        if (WITH_OUT) { if (o->len < o->cap) o->out[o->len] = (u8)a; else o->error = 3; ++o->len; }
        break;
      case 59: a = (a + M[b & mm] + 512u) * 773u; break;
      case 60: H[d & hm] = (H[d & hm] + a + 512u) * 773u; break;
      case 63: pc += (int)((P[pc] + 128u) & 255u) - 127; break;
      ZQ_VM_X8(64, a = x) ZQ_VM_X8(72, b = x) ZQ_VM_X8(80, c = x) ZQ_VM_X8(88, d = x)
      ZQ_VM_X8(96, M[b & mm] = (u8)x) ZQ_VM_X8(104, M[c & mm] = (u8)x) ZQ_VM_X8(112, H[d & hm] = x)
      ZQ_VM_X8(128, a += x) ZQ_VM_X8(136, a -= x) ZQ_VM_X8(144, a *= x)
      ZQ_VM_X8(152, a = x ? a / x : 0u) ZQ_VM_X8(160, a = x ? a % x : 0u)
      ZQ_VM_X8(168, a &= x) ZQ_VM_X8(176, a &= ~x) ZQ_VM_X8(184, a |= x) ZQ_VM_X8(192, a ^= x)
      ZQ_VM_X8(200, a <<= (x & 31u)) ZQ_VM_X8(208, a >>= (x & 31u))
      ZQ_VM_X8(216, f = a == x) ZQ_VM_X8(224, f = a < x) ZQ_VM_X8(232, f = a > x)
      case 255: pc = (int)P[pc] + 256 * (int)P[pc + 1]; break;
      default: stop = 2;
    }
  }
  if (stop == 2) v.error = 1;
  v.a = a; v.b = b; v.c = c; v.d = d; v.f = f;
}
#undef ZQ_VM_X8

// (two branch-free forms of this interpreter -- arithmetic selects, with and without predicated loads -- were slower
//  than the switch on BWT blocks and were removed)
template <int VM, bool WITH_OUT>
__device__ __forceinline__ void cm_vm_run(CmVm& v, u32 input, VmOut* o) { cm_vm_run_switch<WITH_OUT>(v, input, o); }

__device__ __forceinline__ int cm_clamp2k(int x) { return min(max(x, -2048), 2047); }
__device__ __forceinline__ int cm_clamp512k(int x) { return min(max(x, -(1 << 19)), (1 << 19) - 1); }

// Everything one lane knows about its component.
struct CmLane {
  u32 type, level;
  u32 a2, a3, a4, a5;    // descriptor bytes cp[2..5]
  u32 in1, in2;          // lanes of the inputs (AVG j,k / MIX2 j,k / ISSE j / SSE j)
  u32* cm; u8* ht; u32 cm_mask, ht_mask;
  u32 chkshift;          // ICM/ISSE: a1 + 2
  u32 h;                 // context hash H[i]
  int p;                 // stretched prediction of this component
  u32 cxt, limit, ca, cb, cc;
  u32 pn;                // table entry fetched for predict (trained in update)
  int w0, w1, pj, pk;    // ISSE weights / MIX2 weight in w0; inputs seen at predict time
  u32 rowpos, rowok;     // where the cached hash row came from
  u8* row;               // this lane's 16 B row cache in shared memory
  int* wp0; int* wp1;    // this lane's weight column in the first / second MIX it feeds (else null)
  int wv0, wv1;          // those weights for the current bit
  u32 mr0, mr1;          // and their row offsets
  u32 mixinfo;           // MIX lanes: j0 | m << 8 | rate << 16
};

// Predictor::find (Z:15254) on this lane's hash table + switch of the shared-memory cached row.
// The three candidate rows share one 64-byte block, fetched whole in one round trip.
__device__ __forceinline__ void cm_row_switch(CmLane& L, u32 cxt) {
  uint4* rc = (uint4*)L.row;
  if (L.rowok) *(uint4*)(L.ht + L.rowpos) = *rc;
  const u32 chk = (cxt >> L.chkshift) & 255u;
  const u32 h0 = (cxt * 16u) & (L.ht_mask - 15u), h1 = h0 ^ 16u, h2 = h0 ^ 32u;
  const uint4 r0 = *(const uint4*)(L.ht + h0), r1 = *(const uint4*)(L.ht + h1), r2 = *(const uint4*)(L.ht + h2);
  u32 r; uint4 row;
  if ((r0.x & 255u) == chk) { r = h0; row = r0; }
  else if ((r1.x & 255u) == chk) { r = h1; row = r1; }
  else if ((r2.x & 255u) == chk) { r = h2; row = r2; }
  else {
    const u32 p0 = (r0.x >> 8) & 255u, p1 = (r1.x >> 8) & 255u, p2 = (r2.x >> 8) & 255u;
    if (p0 <= p1 && p0 <= p2) r = h0; else if (p1 < p2) r = h1; else r = h2;
    row = make_uint4(chk, 0, 0, 0);
  }
  *rc = row;
  L.rowpos = r; L.rowok = 1;
}

struct CmCtx {             // warp-uniform per-block state
  int n, nlevels, c8, hmap4;
  u32 mix_mask;            // lanes that are MIX components
  u32 mix_levels;          // bit L: some MIX sits at dependency level L
  u32 other_levels;        // bit L: an AVG, MIX2 or SSE sits at level L (ISSE links need no flag)
  int mix0, mix1;          // lanes of the first two MIX components (-1: none)
};

// p for the next bit: Predictor::predict0 (Z:15041)
__device__ int cm_predict(CmLane& L, const CmCtx& X, const CmSmem& T) {
  const u32 lane = lane_id();
  const int c8 = X.c8, hmap4 = X.hmap4;
  const bool nib = c8 == 1 || (c8 & 0xf0) == 16;
  // phase 1: every table fetch whose address does not depend on another component's prediction
  const bool hashed = L.type == ZQ_ICM || L.type == ZQ_ISSE;   // one pass over the hash rows for both kinds
  if (hashed) {
    if (nib) cm_row_switch(L, L.h + 16u * (u32)c8);
    L.cxt = L.row[hmap4 & 15];
  }
  switch (L.type) {
    case ZQ_CM:
      L.cxt = (L.h ^ (u32)hmap4) & L.cm_mask;
      L.pn = L.cm[L.cxt];
      L.p = T.stretch[L.pn >> 17];
      break;
    case ZQ_ICM:
      L.pn = L.cm[L.cxt];
      L.p = T.stretch[L.pn >> 8];
      break;
    case ZQ_ISSE: {
      const int2 w = *(const int2*)(L.cm + L.cxt * 2);
      L.w0 = w.x; L.w1 = w.y;
      break;
    }
    case ZQ_MATCH:
      if (L.ca == 0) L.p = 0;
      else {
        L.cc = (L.ht[(L.limit - L.cb) & L.ht_mask] >> (7 - L.cxt)) & 1u;
        L.p = T.stretch[(T.dt2k[L.ca] * (L.cc ? -1 : 1)) & 32767];
      }
      break;
    case ZQ_MIX2:
      L.cxt = (L.h + ((u32)c8 & L.a5)) & L.cm_mask;
      L.w0 = ((const u16*)L.cm)[L.cxt];
      break;
    case ZQ_MIX:
      L.cxt = ((L.h + ((u32)c8 & L.a5)) & L.cm_mask) * L.a3;   // first weight of this bit's row
      break;
    case ZQ_SSE:
      zq_prefetch_l1(L.cm + (((L.h + (u32)c8) * 32u) & L.cm_mask));   // the bit's 32-bucket row = one 128 B line
      break;
    default: break;
  }
  if (X.mix0 >= 0) { L.mr0 = __shfl_sync(ZQ_FULL, L.cxt, X.mix0); if (L.wp0) L.wv0 = L.wp0[L.mr0]; }
  if (X.mix1 >= 0) { L.mr1 = __shfl_sync(ZQ_FULL, L.cxt, X.mix1); if (L.wp1) L.wv1 = L.wp1[L.mr1]; }
  // phase 2: dependency levels.  ISSE links are by far the most common inner node (chains of up to 7 in the
  // built-in models): they are evaluated as predicated arithmetic by every lane, no branch; AVG / MIX2 / SSE only
  // run at the levels the host flagged for them.
  const bool isse = L.type == ZQ_ISSE;
  for (int lev = 1; lev < X.nlevels; ++lev) {
    const int pj = __shfl_sync(ZQ_FULL, L.p, L.in1);
    const int pi = cm_clamp2k((L.w0 * pj + L.w1 * 64) >> 16);
    if (isse && (int)L.level == lev) { L.pj = pj; L.p = pi; }
    if ((X.other_levels >> lev) & 1u) {
      const int pk = __shfl_sync(ZQ_FULL, L.p, L.in2);
      if ((int)L.level == lev) {
        switch (L.type) {
          case ZQ_AVG: L.p = (pj * (int)L.a3 + pk * (256 - (int)L.a3)) >> 8; break;
          case ZQ_MIX2: L.pj = pj; L.pk = pk; L.p = (L.w0 * pj + (65536 - L.w0) * pk) >> 16; break;
          case ZQ_SSE: {
            u32 cx = (L.h + (u32)c8) * 32u;
            int pq = min(max(pj + 992, 0), 1983);
            const int wt = pq & 63;
            pq >>= 6;
            cx += (u32)pq;
            const u32 e0 = L.cm[cx & L.cm_mask], e1 = L.cm[(cx + 1) & L.cm_mask];
            L.p = T.stretch[((e0 >> 10) * (u32)(64 - wt) + (e1 >> 10) * (u32)wt) >> 13];
            cx += (u32)(wt >> 5);
            L.cxt = cx & L.cm_mask;
            L.pn = (wt >> 5) ? e1 : e0;
            break;
          }
          default: break;
        }
      }
    }
    // mixers of this level: every input lane multiplies its own p by its weight, one REDUX sums
    u32 mm = ((X.mix_levels >> lev) & 1u) ? __ballot_sync(ZQ_FULL, L.type == ZQ_MIX && (int)L.level == lev) : 0u;
    while (mm) {
      const int xl = __ffs(mm) - 1;
      mm &= mm - 1;
      int term = 0;
      if (xl == X.mix0) { if (L.wp0) term = (L.wv0 >> 8) * L.p; }
      else if (xl == X.mix1) { if (L.wp1) term = (L.wv1 >> 8) * L.p; }
      else {   // third and later mixers of a model: weight fetched here
        const u32 info = __shfl_sync(ZQ_FULL, L.mixinfo, xl), row = __shfl_sync(ZQ_FULL, L.cxt, xl);
        const u64 base = __shfl_sync(ZQ_FULL, (u64)(uintptr_t)L.cm, xl);
        const u32 j0 = info & 255u, m = (info >> 8) & 255u;
        if (lane >= j0 && lane < j0 + m) term = (((const int*)(uintptr_t)base)[row + lane - j0] >> 8) * L.p;
      }
      const int sum = __reduce_add_sync(ZQ_FULL, term);
      if ((int)lane == xl) L.p = cm_clamp2k(sum >> 8);
    }
  }
  return T.squash[__shfl_sync(ZQ_FULL, L.p, X.n - 1) + 2048];
}

// train all components on bit y and advance the bit context; Predictor::update0 (Z:15139).
// Returns true when a byte was completed (the context machine's output for it is due).
__device__ bool cm_update(CmLane& L, CmCtx& X, const CmSmem& T, int y) {
  const u32 lane = lane_id();
  // mixers first need every lane's p as seen at predict time: p is unchanged until the next predict
  u32 mm = X.mix_mask;
  while (mm) {
    const int xl = __ffs(mm) - 1;
    mm &= mm - 1;
    const int pX = __shfl_sync(ZQ_FULL, L.p, xl);
    const u32 info = __shfl_sync(ZQ_FULL, L.mixinfo, xl);
    const int err = ((y * 32767 - (int)T.squash[pX + 2048]) * (int)(info >> 16)) >> 4;
    if (xl == X.mix0) { if (L.wp0) L.wp0[L.mr0] = cm_clamp512k(L.wv0 + ((err * L.p + (1 << 12)) >> 13)); }
    else if (xl == X.mix1) { if (L.wp1) L.wp1[L.mr1] = cm_clamp512k(L.wv1 + ((err * L.p + (1 << 12)) >> 13)); }
    else {
      const u32 row = __shfl_sync(ZQ_FULL, L.cxt, xl);
      const u64 base = __shfl_sync(ZQ_FULL, (u64)(uintptr_t)L.cm, xl);
      const u32 j0 = info & 255u, m = (info >> 8) & 255u;
      if (lane >= j0 && lane < j0 + m) {
        int* wp = (int*)(uintptr_t)base + row + lane - j0;
        *wp = cm_clamp512k(*wp + ((err * L.p + (1 << 12)) >> 13));
      }
    }
  }
  if (L.type == ZQ_ICM || L.type == ZQ_ISSE) L.row[X.hmap4 & 15] = T.ns[L.cxt * 4 + y];   // next bit history
  switch (L.type) {
    case ZQ_CM: case ZQ_SSE: {
      const u32 count = L.pn & 0x3ffu;
      const int error = y * 32767 - (int)(L.pn >> 17);
      L.pn += (u32)((error * T.dt[count]) & -1024) + (count < L.limit ? 1u : 0u);
      L.cm[L.cxt] = L.pn;
      break;
    }
    case ZQ_ICM: {
      L.pn += (u32)(((int)(y * 32767 - (int)(L.pn >> 8))) >> 2);
      L.cm[L.cxt] = L.pn;
      break;
    }
    case ZQ_ISSE: {
      const int err = y * 32767 - (int)T.squash[L.p + 2048];
      int2 w;
      w.x = cm_clamp512k(L.w0 + ((err * L.pj + (1 << 12)) >> 13));
      w.y = cm_clamp512k(L.w1 + ((err + 16) >> 5));
      *(int2*)(L.cm + L.cxt * 2) = w;
      break;
    }
    case ZQ_MIX2: {
      const int err = ((y * 32767 - (int)T.squash[L.p + 2048]) * (int)L.a4) >> 5;
      int w = L.w0 + ((err * (L.pj - L.pk) + (1 << 12)) >> 13);
      w = min(max(w, 0), 65535);
      ((u16*)L.cm)[L.cxt] = (u16)w;
      break;
    }
    case ZQ_MATCH: {
      // The reference shifts y into ht[limit] bit by bit; the partial byte is never read (matches and the
      // predicted bit look at earlier positions), so the finished byte is stored once.
      const u32 hm = L.ht_mask;
      if ((int)L.cc != y) L.ca = 0;
      if (++L.cxt == 8) {
        L.ht[L.limit & hm] = (u8)(X.c8 * 2 + y);
        L.cxt = 0;
        L.limit = (L.limit + 1) & hm;
        if (L.ca == 0) {
          L.cb = L.limit - L.cm[L.h & L.cm_mask];
          if (L.cb & hm)
            while (L.ca < 255 && L.ht[(L.limit - L.ca - 1) & hm] == L.ht[(L.limit - L.ca - L.cb - 1) & hm]) ++L.ca;
        } else L.ca += L.ca < 255;
        L.cm[L.h & L.cm_mask] = L.limit;
      }
      break;
    }
    default: break;
  }
  X.c8 += X.c8 + y;
  if (X.c8 >= 256) { X.hmap4 = 1; X.c8 = 1; return true; }
  if (X.c8 >= 16 && X.c8 < 32) X.hmap4 = (X.hmap4 & 0xf) << 5 | y << 4 | 1;
  else X.hmap4 = (X.hmap4 & 0x1f0) | (((X.hmap4 & 0xf) * 2 + y) & 0xf);
  return false;
}

}  // namespace zqdev
#include "zq_cm_wide.cuh"
namespace zqdev {

// Lane state for a block: component `lane` of plan `cp`, tables in `model`, row cache in `S`.
__device__ __forceinline__ void cm_setup(CmLane& L, CmCtx& X, const ZqCmPlan& cp, u8* model, CmUnitSmem& S) {
  const u32 lane = lane_id();
  X.n = cp.n; X.nlevels = cp.nlevels; X.c8 = 1; X.hmap4 = 1; X.mix_mask = cp.mix_mask;
  const bool act = lane < (u32)cp.n;
  const ZqCmComp c = cp.comp[act ? lane : 0];
  L.type = act ? c.type : 0; L.level = act ? c.level : 255;
  L.a2 = c.a2; L.a3 = c.a3; L.a4 = c.a4; L.a5 = c.a5;
  X.mix_levels = __reduce_or_sync(ZQ_FULL, (act && c.type == ZQ_MIX) ? (1u << c.level) : 0u);
  X.other_levels = __reduce_or_sync(ZQ_FULL, (act && (c.type == ZQ_AVG || c.type == ZQ_MIX2 || c.type == ZQ_SSE)) ? (1u << c.level) : 0u);
  L.cm = (u32*)(model + c.cm_off); L.ht = model + c.ht_off; L.cm_mask = c.cm_mask; L.ht_mask = c.ht_mask;
  L.chkshift = (u32)c.a1 + 2;
  L.in1 = 0; L.in2 = 0;
  if (L.type == ZQ_AVG) { L.in1 = c.a1; L.in2 = c.a2; }
  else if (L.type == ZQ_MIX2) { L.in1 = c.a2; L.in2 = c.a3; }
  else if (L.type == ZQ_ISSE || L.type == ZQ_SSE) L.in1 = c.a2;
  L.h = 0; L.p = L.type == ZQ_CONS ? ((int)c.a1 - 128) * 4 : 0;
  L.cxt = 0; L.ca = L.cb = L.cc = 0; L.pn = 0; L.w0 = L.w1 = L.pj = L.pk = 0;
  L.limit = L.type == ZQ_CM ? c.a2 * 4u : L.type == ZQ_SSE ? c.a4 * 4u : L.type == ZQ_ICM ? 1023u : 0u;
  L.rowpos = 0; L.rowok = 0; L.row = S.rows[lane];
  L.mixinfo = (u32)c.a2 | (u32)c.a3 << 8 | (u32)c.a4 << 16;
  // the first two mixers keep their weights in registers between predict and update
  X.mix0 = X.mix_mask ? __ffs(X.mix_mask) - 1 : -1;
  const u32 rest = X.mix_mask & (X.mix_mask - 1);
  X.mix1 = rest ? __ffs(rest) - 1 : -1;
  L.wp0 = nullptr; L.wp1 = nullptr; L.wv0 = L.wv1 = 0; L.mr0 = L.mr1 = 0;
  if (X.mix0 >= 0) {
    const ZqCmComp& m0 = cp.comp[X.mix0];
    if (lane >= m0.a2 && lane < (u32)m0.a2 + m0.a3) L.wp0 = (int*)(model + m0.cm_off) + (lane - m0.a2);
  }
  if (X.mix1 >= 0) {
    const ZqCmComp& m1 = cp.comp[X.mix1];
    if (lane >= m1.a2 && lane < (u32)m1.a2 + m1.a3) L.wp1 = (int*)(model + m1.cm_off) + (lane - m1.a2);
  }
}

// Context machine of a block: memory M, R in the model region; H in shared memory when it fits.
__device__ __forceinline__ void cm_vm_setup(CmVm& vm, const ZqCmPlan& cp, u8* model, const u8* blob, CmUnitSmem& S) {
  const u32 lane = lane_id();
  vm.a = vm.b = vm.c = vm.d = 0; vm.f = 0; vm.error = 0;
  vm.m = model + cp.m_off; vm.r = (u32*)(model + cp.r_off);
  vm.mmask = (1u << cp.hm) - 1; vm.hmask = (1u << cp.hh) - 1;
  if ((1u << cp.hh) <= ZQ_CM_HBUF) {
    vm.h = S.hbuf;
    for (u32 k = lane; k < (1u << cp.hh); k += 32) S.hbuf[k] = 0;
  } else vm.h = (u32*)(model + cp.h_off);
  vm.len = (int)cp.hcomp_len;
  if (cp.hcomp_len < ZQ_CM_CODE_CAP) {   // strictly: the interpreter reads the byte after an opcode
    for (u32 k = lane; k < cp.hcomp_len; k += 32) S.code[k] = blob[cp.hcomp_off + k];
    vm.code = S.code;
  } else vm.code = blob + cp.hcomp_off;
  __syncwarp();
}

// The context warp tells the memory system what the coder will touch while coding byte `nb` with the
// contexts `h` (lane = component): ICM/ISSE hash-row blocks and CM lines of both nibbles, the 8 rows of
// mixer weights / MIX2 weights / SSE buckets (one per bit: they are selected by the partial byte).
__device__ __forceinline__ void cm_prefetch_byte(const ZqCmComp& c, u8* model, u32 h, u32 nb) {
  const u32 hi = nb >> 4;
  switch (c.type) {
    case ZQ_ICM: case ZQ_ISSE: {
      const u8* ht = model + c.ht_off;
      zq_prefetch_l2(ht + (((h + 16u) * 16u) & (c.ht_mask - 63u)));
      zq_prefetch_l2(ht + (((h + 16u * (16u + hi)) * 16u) & (c.ht_mask - 63u)));
      break;
    }
    case ZQ_CM: {
      const u32* cm = (const u32*)(model + c.cm_off);
      const u32 x2 = ((8u + (hi >> 1)) << 5) | ((hi & 1u) << 4);
      zq_prefetch_l2(cm + (h & c.cm_mask & ~15u));
      zq_prefetch_l2(cm + ((h ^ x2) & c.cm_mask & ~15u));
      break;
    }
    case ZQ_MIX: case ZQ_MIX2: case ZQ_SSE: {
      const u8* base = model + c.cm_off;
      for (u32 i = 0; i < 8; ++i) {
        const u32 c8 = (1u << i) | (nb >> (8 - i));
        if (c.type == ZQ_MIX) {
          const u32 row = ((h + (c8 & c.a5)) & c.cm_mask) * c.a3;
          zq_prefetch_l2(base + (u64)row * 4);
          zq_prefetch_l2(base + (u64)(row + c.a3 - 1) * 4);
        } else if (c.type == ZQ_MIX2) zq_prefetch_l2(base + (u64)((h + (c8 & c.a5)) & c.cm_mask) * 2);
        else zq_prefetch_l2(base + (u64)(((h + c8) * 32u) & c.cm_mask) * 4);
      }
      break;
    }
    default: break;
  }
}

// ---- encoder fast path for the chain ICM -> ISSE (built-in level 3: "ci1" after BWT, "c0,0,511i2" after LZ77) ----
// The compressor knows the whole byte before coding it, so the tree nodes (hash-row slots) of a nibble's
// four bits are known up front: their bit-history states come out of the cached row at once and the four
// probability / weight fetches are issued together; the bits are then pure arithmetic on registers (a later
// bit that lands on the same state as an earlier one of the nibble takes the updated value instead of the
// fetched one).  Nothing here depends on another lane: the coder warp runs it on lane 0, straight-line.
struct ChainComp {
  u32* cm; u8* ht;
  u32 ht_mask, chkshift, rowpos, rowok;
  uint4 row;
};
__device__ __forceinline__ void chain_setup(ChainComp& C, const ZqCmComp& c, u8* model) {
  C.cm = (u32*)(model + c.cm_off); C.ht = model + c.ht_off; C.ht_mask = c.ht_mask; C.chkshift = (u32)c.a1 + 2;
  C.rowpos = 0; C.rowok = 0; C.row = make_uint4(0, 0, 0, 0);
}
// Predictor::find (Z:15254) with the row held in registers
__device__ __forceinline__ void chain_row_switch(ChainComp& C, u32 cxt) {
  if (C.rowok) *(uint4*)(C.ht + C.rowpos) = C.row;
  const u32 chk = (cxt >> C.chkshift) & 255u;
  const u32 h0 = (cxt * 16u) & (C.ht_mask - 15u), h1 = h0 ^ 16u, h2 = h0 ^ 32u;
  const uint4 r0 = *(const uint4*)(C.ht + h0), r1 = *(const uint4*)(C.ht + h1), r2 = *(const uint4*)(C.ht + h2);
  u32 r; uint4 row;
  if ((r0.x & 255u) == chk) { r = h0; row = r0; }
  else if ((r1.x & 255u) == chk) { r = h1; row = r1; }
  else if ((r2.x & 255u) == chk) { r = h2; row = r2; }
  else {
    const u32 p0 = (r0.x >> 8) & 255u, p1 = (r1.x >> 8) & 255u, p2 = (r2.x >> 8) & 255u;
    if (p0 <= p1 && p0 <= p2) r = h0; else if (p1 < p2) r = h1; else r = h2;
    row = make_uint4(chk, 0, 0, 0);
  }
  C.row = row; C.rowpos = r; C.rowok = 1;
}
__device__ __forceinline__ u32 chain_get(u32 word, u32 k) { return (word >> (8 * k)) & 255u; }
__device__ __forceinline__ u32 chain_put(u32 word, u32 k, u32 v) { return (word & ~(255u << (8 * k))) | (v << (8 * k)); }

// four bits (MSB first in `nib`) through ICM `A` -> ISSE `B`
__device__ __forceinline__ void chain1_nibble(ChainComp& A, ChainComp& B, CmCoder& E, const CmSmem& T, u32 nib) {
  const u32 y0 = (nib >> 3) & 1u, y1 = (nib >> 2) & 1u, y2 = (nib >> 1) & 1u, y3 = nib & 1u;
  const u32 i1 = 2u + y0, i2 = (4u + 2u * y0 + y1) & 3u, i3 = 8u + 4u * y0 + 2u * y1 + y2;   // slots 1, i1, 4+i2, i3
  const bool lo3 = i3 < 12u;
  const u32 k3 = i3 & 3u;
  // bit histories of the four nodes, both components
  const u32 sa0 = chain_get(A.row.x, 1), sa1 = chain_get(A.row.x, i1), sa2 = chain_get(A.row.y, i2), sa3 = chain_get(lo3 ? A.row.z : A.row.w, k3);
  const u32 sb0 = chain_get(B.row.x, 1), sb1 = chain_get(B.row.x, i1), sb2 = chain_get(B.row.y, i2), sb3 = chain_get(lo3 ? B.row.z : B.row.w, k3);
  // their adaptive probabilities (ICM) and weight pairs (ISSE): eight independent fetches
  u32 pn0 = A.cm[sa0], pn1 = A.cm[sa1], pn2 = A.cm[sa2], pn3 = A.cm[sa3];
  int2 w0 = *(const int2*)(B.cm + sb0 * 2), w1 = *(const int2*)(B.cm + sb1 * 2), w2 = *(const int2*)(B.cm + sb2 * 2),
       w3 = *(const int2*)(B.cm + sb3 * 2);
#define ZQ_CHAIN_BIT(PN, W, SA, SB, YB)                                                         \
  {                                                                                               \
    const int pa = T.stretch[(PN) >> 8];                                                          \
    const int pb = cm_clamp2k(((W).x * pa + (W).y * 64) >> 16);                                   \
    const int pr = T.squash[pb + 2048];                                                           \
    E.encode((int)(YB), (u32)pr * 2 + 1);                                                         \
    (PN) += (u32)(((int)((YB) * 32767u) - (int)((PN) >> 8)) >> 2);                                \
    A.cm[SA] = (PN);                                                                              \
    const int err = (int)((YB) * 32767u) - pr;                                                    \
    (W).x = cm_clamp512k((W).x + ((err * pa + (1 << 12)) >> 13));                                 \
    (W).y = cm_clamp512k((W).y + ((err + 16) >> 5));                                              \
    *(int2*)(B.cm + (SB) * 2) = (W);                                                              \
  }
  ZQ_CHAIN_BIT(pn0, w0, sa0, sb0, y0)
  if (sa1 == sa0) pn1 = pn0;
  if (sb1 == sb0) w1 = w0;
  ZQ_CHAIN_BIT(pn1, w1, sa1, sb1, y1)
  if (sa2 == sa0) pn2 = pn0;
  if (sa2 == sa1) pn2 = pn1;
  if (sb2 == sb0) w2 = w0;
  if (sb2 == sb1) w2 = w1;
  ZQ_CHAIN_BIT(pn2, w2, sa2, sb2, y2)
  if (sa3 == sa0) pn3 = pn0;
  if (sa3 == sa1) pn3 = pn1;
  if (sa3 == sa2) pn3 = pn2;
  if (sb3 == sb0) w3 = w0;
  if (sb3 == sb1) w3 = w1;
  if (sb3 == sb2) w3 = w2;
  ZQ_CHAIN_BIT(pn3, w3, sa3, sb3, y3)
#undef ZQ_CHAIN_BIT
  // next states into the rows
  A.row.x = chain_put(chain_put(A.row.x, 1, T.ns[sa0 * 4 + y0]), i1, T.ns[sa1 * 4 + y1]);
  A.row.y = chain_put(A.row.y, i2, T.ns[sa2 * 4 + y2]);
  B.row.x = chain_put(chain_put(B.row.x, 1, T.ns[sb0 * 4 + y0]), i1, T.ns[sb1 * 4 + y1]);
  B.row.y = chain_put(B.row.y, i2, T.ns[sb2 * 4 + y2]);
  const u32 na3 = T.ns[sa3 * 4 + y3], nb3 = T.ns[sb3 * 4 + y3];
  if (lo3) { A.row.z = chain_put(A.row.z, k3, na3); B.row.z = chain_put(B.row.z, k3, nb3); }
  else { A.row.w = chain_put(A.row.w, k3, na3); B.row.w = chain_put(B.row.w, k3, nb3); }
}

// whole block through the chain model, on the calling lane; contexts come from the pair's ring
__device__ void cm_code_chain1(const ZqCmPlan& cp, u8* model, CmUnitSmem& S, const CmSmem& T, CmCoder& E,
                               const u8* __restrict__ head, u32 hlen, const u8* __restrict__ stream, u32 K) {
  ChainComp A, B;
  chain_setup(A, cp.comp[0], model);
  chain_setup(B, cp.comp[1], model);
  u32 ha = 0, hb = 0;
  for (u32 k = 0; k < K; ++k) {
    if (k > 0) {
      while (S.produced < k) __nanosleep(32);
      __threadfence_block();
      ha = S.ring[(k - 1) % ZQ_CM_RING][0]; hb = S.ring[(k - 1) % ZQ_CM_RING][1];
      __threadfence_block();
      S.consumed = k;
    }
    const u32 c = k < hlen ? head[k] : stream[k - hlen];
    E.encode(0, 0);
    chain_row_switch(A, ha + 16u); chain_row_switch(B, hb + 16u);
    chain1_nibble(A, B, E, T, c >> 4);
    const u32 c8 = 16u + (c >> 4);
    chain_row_switch(A, ha + 16u * c8); chain_row_switch(B, hb + 16u * c8);
    chain1_nibble(A, B, E, T, c & 15u);
  }
}

// Arguments of a translated context kernel (zq_jit.cpp: zq_ctx_kernel) for the listed units: where each block's
// coded bytes start and how many there are (the LZ/BWT stream lengths only exist on the device), model region, slot
// in the context buffer.
__global__ void k_ctx_args(const ZqUnit* __restrict__ units, const ZqPlan* __restrict__ plans, const int* __restrict__ ids, int n,
                           const u32* __restrict__ lz_len, const u64* __restrict__ ctx_off_by_unit, u64* __restrict__ soff,
                           u32* __restrict__ slen, u64* __restrict__ model_off, u64* __restrict__ ctx_off,
                           u64* __restrict__ coded_off, u32* __restrict__ coded_cap) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int ui = ids[t];
  const ZqUnit u = units[ui];
  if (plans[u.plan].lz_level) { soff[t] = u.lz_off; slen[t] = lz_len[ui]; } else { soff[t] = u.in_off; slen[t] = u.n; }
  model_off[t] = u.model_off;
  ctx_off[t] = ctx_off_by_unit[ui];
  coded_off[t] = u.coded_off; coded_cap[t] = u.coded_cap;
}

// grid of persistent CTAs of `blockDim.x / 64` warp pairs (even warp: coder, odd warp: context machine);
// pairs pull modeled units from a counter.  Dynamic shared memory: CmSmem + one CmUnitSmem per pair.
#define ZQ_CM_MAX_PAIRS 12   // 768 threads: 80 registers per thread (sm_90a: 44 bytes spilled); 1 584 blocks resident on 132 SMs
template <int VM, bool CTX>   // CTX: contexts of some blocks arrive precomputed (translated HCOMP, zq_jit.cpp)
__global__ void __launch_bounds__(64 * ZQ_CM_MAX_PAIRS, 1)
k_cm_encode(const u8* __restrict__ in_base, const ZqUnit* __restrict__ units, const ZqPlan* __restrict__ plans,
            const ZqCmPlan* __restrict__ cmplans, const int* __restrict__ todo, int ntodo,
            const CmTablesDev* __restrict__ tab, const u8* __restrict__ blob, const u8* __restrict__ lz_base,
            const u32* __restrict__ lz_len, u8* __restrict__ model_base, u8* __restrict__ coded_base,
            u32* __restrict__ coded_len, u32* __restrict__ err_flag, u32* __restrict__ next_unit, int prefetch, int fast,
            const u32* __restrict__ ctx_base, const u64* __restrict__ ctx_off) {
  ZQ_DYN_SMEM(smem_raw);
  CmSmem& T = *reinterpret_cast<CmSmem*>(smem_raw);
  {
    const uint4* src = (const uint4*)tab;
    uint4* dst = (uint4*)smem_raw;
    for (u32 k = threadIdx.x; k < sizeof(CmSmem) / 16; k += blockDim.x) dst[k] = src[k];
  }
  __syncthreads();
  const u32 lane = lane_id(), warp = threadIdx.x >> 5, pair = warp >> 1, role = warp & 1;
  CmUnitSmem& S = reinterpret_cast<CmUnitSmem*>(smem_raw + sizeof(CmSmem))[pair];
  for (;;) {
    if (role == 0 && lane == 0) { S.unit = (int)atomicAdd(next_unit, 1u); S.produced = 0; S.consumed = 0; }
    zq_pair_sync(pair);
    const int t = S.unit;
    zq_pair_sync(pair);     // both warps hold t before the coder may publish the next one
    if (t >= ntodo) break;
    const int ui = todo[t];
    const ZqUnit u = units[ui];
    const ZqPlan pl = plans[u.plan];
    const ZqCmPlan& cp = cmplans[pl.cm_plan];
    u8* model = model_base + u.model_off;
    // the coded stream: post-processor selector (+ PCOMP bytes), then the (pre-processed) data
    const u8* __restrict__ stream; u32 slen;
    if (pl.lz_level) { stream = lz_base + u.lz_off; slen = lz_len[ui]; }
    else { stream = in_base + u.in_off; slen = u.n; }
    const u8* __restrict__ head = blob + pl.payload_off;
    const u32 hlen = pl.payload_len, K = hlen + slen;
    if (cp.n > ZQ_CM_LANES) {
      // ---- a model wider than the warp: the coder warp's lane 0 runs the context machine and every component itself
      if (role == 0) {
        CmVm vm;
        cm_vm_setup(vm, cp, model, blob, S);
        if (lane == 0) {
          CmCoder E; E.init(coded_base + u.coded_off, u.coded_cap);
          CmWide W;
          cmw_setup(W, cp, model);
          for (u32 k = 0; k < K; ++k) {
            const u32 c = k < hlen ? head[k] : stream[k - hlen];
            E.encode(0, 0);
            for (int i = 7; i >= 0; --i) {
              const u32 p16 = (u32)cmw_predict(W, vm.h, vm.hmask, T) * 2 + 1;
              const int y = (c >> i) & 1;
              E.encode(y, p16);
              cmw_update(W, vm.h, vm.hmask, T, y);
            }
            if (k + 1 < K) cm_vm_run<VM, false>(vm, c, nullptr);
          }
          E.encode(1, 0);   // end of segment
          coded_len[ui] = (u32)(E.out - (coded_base + u.coded_off));
          if (E.overflow) atomicOr(err_flag, 1u);
          if (vm.error) atomicOr(err_flag, 2u);
        }
        __syncwarp();
      }
      continue;
    }
    if (role == 1) {
      // ---- context warp: HCOMP on byte k -> ring slot k, for every byte but the last.  When the block's contexts
      // were already computed by the translated program (zq_jit.cpp: ctx_off[ui] != ~0), they are only streamed in.
      CmVm vm;
      cm_vm_setup(vm, cp, model, blob, S);
      const bool act = lane < (u32)cp.n;
      const ZqCmComp comp = cp.comp[act ? lane : 0];
      const u32* __restrict__ cx = (CTX && ctx_base && ctx_off[ui] != ~(u64)0) ? ctx_base + ctx_off[ui] : nullptr;
      for (u32 k = 0; k + 1 < K; ++k) {
        if (!CTX || !cx) {
          const u32 c = k < hlen ? head[k] : stream[k - hlen];
          if (lane == 0) cm_vm_run<VM, false>(vm, c, nullptr);
          __syncwarp();
        }
        while (k - S.consumed >= ZQ_CM_RING) __nanosleep(64);
        const u32 hv = !act ? 0u : (CTX && cx) ? cx[(u64)k * (u32)cp.n + lane] : vm.h[lane & vm.hmask];
        S.ring[k % ZQ_CM_RING][lane] = hv;
        if (prefetch && act) cm_prefetch_byte(comp, model, hv, k + 1 < hlen ? head[k + 1] : stream[k + 1 - hlen]);
        __syncwarp();
        if (lane == 0) { __threadfence_block(); S.produced = k + 1; }
      }
      if (lane == 0 && vm.error) atomicOr(err_flag, 2u);
    } else {
      // ---- coder warp
      CmCoder E; E.init(coded_base + u.coded_off, u.coded_cap);
      if (cp.chain == 1 && fast) {
        if (lane == 0) {
          cm_code_chain1(cp, model, S, T, E, head, hlen, stream, K);
          E.encode(1, 0);   // end of segment
          coded_len[ui] = (u32)(E.out - (coded_base + u.coded_off));
          if (E.overflow) atomicOr(err_flag, 1u);
        }
        __syncwarp();
        continue;
      }
      CmCtx X; CmLane L;
      cm_setup(L, X, cp, model, S);
      for (u32 k = 0; k < K; ++k) {
        if (k > 0) {
          while (S.produced < k) __nanosleep(32);
          __threadfence_block();
          L.h = S.ring[(k - 1) % ZQ_CM_RING][lane];
          __syncwarp();
          if (lane == 0) S.consumed = k;
        }
        const u32 c = k < hlen ? head[k] : stream[k - hlen];
        E.encode(0, 0);
        for (int i = 7; i >= 0; --i) {
          const u32 p16 = (u32)cm_predict(L, X, T) * 2 + 1;
          const int y = (c >> i) & 1;
          E.encode(y, p16);
          cm_update(L, X, T, y);
        }
      }
      E.encode(1, 0);   // end of segment
      if (lane == 0) {
        coded_len[ui] = (u32)(E.out - (coded_base + u.coded_off));
        if (E.overflow) atomicOr(err_flag, 1u);
      }
    }
  }
}

}  // namespace zqdev
