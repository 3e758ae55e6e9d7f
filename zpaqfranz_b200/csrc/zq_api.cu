// zq_api.cu -- context, wave orchestration and the extern "C" boundary (include/zq_b200.h).
// Host C++ above the C ABI stays tiny: method planning (zq_config.cpp), descriptor upload, kernel
// launches on one stream, one small D2H (stream lengths) to lay the finished blocks back to back.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/zq_b200.h"
#include "zq_cm.cuh"
#include "zq_cm_host.h"
#include "zq_jit.h"
#include "zq_common.cuh"
#include "zq_config.h"
#include "zq_decode.cuh"
#include "zq_fragment.cuh"
#include "zq_frame.cuh"
#include "zq_hashes.cuh"
#include "zq_hashes2.cuh"
#include "zq_hashes3.cuh"
#include "zq_lz77.cuh"
#include "zq_lz77_scan.cuh"
#include "zq_sha1.cuh"
#include "zq_sufsort.cuh"
#include "zq_sufsort16.cuh"

namespace {

thread_local std::string g_create_error;

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) { e = cudaMalloc(&p, bytes); want = bytes; }
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct Timer {
  cudaEvent_t a = nullptr, b = nullptr;
  bool used = false;
};

}  // namespace

struct zq_ctx {
  int device = 0;
  int num_sms = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t own_stream = nullptr;
  std::string err;
  uint64_t launches = 0;
  DevBuf d_in, d_out, d_units, d_plans, d_blob, d_todo, d_outoff, d_work, d_ht, d_todo2, d_todo3, d_todo4, d_todo5, d_dec, d_tok, d_bitpos, d_lz, d_lzlen, d_sha, d_tables, d_cmplans, d_fills, d_model, d_coded, d_codedlen,
      d_kbuf, d_vbuf, d_err, d_misc, d_lzs, d_sortflag;
  Timer tm[16];
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};   // h2d / d2h timing of the host-pointer entry point
  bool attr_cm_enc = false, attr_cm_dec = false, attr_sort16 = false;
  int sort16 = 1;                         // blocks <= 64 KiB: shared-memory sort (zq_sufsort16.cuh); ZQ_SORT16=0 sends everything to k_suffix_sort
  float last_ms[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  size_t wave_bytes = 0;                 // sa|isa|lcp|bwt|scan-table bytes per wave (zq_create: 1/16 of device memory)
  size_t model_budget = (size_t)120 << 30; // component-table bytes per wave (capped by free memory)
  int sort_nt = 256, sort_minb = 4;       // suffix-sort CTA size and CTAs per SM (ZQ_SORT_NT / ZQ_SORT_MINB select the others)
  uint64_t frag_seg = 128 << 10;          // fragmenter segment size
  int lz_old = 0;                         // 1: warp-per-block LZ77 parser for every block (ZQ_LZ_OLD=1); 0: position-parallel scan/walk/emit (zq_lz77_scan.cuh)
  int scan_occ[2][2] = {{0, 0}, {0, 0}};  // resident CTAs per SM of k_lz_scan<u16/u32, pass> (queried once)
  int cm_jit = 1;                         // 1: contexts from the translated HCOMP (zq_jit.cpp, NVRTC) instead of the interpreter; 2: generated coder too (ZQ_CM_JIT)
  std::vector<zq_segment> last_segs;      // every segment of the last zq_decompress_* call, in (block, position) order
  void (*gate_fn)(void*, int) = nullptr;  // zq_set_compute_gate: called with 1 before the first kernel of a batch, 0 after its last
  void* gate_arg = nullptr;
  bool copy_held = false;                 // between fn(arg, 2) and fn(arg, 3): this batch's input copy owns the H2D turn
  bool cm_jit_auto = true;                // no ZQ_CM_JIT in the environment: translate only the models whose context warp is the bottleneck (<= 8 components)
  struct JitProg { cudaLibrary_t lib = nullptr; cudaKernel_t ctx = nullptr, code = nullptr; };
  std::map<std::string, JitProg> jit_cache;   // translated context program (+ generated coder) per model header
  DevBuf d_ctx, d_ctxoff, d_ctxargs;
  int cm_fast = 1;                        // encoder fast path for chain models (ZQ_CM_FAST=0: generic lanes)
  int cm_prefetch = 1;                    // context warp prefetches the coder's table lines (ZQ_CM_PREFETCH=0 to turn off)
};

namespace {

int fail(zq_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg; else g_create_error = msg;
  return code;
}
#define ZQ_CUDA(c, call)                                                                          \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(c, e_ == cudaErrorMemoryAllocation ? ZQ_E_NOMEM : ZQ_E_NODEVICE,                 \
                  std::string(e_ == cudaErrorMemoryAllocation ? "Out of memory: " : "CUDA error: ") + \
                      cudaGetErrorString(e_) + " at " #call);                                      \
  } while (0)

void tstart(zq_ctx* c, int k) { cudaEventRecord(c->tm[k].a, c->stream); c->tm[k].used = true; }
void tstop(zq_ctx* c, int k) { cudaEventRecord(c->tm[k].b, c->stream); }

struct HostPlan {
  zq::BlockPlan bp;
  std::vector<uint8_t> payload;  // selector + pcomp
};

// A caller-supplied model (the Compressor class: startBlock(hcomp) / postProcess(pcomp) / endSegment(sha1)).
struct RawModel {
  zq::Assembled code;            // parsed COMP/HCOMP header
  std::vector<uint8_t> pcomp;    // PCOMP bytecode announced in the first segment (may be empty)
  bool tag = true;               // writeTag()
  const uint8_t* digests = nullptr;  // n x 20 bytes to store as FD sha1, or null -> FE
};

static const unsigned char kTag[13] = {0x37, 0x6b, 0x53, 0x74, 0xa0, 0x31, 0x83, 0xd3, 0x8c, 0xb2, 0x28, 0xb0, 0xd3};

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// The core: inputs and outputs already on the device.
struct GateHold {   // the batch's kernels run between acquire() and the end of the scope
  zq_ctx* c; bool held = false;
  explicit GateHold(zq_ctx* c_) : c(c_) {}
  void acquire() {
    if (c->gate_fn && c->copy_held) {   // the input copy (queued before the planning above) must have landed: next batch's turn to copy
      cudaEventSynchronize(c->ev[1]);
      c->gate_fn(c->gate_arg, 3); c->copy_held = false;
    }
    if (c->gate_fn && !held) { c->gate_fn(c->gate_arg, 1); held = true; }
  }
  ~GateHold() { if (held) c->gate_fn(c->gate_arg, 0); }
};

int compress_core(zq_ctx* c, int n, const uint8_t* d_in, const uint64_t* in_off, const uint32_t* in_len,
                  const char* const* method, const char* const* filename, const char* const* comment,
                  int uniform, int dosha1, uint8_t* d_out, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len,
                  const RawModel* raw = nullptr) {
  using namespace zqdev;
  if (n < 0 || (n > 0 && (!in_off || !in_len || !out_off || !out_len))) return fail(c, ZQ_E_ARG, "bad argument");
  if (n == 0) return ZQ_OK;
  // ---- plans -----------------------------------------------------------------------------------
  std::vector<HostPlan> plans;
  std::map<std::string, int> plan_idx;   // expanded method | size class -> plan
  std::map<std::string, std::string> expand_cache;
  std::vector<ZqUnit> units(n);
  std::vector<uint8_t> blob;
  // digit levels >= 5 pick their periodic models from the data: analysed on the device
  std::vector<int> periods;
  {
    std::vector<int> need;
    for (int u = 0; u < n && !raw; ++u) {
      const char* m = method ? method[uniform ? 0 : u] : "1";
      if (m && isdigit((unsigned char)m[0]) && m[0] >= '5') need.push_back(u);
    }
    if (!need.empty()) {
      const int k = (int)need.size();
      std::vector<uint64_t> o(k); std::vector<uint32_t> l(k);
      for (int j = 0; j < k; ++j) { o[j] = in_off[need[j]]; l[j] = in_len[need[j]]; }
      ZQ_CUDA(c, c->d_misc.ensure((size_t)k * 20 + 64));
      u64* d_o = c->d_misc.as<u64>(); u32* d_l = (u32*)(d_o + k); int* d_p = (int*)(d_l + k);
      ZQ_CUDA(c, cudaMemcpyAsync(d_o, o.data(), (size_t)k * 8, cudaMemcpyHostToDevice, c->stream));
      ZQ_CUDA(c, cudaMemcpyAsync(d_l, l.data(), (size_t)k * 4, cudaMemcpyHostToDevice, c->stream));
      k_gap_periods<<<std::min(k, c->num_sms * 8), 256, 0, c->stream>>>(d_in, d_o, d_l, k, d_p);
      ++c->launches;
      std::vector<int> pk((size_t)k * 2);
      ZQ_CUDA(c, cudaMemcpyAsync(pk.data(), d_p, (size_t)k * 8, cudaMemcpyDeviceToHost, c->stream));
      ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
      periods.assign((size_t)n * 2, 0);
      for (int j = 0; j < k; ++j) { periods[2 * need[j]] = pk[2 * j]; periods[2 * need[j] + 1] = pk[2 * j + 1]; }
    }
  }
  try {
    for (int u = 0; u < n; ++u) {
      const char* m = raw ? "(caller's model)" : method ? method[uniform ? 0 : u] : "1";
      if (!m || !*m) return fail(c, ZQ_E_ARG, "empty method");
      const uint32_t len = in_len[u];
      int arg0 = zq::bitlen(len + 4095) - 20; if (arg0 < 0) arg0 = 0;
      const bool data_dependent = !raw && isdigit((unsigned char)m[0]) && m[0] >= '5';
      std::string expanded;
      if (raw) { expanded = m; arg0 = 0; }
      else if (data_dependent) {
        expanded = zq::expand_method_periods(m, len, &periods[2 * u]);
      } else {
        const std::string ck = std::string(m) + "|" + std::to_string(arg0);
        auto it = expand_cache.find(ck);
        if (it == expand_cache.end()) it = expand_cache.emplace(ck, zq::expand_method(m, nullptr, len)).first;
        expanded = it->second;
      }
      const std::string key = expanded + "|" + std::to_string(arg0);
      int pi;
      auto it = plan_idx.find(key);
      if (it != plan_idx.end()) pi = it->second;
      else {
        HostPlan hp;
        if (raw) {   // data goes to the coder as is; the caller did its own pre-processing
          hp.bp.method = expanded; memset(hp.bp.args, 0, sizeof hp.bp.args);
          hp.bp.code = raw->code; hp.bp.code.pcomp = raw->pcomp;
          hp.bp.lz_level = 0; hp.bp.e8e9 = false; hp.bp.use_sa = false; hp.bp.stored = false;
        } else hp.bp = zq::plan_block(expanded, nullptr, len);
        const auto& pc = hp.bp.code.pcomp;
        if (!pc.empty()) { hp.payload.push_back(1); hp.payload.push_back(pc.size() & 255); hp.payload.push_back(pc.size() >> 8); hp.payload.insert(hp.payload.end(), pc.begin(), pc.end()); }
        else hp.payload.push_back(0);
        pi = (int)plans.size();
        plans.push_back(std::move(hp));
        plan_idx[key] = pi;
      }
      const HostPlan& hp = plans[pi];
      ZqUnit& zu = units[u];
      memset(&zu, 0, sizeof zu);
      zu.in_off = in_off[u]; zu.n = len; zu.plan = (u32)pi;
      // prefix: tag, "zPQ", level, 1, header, 1, filename, 0, "<n>[ comment]", 0, 0
      zu.prefix_off = (u32)blob.size();
      if (!raw || raw->tag) blob.insert(blob.end(), kTag, kTag + 13);
      blob.push_back('z'); blob.push_back('P'); blob.push_back('Q');
      blob.push_back(1 + (hp.bp.code.ncomp == 0)); blob.push_back(1);
      blob.insert(blob.end(), hp.bp.code.header.begin(), hp.bp.code.header.end());
      blob.push_back(1);
      const char* fn = filename ? filename[uniform ? 0 : u] : nullptr;
      if (fn) blob.insert(blob.end(), fn, fn + strlen(fn));
      blob.push_back(0);
      std::string cs = raw ? std::string() : std::to_string(len);   // startSegment() stores the comment verbatim (Z:16070)
      const char* cm = comment ? comment[uniform ? 0 : u] : nullptr;
      if (cm) { if (!raw) cs += " "; cs += cm; }
      blob.insert(blob.end(), cs.begin(), cs.end());
      blob.push_back(0); blob.push_back(0);
      zu.prefix_len = (u32)blob.size() - zu.prefix_off;
    }
  } catch (const zq::Error& e) {
    return fail(c, ZQ_E_METHOD, e.msg);
  }
  std::vector<ZqPlan> dplans(plans.size());
  std::vector<ZqCmPlan> cmplans;
  std::vector<ZqCmFill> fills;
  bool any_modeled = false;
  for (size_t i = 0; i < plans.size(); ++i) {
    ZqPlan& p = dplans[i];
    memcpy(p.args, plans[i].bp.args, sizeof p.args);
    p.payload_off = (u32)blob.size(); p.payload_len = (u32)plans[i].payload.size();
    blob.insert(blob.end(), plans[i].payload.begin(), plans[i].payload.end());
    p.lz_level = plans[i].bp.lz_level; p.use_sa = plans[i].bp.use_sa; p.e8e9 = plans[i].bp.e8e9;
    p.modeled = plans[i].bp.code.ncomp > 0; p.cm_plan = 0;
    if (p.lz_level && !p.use_sa && (p.args[5] < 4 || p.args[5] > 30 || p.args[4] > 16 || p.args[0] > 11))
      return fail(c, ZQ_E_UNSUPPORTED, "LZ77 hash table parameters outside the device path: " + plans[i].bp.method);
    if ((p.lz_level == 1 || p.lz_level == 2) && (p.args[2] < (p.lz_level == 1 ? 4 : 1) || p.args[2] > 64 + 191 * (p.lz_level == 1)))
      return fail(c, ZQ_E_METHOD, "match length $3 too small");
    if (p.modeled) {
      any_modeled = true;
      try {
        ZqCmPlan cp = zq::make_cm_plan(plans[i].bp.code, fills);
        cp.hcomp_off = (u32)blob.size(); cp.hcomp_len = (u32)plans[i].bp.code.hcomp.size();
        blob.insert(blob.end(), plans[i].bp.code.hcomp.begin(), plans[i].bp.code.hcomp.end());
        p.cm_plan = (u32)cmplans.size();
        cmplans.push_back(cp);
      } catch (const zq::Error& e) {
        return fail(c, ZQ_E_UNSUPPORTED, e.msg + ": " + plans[i].bp.method);
      }
    }
  }
  if (any_modeled && !c->d_tables.p) {
    try {
      const zq::CmTables& t = zq::cm_tables();
      ZQ_CUDA(c, c->d_tables.ensure(sizeof(zq::CmTables)));
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_tables.p, &t, sizeof t, cudaMemcpyHostToDevice, c->stream));
    } catch (const zq::Error& e) { return fail(c, ZQ_E_METHOD, e.msg); }
  }
  // ---- device tables -----------------------------------------------------------------------------
  for (int k = 0; k < 16; ++k) c->tm[k].used = false;
  tstart(c, 0);
  ZQ_CUDA(c, c->d_plans.ensure(dplans.size() * sizeof(ZqPlan)));
  ZQ_CUDA(c, c->d_blob.ensure(blob.size() + 16));
  ZQ_CUDA(c, c->d_units.ensure((size_t)n * sizeof(ZqUnit)));
  ZQ_CUDA(c, c->d_outoff.ensure((size_t)n * 8));
  ZQ_CUDA(c, c->d_lzlen.ensure((size_t)n * 4));
  ZQ_CUDA(c, c->d_codedlen.ensure((size_t)n * 4));
  ZQ_CUDA(c, c->d_todo.ensure((size_t)n * 4));
  ZQ_CUDA(c, c->d_err.ensure(64));
  if (dosha1) ZQ_CUDA(c, c->d_sha.ensure((size_t)n * 20));
  ZQ_CUDA(c, cudaMemsetAsync(c->d_err.p, 0, 64, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_plans.p, dplans.data(), dplans.size() * sizeof(ZqPlan), cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_blob.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, c->stream));
  if (!cmplans.empty()) {
    ZQ_CUDA(c, c->d_cmplans.ensure(cmplans.size() * sizeof(ZqCmPlan)));
    ZQ_CUDA(c, c->d_fills.ensure(fills.size() * sizeof(ZqCmFill)));
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_cmplans.p, cmplans.data(), cmplans.size() * sizeof(ZqCmPlan), cudaMemcpyHostToDevice, c->stream));
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_fills.p, fills.data(), fills.size() * sizeof(ZqCmFill), cudaMemcpyHostToDevice, c->stream));
  }
  size_t model_budget = c->model_budget;
  if (any_modeled) {
    size_t fr = 0, tot = 0;
    cudaMemGetInfo(&fr, &tot);
    fr += c->d_model.cap;                       // our own cached arena can be reused
    model_budget = std::min<size_t>(model_budget, fr > ((size_t)6 << 30) ? fr - ((size_t)6 << 30) : fr / 2);
  }
  // waves: contiguous unit ranges whose suffix-array and model footprints fit the budgets
  GateHold gate(c);
  gate.acquire();
  std::vector<uint32_t> lz_len_h(n, 0), coded_len_h(n, 0);
  uint64_t out_pos = 0;
  float stage_ms[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // per stage, summed over the waves
  int w0 = 0;
  while (w0 < n) {
    size_t work = 0, lzbytes = 0, maxn = 0, model = 0, coded = 0, htbytes = 0;
    int w1 = w0, maxjobs = 0;
    std::vector<int> todo_sa, todo_bwt, todo_cm, todo_hash, todo_e8;
    while (w1 < n) {
      ZqUnit& zu = units[w1];
      const ZqPlan& p = dplans[zu.plan];
      zu.idx16 = zu.n <= 65536 ? 1 : 0;
      const bool hashlz = p.lz_level && !p.use_sa;
      if (p.e8e9) todo_e8.push_back(w1 - w0);
      const bool scan_ok = p.use_sa && p.lz_level != 3 && !c->lz_old && p.args[4] <= 7 && p.args[6] <= 1;   // covered by the scan pipeline
      zu.want_pk = scan_ok ? 1 : 0;
      const size_t e = !p.use_sa ? 0 : scan_ok ? (size_t)zq_work_bytes_scan(zu.n, zu.idx16 ? 2 : 4) : (size_t)zq_work_bytes(zu.n, zu.idx16 ? 2 : 4);
      const size_t hb = hashlz ? ((size_t)4 << p.args[5]) : 0;
      const size_t mb = p.modeled ? (size_t)cmplans[p.cm_plan].model_bytes : 0;
      if (w1 > w0 && (work + e + htbytes + hb > c->wave_bytes || model + mb > model_budget)) break;
      if (hashlz) { zu.work_off = htbytes; htbytes += hb; todo_hash.push_back(w1 - w0); }
      else { zu.work_off = work; work += e; }
      uint32_t slen_max = zu.n;
      if (p.lz_level) {
        zu.lz_off = lzbytes; zu.lz_cap = zu.n + zu.n / 32 + 64; lzbytes += align_up(zu.lz_cap, 16);
        slen_max = zu.lz_cap;
        if (p.lz_level == 3) todo_bwt.push_back(w1 - w0);
        if (p.use_sa) { todo_sa.push_back(w1 - w0); maxn = std::max(maxn, (size_t)zu.n); }
      }
      if (p.modeled) {
        zu.model_off = model; model += mb;
        zu.coded_off = coded; zu.coded_cap = slen_max + slen_max / 8 + p.payload_len * 2 + 1024; coded += align_up(zu.coded_cap, 16);
        todo_cm.push_back(w1 - w0);
        maxjobs = std::max(maxjobs, (int)cmplans[p.cm_plan].fill_count);
      }
      ++w1;
    }
    const int wn = w1 - w0;
    if (model > model_budget && wn == 1 && model > c->d_model.cap) {
      // a single block whose model does not fit: let cudaMalloc decide
    }
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_units.p, units.data() + w0, (size_t)wn * sizeof(ZqUnit), cudaMemcpyHostToDevice, c->stream));
    const ZqUnit* du = c->d_units.as<ZqUnit>();
    const ZqPlan* dp = c->d_plans.as<ZqPlan>();
    if (dosha1 && raw && raw->digests) {   // endSegment(sha1string): the caller's digest of the original data
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_sha.p, raw->digests + (size_t)w0 * 20, (size_t)wn * 20, cudaMemcpyHostToDevice, c->stream));
    } else if (dosha1) {
      tstart(c, 1);
      k_sha1_units<<<(wn + 127) / 128, 128, 0, c->stream>>>(d_in, du, wn, c->d_sha.as<u8>());
      ++c->launches;
      tstop(c, 1);
    }
    if (lzbytes) ZQ_CUDA(c, c->d_lz.ensure(lzbytes));
    if (!todo_e8.empty()) {   // after the SHA-1 of the original bytes, like compressBlock (Z:20285 then Z:19363/20414)
      const int nt = (int)todo_e8.size();
      ZQ_CUDA(c, c->d_todo5.ensure((size_t)nt * 4));
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo5.p, todo_e8.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, c->stream));
      k_e8e9<<<(nt + 63) / 64, 64, 0, c->stream>>>(const_cast<u8*>(d_in), du, c->d_todo5.as<int>(), nt);
      ++c->launches;
    }
    if (!todo_sa.empty()) {
      const int nt = (int)todo_sa.size();
      ZQ_CUDA(c, c->d_work.ensure(work));
      const size_t scr = align_up(maxn + 1, 64);
      int sort_nt = c->sort_nt, sort_minb = c->sort_minb;
      const int sort_grid = std::min(nt, c->num_sms * sort_minb);
      ZQ_CUDA(c, c->d_kbuf.ensure((size_t)sort_grid * 2 * scr * 8));
      ZQ_CUDA(c, c->d_vbuf.ensure((size_t)sort_grid * 6 * scr * 4));
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo.p, todo_sa.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, c->stream));
      tstart(c, 2);
      // blocks of up to 64 KiB: sorted in shared memory (zq_sufsort16.cuh); what that kernel hands back (larger blocks,
      // blocks with long repeats) goes to the general prefix-doubling sort
      const u32* d_only = nullptr;
      if (c->sort16) {
        ZQ_CUDA(c, c->d_sortflag.ensure((size_t)nt * 4 + 16));
        u32* ctr16 = c->d_err.as<u32>() + 3;
        ZQ_CUDA(c, cudaMemsetAsync(ctr16, 0, 4, c->stream));
        if (!c->attr_sort16) { cudaFuncSetAttribute(k_suffix_sort16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Sort16Smem)); c->attr_sort16 = true; }
        k_suffix_sort16<<<std::min(nt, c->num_sms), S16_NT, sizeof(Sort16Smem), c->stream>>>(d_in, du, c->d_todo.as<int>(), nt, c->d_work.as<u8>(),
                                                                                         c->d_sortflag.as<u32>(), ctr16);
        ++c->launches;
        d_only = c->d_sortflag.as<u32>();
      }
#define ZQ_SORT_LAUNCH(NT, MB)                                                                                            \
  do {                                                                                                                   \
    cudaFuncSetAttribute(k_suffix_sort<NT, MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SortSmem<NT>)); \
    k_suffix_sort<NT, MB><<<sort_grid, NT, sizeof(SortSmem<NT>), c->stream>>>(                                           \
        d_in, du, c->d_todo.as<int>(), nt, c->d_work.as<u8>(), c->d_kbuf.as<u64>(), c->d_vbuf.as<u32>(), scr, d_only);  \
  } while (0)
      if (sort_nt == 1024) ZQ_SORT_LAUNCH(1024, 1);
      else if (sort_nt == 512 && sort_minb == 2) ZQ_SORT_LAUNCH(512, 2);
      else if (sort_nt == 512) ZQ_SORT_LAUNCH(512, 4);
      else if (sort_nt == 256 && sort_minb == 4) ZQ_SORT_LAUNCH(256, 4);
      else if (sort_nt == 256) ZQ_SORT_LAUNCH(256, 8);
      else if (sort_nt == 128 && sort_minb == 8) ZQ_SORT_LAUNCH(128, 8);
      else ZQ_SORT_LAUNCH(128, 16);
#undef ZQ_SORT_LAUNCH
      ++c->launches;
      tstop(c, 2);
      tstart(c, 3);
      {
        // LZ77 parse.  Blocks the scan pipeline covers (bucket <= 127, look-ahead <= 1: every built-in method) go
        // through k_lz_scan<0/1> -> k_lz_walk -> k_lz_emit, per index width; the rest through the warp-per-block
        // parser.  BWT units go to their own kernel.
        std::vector<int> lists[4];   // 0/1: scan pipeline u16/u32; 2/3: warp-per-block parser u16/u32
        for (int t : todo_sa) {
          const ZqUnit& zu = units[w0 + t];
          const ZqPlan& p = dplans[zu.plan];
          if (p.lz_level == 3) continue;
          lists[(zu.want_pk ? 0 : 2) + (zu.idx16 ? 0 : 1)].push_back(t);
        }
        size_t lo = 0;
        std::vector<int> flat;
        for (auto& l : lists) flat.insert(flat.end(), l.begin(), l.end());
        const size_t nscan = lists[0].size() + lists[1].size();
        flat.insert(flat.end(), todo_bwt.begin(), todo_bwt.end());
        ZQ_CUDA(c, c->d_todo2.ensure(flat.size() * 4 + 4));
        ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo2.p, flat.data(), flat.size() * 4, cudaMemcpyHostToDevice, c->stream));
        ZQ_CUDA(c, cudaMemsetAsync(c->d_err.as<u32>() + 4, 0, 48, c->stream));   // the work-queue counters of this wave
        ZQ_CUDA(c, cudaMemsetAsync(c->d_err.as<u32>() + 1, 0, 8, c->stream));    // (slots 1, 2: the exact walk's)
        if (nscan) {
          const size_t LZS_SMEM16 = sizeof(LzsSmem<u16>) + (LZS_NT / 32) * sizeof(LzsQueue<u16>);
          const size_t LZS_SMEM32 = sizeof(LzsSmem<u32>) + (LZS_NT / 32) * sizeof(LzsQueue<u32>);
          // per list: tile_first[cnt+1] (u32); over both lists: tok_off[nscan] (u64), ntok[nscan] (u32)
          std::vector<uint64_t> tok_off(nscan);
          std::vector<uint32_t> tile_first[2];
          uint64_t ntokcap = 0; bool big = false;
          for (size_t k = 0; k < nscan; ++k) {
            const ZqUnit& zu = units[w0 + flat[k]];
            const ZqPlan& p = dplans[zu.plan];
            tok_off[k] = ntokcap; ntokcap += zu.n / std::max(p.args[2], 1) + zu.n / 4096 + 4;
            big = big || zu.lz_cap > LZE_SMEM_STREAM;
          }
          for (int v = 0; v < 2; ++v) {
            tile_first[v].push_back(0);
            for (int t : lists[v]) tile_first[v].push_back(tile_first[v].back() + lzs_tiles(units[w0 + t].n));
          }
          const size_t tf_bytes = align_up((lists[0].size() + lists[1].size() + 2) * 4, 16);
          ZQ_CUDA(c, c->d_lzs.ensure(tf_bytes + nscan * 12 + 64));
          u32* d_tf0 = c->d_lzs.as<u32>(); u32* d_tf1 = d_tf0 + lists[0].size() + 1;
          u64* d_tokoff = (u64*)(c->d_lzs.as<u8>() + tf_bytes); u32* d_ntok = (u32*)(d_tokoff + nscan);
          ZQ_CUDA(c, cudaMemcpyAsync(d_tf0, tile_first[0].data(), tile_first[0].size() * 4, cudaMemcpyHostToDevice, c->stream));
          ZQ_CUDA(c, cudaMemcpyAsync(d_tf1, tile_first[1].data(), tile_first[1].size() * 4, cudaMemcpyHostToDevice, c->stream));
          ZQ_CUDA(c, cudaMemcpyAsync(d_tokoff, tok_off.data(), nscan * 8, cudaMemcpyHostToDevice, c->stream));
          ZQ_CUDA(c, c->d_tok.ensure(ntokcap * 16 + 64));
          ZQ_CUDA(c, c->d_bitpos.ensure(ntokcap * 8 + 64));
          if (big) ZQ_CUDA(c, cudaMemsetAsync(c->d_lz.p, 0, lzbytes, c->stream));   // streams too large for shared memory are OR-ed in place
          if (!c->scan_occ[0][0]) {
            cudaFuncSetAttribute(k_lz_scan<u16, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZS_SMEM16);
            cudaFuncSetAttribute(k_lz_scan<u16, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZS_SMEM16);
            cudaFuncSetAttribute(k_lz_scan<u32, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZS_SMEM32);
            cudaFuncSetAttribute(k_lz_scan<u32, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZS_SMEM32);
            cudaFuncSetAttribute(k_lz_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LzeSmem));
            int o[2][2] = {{1, 1}, {1, 1}};
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o[0][0], k_lz_scan<u16, 0>, LZS_NT, LZS_SMEM16);
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o[0][1], k_lz_scan<u16, 1>, LZS_NT, LZS_SMEM16);
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o[1][0], k_lz_scan<u32, 0>, LZS_NT, LZS_SMEM32);
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o[1][1], k_lz_scan<u32, 1>, LZS_NT, LZS_SMEM32);
            for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) c->scan_occ[a][b] = std::max(o[a][b], 1);
          }
          u32* ctr = c->d_err.as<u32>() + 10;   // [10..15]: tile / unit counters of this wave
          size_t first = 0;
          for (int v = 0; v < 2; ++v) {
            const int cnt = (int)lists[v].size();
            if (!cnt) continue;
            const int* tl = c->d_todo2.as<int>() + first;
            const u32* tf = v == 0 ? d_tf0 : d_tf1;
            const u32 ntiles = tile_first[v].back();
            u32 tpu = lzs_tiles(units[w0 + lists[v][0]].n);      // all blocks of the list cut into the same number of tiles?
            for (int t : lists[v]) if (lzs_tiles(units[w0 + t].n) != tpu) { tpu = 0; break; }
            // a CTA keeps LZS_NB tiles resident: fewer CTAs than that many tiles would leave SMs empty
            const u32 want_ctas = std::max<u32>(1, (ntiles + LZS_NB - 1) / LZS_NB);
            const unsigned sgrid0 = (unsigned)std::min<u32>(want_ctas, (u32)(c->num_sms * c->scan_occ[v][0]));
            const unsigned sgrid1 = (unsigned)std::min<u32>(want_ctas, (u32)(c->num_sms * c->scan_occ[v][1]));
            const unsigned wgrid = (unsigned)std::min((cnt + 3) / 4, c->num_sms * 16);
            tstart(c, 8 + 0);
            if (v == 0) k_lz_scan<u16, 0><<<sgrid0, LZS_NT, LZS_SMEM16, c->stream>>>(du, dp, tl, tf, cnt, tpu, c->d_work.as<u8>(), ctr + 3 * v);
            else k_lz_scan<u32, 0><<<sgrid0, LZS_NT, LZS_SMEM32, c->stream>>>(du, dp, tl, tf, cnt, tpu, c->d_work.as<u8>(), ctr + 3 * v);
            tstop(c, 8 + 0);
            tstart(c, 8 + 1);
            if (v == 0) k_lz_scan<u16, 1><<<sgrid1, LZS_NT, LZS_SMEM16, c->stream>>>(du, dp, tl, tf, cnt, tpu, c->d_work.as<u8>(), ctr + 3 * v + 1);
            else k_lz_scan<u32, 1><<<sgrid1, LZS_NT, LZS_SMEM32, c->stream>>>(du, dp, tl, tf, cnt, tpu, c->d_work.as<u8>(), ctr + 3 * v + 1);
            tstop(c, 8 + 1);
            tstart(c, 8 + 2);
            // lean walk first, then the form with the exact evaluator for the blocks that met a deferred position
            ZQ_CUDA(c, cudaMemsetAsync(d_ntok + first, 0, (size_t)cnt * 4, c->stream));
            if (v == 0) {
              k_lz_walk<u16, false><<<wgrid, 128, 0, c->stream>>>(d_in, du, dp, tl, cnt, c->d_work.as<u8>(), d_tokoff + first, c->d_tok.as<LzToken>(), d_ntok + first, ctr + 3 * v + 2);
              k_lz_walk<u16, true><<<wgrid, 128, 0, c->stream>>>(d_in, du, dp, tl, cnt, c->d_work.as<u8>(), d_tokoff + first, c->d_tok.as<LzToken>(), d_ntok + first, c->d_err.as<u32>() + 2);
            } else {
              k_lz_walk<u32, false><<<wgrid, 128, 0, c->stream>>>(d_in, du, dp, tl, cnt, c->d_work.as<u8>(), d_tokoff + first, c->d_tok.as<LzToken>(), d_ntok + first, ctr + 3 * v + 2);
              k_lz_walk<u32, true><<<wgrid, 128, 0, c->stream>>>(d_in, du, dp, tl, cnt, c->d_work.as<u8>(), d_tokoff + first, c->d_tok.as<LzToken>(), d_ntok + first, c->d_err.as<u32>() + 1);
            }
            ++c->launches;
            tstop(c, 8 + 2);
            c->launches += 3;
            first += cnt;
          }
          tstart(c, 8 + 3);
          k_lz_emit<<<(unsigned)std::min<size_t>(nscan, (size_t)c->num_sms * 3), LZE_NT, sizeof(LzeSmem), c->stream>>>(
              d_in, du, dp, c->d_todo2.as<int>(), (int)nscan, d_tokoff, c->d_tok.as<LzToken>(), d_ntok, c->d_bitpos.as<u64>(), c->d_lz.as<u8>(),
              c->d_lzlen.as<u32>(), c->d_err.as<u32>());
          tstop(c, 8 + 3);
          ++c->launches;
          lo = nscan;
        }
        for (int v = 2; v < 4; ++v) {
          const int cnt = (int)lists[v].size();
          if (!cnt) continue;
          const int* tl = c->d_todo2.as<int>() + lo;
          lo += cnt;
          const int pgrid = std::min((cnt + 3) / 4, c->num_sms * 6);
          u32* ctr = c->d_err.as<u32>() + 4 + v;
          if (v == 2) k_lz77_sa<u16><<<pgrid, 128, 0, c->stream>>>(d_in, du, dp, tl, cnt, c->d_work.as<u8>(), c->d_lz.as<u8>(), c->d_lzlen.as<u32>(), c->d_err.as<u32>(), ctr);
          else k_lz77_sa<u32><<<pgrid, 128, 0, c->stream>>>(d_in, du, dp, tl, cnt, c->d_work.as<u8>(), c->d_lz.as<u8>(), c->d_lzlen.as<u32>(), c->d_err.as<u32>(), ctr);
          ++c->launches;
        }
        if (!todo_bwt.empty()) {
          k_bwt_stream<<<std::min((int)todo_bwt.size(), c->num_sms * 8), 256, 0, c->stream>>>(
              d_in, du, c->d_todo2.as<int>() + lo, (int)todo_bwt.size(), c->d_work.as<u8>(), c->d_lz.as<u8>(), c->d_lzlen.as<u32>());
          ++c->launches;
        }
      }
      tstop(c, 3);
    }
    if (!todo_hash.empty()) {
      const int nt = (int)todo_hash.size();
      ZQ_CUDA(c, c->d_ht.ensure(htbytes));
      ZQ_CUDA(c, cudaMemsetAsync(c->d_ht.p, 0, htbytes, c->stream));
      ZQ_CUDA(c, c->d_todo4.ensure((size_t)nt * 4));
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo4.p, todo_hash.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, c->stream));
      u32* ctr = c->d_err.as<u32>() + 9;
      ZQ_CUDA(c, cudaMemsetAsync(ctr, 0, 4, c->stream));
      if (todo_sa.empty()) tstart(c, 3);
      k_lz77_hash<8><<<std::min((nt + 3) / 4, c->num_sms * 8), 128, 0, c->stream>>>(
          d_in, du, dp, c->d_todo4.as<int>(), nt, c->d_ht.as<u8>(), c->d_lz.as<u8>(), c->d_lzlen.as<u32>(), c->d_err.as<u32>(), ctr);
      ++c->launches;
      tstop(c, 3);
    }
    if (!todo_cm.empty()) {
      const int nt = (int)todo_cm.size();
      ZQ_CUDA(c, c->d_model.ensure(model));
      ZQ_CUDA(c, c->d_coded.ensure(coded));
      ZQ_CUDA(c, c->d_todo3.ensure((size_t)nt * 4));
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo3.p, todo_cm.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, c->stream));
      u32* ctr = c->d_err.as<u32>() + 8;
      ZQ_CUDA(c, cudaMemsetAsync(ctr, 0, 4, c->stream));
      tstart(c, 5);
      k_cm_init<<<nt * maxjobs, 256, 0, c->stream>>>(du, dp, c->d_cmplans.as<ZqCmPlan>(), c->d_fills.as<ZqCmFill>(), c->d_todo3.as<int>(), nt,
                                                     maxjobs, c->d_tables.as<CmTablesDev>(), c->d_model.as<u8>());
      ++c->launches;
      // ---- optional: translated context program (ZQ_CM_JIT=1) and generated straight-line coder (ZQ_CM_JIT=2), one
      // NVRTC-compiled module per model, cached.  Blocks whose program the translator does not cover stay with
      // k_cm_encode's interpreter; with JIT=2 the others do not go through k_cm_encode at all.
      const u32* d_ctx = nullptr; const u64* d_ctxoff = nullptr;
      std::vector<int> todo_rest = todo_cm;     // what k_cm_encode still has to code
      if (c->cm_jit) {
        std::vector<uint64_t> ctxoff(units.size(), ~(uint64_t)0);     // by unit id, in u32 elements; ~0: interpret
        std::map<u32, std::vector<int>> groups;                       // cm plan -> units of this wave
        for (int ui : todo_cm) groups[dplans[units[w0 + ui].plan].cm_plan].push_back(ui);   // ui: index inside this wave
        struct Launch { zq_ctx::JitProg prog; std::vector<int> ids; u32 plan; };
        std::vector<Launch> launches;
        uint64_t ctx_elems = 0;
        for (auto& g : groups) {
          const ZqCmPlan& cp = cmplans[g.first];
          // the translated program pays off for small models (-m3, 2 components); -m5 (22) is slower with it: its coder is
          // the critical path and the context table of every byte costs traffic
          if (c->cm_jit_auto && cp.n > 8) continue;
          if (cp.n > ZQ_CM_LANES) continue;                                // wide models: one lane does everything (zq_cm_wide.cuh)
          const u8* hc = blob.data() + cp.hcomp_off;
          ZqCmPlan kp = cp; kp.hcomp_off = 0; kp.fill_first = 0;       // per-call positions are not part of the model
          std::string key((const char*)&kp, sizeof(ZqCmPlan));          // components, sizes and table offsets
          key.append((const char*)hc, cp.hcomp_len);
          auto it = c->jit_cache.find(key);
          if (it == c->jit_cache.end()) {
            std::string src, why, log; std::vector<char> cubin;
            zq_ctx::JitProg P;
            if (zq::jit_context_source(hc, cp.hcomp_len, cp.hh, cp.hm, cp.n, src, why) && (c->cm_jit < 2 || zq::jit_coder_source(&cp, src, why)) &&
                zq::jit_compile(src, cubin, log) == 0 &&
                cudaLibraryLoadData(&P.lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0) == cudaSuccess) {
              if (cudaLibraryGetKernel(&P.ctx, P.lib, "zq_ctx_kernel") != cudaSuccess) P.ctx = nullptr;
              if (c->cm_jit < 2 || cudaLibraryGetKernel(&P.code, P.lib, "zq_code_kernel") != cudaSuccess) P.code = nullptr;
            }
            cudaGetLastError();   // a program that could not be built simply stays interpreted
            it = c->jit_cache.emplace(key, P).first;
          }
          if (!it->second.ctx) continue;
          Launch L; L.prog = it->second; L.plan = g.first;
          for (int ui : g.second) {
            const ZqUnit& zu = units[w0 + ui];
            const ZqPlan& p = dplans[zu.plan];
            ctxoff[ui] = ctx_elems;
            ctx_elems += ((uint64_t)p.payload_len + (p.lz_level ? zu.lz_cap : zu.n)) * (uint64_t)cp.n;
            L.ids.push_back(ui);
          }
          launches.push_back(std::move(L));
        }
        if (!launches.empty()) {
          ZQ_CUDA(c, c->d_ctx.ensure(ctx_elems * 4 + 16));
          ZQ_CUDA(c, c->d_ctxoff.ensure(units.size() * 8));
          ZQ_CUDA(c, cudaMemcpyAsync(c->d_ctxoff.p, ctxoff.data(), units.size() * 8, cudaMemcpyHostToDevice, c->stream));
          size_t total = 0;
          for (auto& L : launches) total += L.ids.size();
          // per launch: unit ids | soff | model_off | ctx_off | coded_off | slen | coded_cap   (44 B per unit)
          ZQ_CUDA(c, c->d_ctxargs.ensure(total * 48 + 256 * launches.size() + 256));
          u8* A = c->d_ctxargs.as<u8>();
          size_t at = 0;
          for (auto& L : launches) {
            const int gn = (int)L.ids.size();
            int* d_ids = (int*)(A + at);
            u64* d_soff = (u64*)(A + at + align_up((size_t)gn * 4, 16)); u64* d_moff = d_soff + gn; u64* d_coff = d_moff + gn; u64* d_cdoff = d_coff + gn;
            u32* d_slen = (u32*)(d_cdoff + gn); u32* d_cdcap = d_slen + gn;
            at += align_up((size_t)gn * 48, 256);
            ZQ_CUDA(c, cudaMemcpyAsync(d_ids, L.ids.data(), (size_t)gn * 4, cudaMemcpyHostToDevice, c->stream));
            k_ctx_args<<<(gn + 127) / 128, 128, 0, c->stream>>>(du, dp, d_ids, gn, c->d_lzlen.as<u32>(), c->d_ctxoff.as<u64>(), d_soff, d_slen, d_moff, d_coff,
                                                                d_cdoff, d_cdcap);
            const ZqCmPlan& cp = cmplans[L.plan];
            const ZqPlan& p0 = dplans[units[w0 + L.ids[0]].plan];
            const u8* head = c->d_blob.as<u8>() + p0.payload_off; unsigned hlen = p0.payload_len;
            const u8* sbase = p0.lz_level ? c->d_lz.as<u8>() : d_in;
            u8* mbase = c->d_model.as<u8>(); unsigned long long mo = cp.m_off, ho = cp.h_off, ro = cp.r_off;
            u32* cbase = c->d_ctx.as<u32>(); u32* eflag = c->d_err.as<u32>(); int gnn = gn;
            void* args[] = {&head, &hlen, &sbase, &d_soff, &d_slen, &gnn, &mbase, &d_moff, &mo, &ho, &ro, &cbase, &d_coff, &eflag};
            ZQ_CUDA(c, cudaLaunchKernel((const void*)L.prog.ctx, dim3((gn + 63) / 64), dim3(64), args, 0, c->stream));
            c->launches += 2;
            if (L.prog.code) {
              // the generated coder: lane 0 of every warp codes one block (stride 32), four warps per CTA
              int stride = 32;
              const u8* tabp = c->d_tables.as<u8>(); u8* cdbase = c->d_coded.as<u8>(); u32* cdlen = c->d_codedlen.as<u32>();
              const u32* cbase_c = cbase;
              void* cargs[] = {&head, &hlen, &sbase, &d_soff, &d_slen, &gnn, &stride, &mbase, &d_moff, &cbase_c, &d_coff, &tabp,
                               &cdbase, &d_cdoff, &d_cdcap, &d_ids, &cdlen, &eflag};
              ZQ_CUDA(c, cudaLaunchKernel((const void*)L.prog.code, dim3((gn * stride + 127) / 128), dim3(128), cargs, 0, c->stream));
              ++c->launches;
              for (int ui : L.ids) ctxoff[ui] = ~(uint64_t)0 - 1;   // coded: not k_cm_encode's business
            }
          }
          d_ctx = c->d_ctx.as<u32>(); d_ctxoff = c->d_ctxoff.as<u64>();
          todo_rest.clear();
          for (int ui : todo_cm) if (ctxoff[ui] != ~(uint64_t)0 - 1) todo_rest.push_back(ui);
          if (todo_rest.size() != todo_cm.size() && !todo_rest.empty())
            ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo3.p, todo_rest.data(), todo_rest.size() * 4, cudaMemcpyHostToDevice, c->stream));
        }
      }
      const int nt_enc = (int)todo_rest.size();
      // (coder, context) warp pairs: as many per CTA as spreads the wave over all SMs
      const int pairs = std::max(1, std::min(ZQ_CM_MAX_PAIRS, (nt_enc + c->num_sms - 1) / c->num_sms));
      const size_t cm_smem = sizeof(CmSmem) + (size_t)pairs * sizeof(CmUnitSmem);
      if (!c->attr_cm_enc) {   // per context (= per device): function attributes are per device
        const int cm_smem_max = (int)(sizeof(CmSmem) + ZQ_CM_MAX_PAIRS * sizeof(CmUnitSmem));
        cudaFuncSetAttribute(k_cm_encode<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, cm_smem_max);
        cudaFuncSetAttribute(k_cm_encode<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, cm_smem_max);
        c->attr_cm_enc = true;
      }
      auto cmk = d_ctx ? k_cm_encode<0, true> : k_cm_encode<0, false>;
      if (nt_enc > 0)
      cmk<<<std::min((nt_enc + pairs - 1) / pairs, c->num_sms), pairs * 64, cm_smem, c->stream>>>(
          d_in, du, dp, c->d_cmplans.as<ZqCmPlan>(), c->d_todo3.as<int>(), nt_enc, c->d_tables.as<CmTablesDev>(), c->d_blob.as<u8>(),
          c->d_lz.as<u8>(), c->d_lzlen.as<u32>(), c->d_model.as<u8>(), c->d_coded.as<u8>(), c->d_codedlen.as<u32>(), c->d_err.as<u32>(), ctr,
          c->cm_prefetch, c->cm_fast, d_ctx, d_ctxoff);
      ++c->launches;
      tstop(c, 5);
      ZQ_CUDA(c, cudaMemcpyAsync(coded_len_h.data() + w0, c->d_codedlen.p, (size_t)wn * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    if (lzbytes) ZQ_CUDA(c, cudaMemcpyAsync(lz_len_h.data() + w0, c->d_lzlen.p, (size_t)wn * 4, cudaMemcpyDeviceToHost, c->stream));
    if (lzbytes || !todo_cm.empty()) ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
    // final layout of this wave's blocks
    std::vector<uint64_t> ooff(wn);
    std::vector<int> todo_all(wn);
    for (int k = 0; k < wn; ++k) {
      const ZqUnit& zu = units[w0 + k];
      const ZqPlan& p = dplans[zu.plan];
      uint64_t sz;
      if (p.modeled) sz = (uint64_t)zu.prefix_len + coded_len_h[w0 + k] + 4 + (dosha1 ? 21 : 1) + 1;
      else {
        const uint64_t slen = p.lz_level ? lz_len_h[w0 + k] : zu.n;
        sz = unmodeled_block_size(zu.prefix_len, (uint64_t)p.payload_len + slen, dosha1 != 0);
      }
      if (sz > 0xffffffffull) return fail(c, ZQ_E_OUTPUT, "block too large");
      ooff[k] = out_pos; out_off[w0 + k] = out_pos; out_len[w0 + k] = (uint32_t)sz;
      out_pos += sz;
      todo_all[k] = k;
    }
    if (out_pos > out_cap) return fail(c, ZQ_E_OUTPUT, "output buffer too small");
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_outoff.p, ooff.data(), (size_t)wn * 8, cudaMemcpyHostToDevice, c->stream));
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo.p, todo_all.data(), (size_t)wn * 4, cudaMemcpyHostToDevice, c->stream));
    tstart(c, 4);
    k_frame<<<std::min(wn, c->num_sms * 8), 256, 0, c->stream>>>(
        du, dp, c->d_todo.as<int>(), wn, c->d_blob.as<u8>(), d_in, c->d_lz.as<u8>(), c->d_lzlen.as<u32>(),
        c->d_coded.as<u8>(), c->d_codedlen.as<u32>(), dosha1 ? c->d_sha.as<u8>() : nullptr, c->d_outoff.as<u64>(), d_out);
    ++c->launches;
    tstop(c, 4);
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));  // host vectors of this wave go out of scope
    for (int k = 1; k < 16; ++k) {
      float ms = 0;
      if (c->tm[k].used && cudaEventElapsedTime(&ms, c->tm[k].a, c->tm[k].b) == cudaSuccess) stage_ms[k] += ms;
      c->tm[k].used = false;
    }
    w0 = w1;
  }
  tstop(c, 0);
  uint32_t errflag = 0;
  ZQ_CUDA(c, cudaMemcpyAsync(&errflag, c->d_err.p, 4, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  ZQ_CUDA(c, cudaGetLastError());
  if (errflag & 2) return fail(c, ZQ_E_METHOD, "ZPAQL execution error");
  if (errflag) return fail(c, ZQ_E_OUTPUT, "internal: intermediate stream exceeded its bound");
  c->last_ms[0] = 0;
  cudaEventElapsedTime(&c->last_ms[0], c->tm[0].a, c->tm[0].b);
  for (int k = 1; k < 16; ++k) c->last_ms[k] = stage_ms[k];
  return ZQ_OK;
}

static int stage_buffers(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, std::vector<uint64_t>& roff) {
  uint64_t lo = ~0ull, hi = 0;
  for (int i = 0; i < n; ++i) { lo = std::min(lo, off[i]); hi = std::max(hi, off[i] + len[i]); }
  if (hi < lo) hi = lo;
  ZQ_CUDA(c, c->d_in.ensure(hi - lo + 64));
  if (hi > lo) ZQ_CUDA(c, cudaMemcpyAsync(c->d_in.p, base + lo, hi - lo, cudaMemcpyHostToDevice, c->stream));
  roff.resize(n);
  for (int i = 0; i < n; ++i) roff[i] = off[i] - lo;
  return ZQ_OK;
}


// shared front end of the host-pointer hash entry points: stage data, upload (off,len), run, fetch digests
template <class Launch>
static int hash_many(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests, int dlen, Launch launch) {
  if (!c) return ZQ_E_NODEVICE;
  if (n <= 0) return n == 0 ? ZQ_OK : fail(c, ZQ_E_ARG, "bad argument");
  if (!base || !off || !len || !digests) return fail(c, ZQ_E_ARG, "bad argument");
  cudaSetDevice(c->device);
  std::vector<uint64_t> roff;
  int rc = stage_buffers(c, n, base, off, len, roff);
  if (rc) return rc;
  ZQ_CUDA(c, c->d_misc.ensure((size_t)n * 16));
  ZQ_CUDA(c, c->d_sha.ensure((size_t)n * dlen));
  u64* d_off = c->d_misc.as<u64>(); u64* d_len = d_off + n;
  ZQ_CUDA(c, cudaMemcpyAsync(d_off, roff.data(), (size_t)n * 8, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(d_len, len, (size_t)n * 8, cudaMemcpyHostToDevice, c->stream));
  rc = launch(d_off, d_len, roff);
  if (rc) return rc;
  ZQ_CUDA(c, cudaMemcpyAsync(digests, c->d_sha.p, (size_t)n * dlen, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  ZQ_CUDA(c, cudaGetLastError());
  return ZQ_OK;
}

}  // namespace

// =================================================================================================
extern "C" {

const char* zq_version(void) { return "zpaqfranz_b200 0.1 (sm_90a)"; }

zq_ctx* zq_create(int device) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0) {
    g_create_error = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    return nullptr;
  }
  if (device < 0 || device >= ndev) { g_create_error = "bad device index"; return nullptr; }
  if ((e = cudaSetDevice(device)) != cudaSuccess) { g_create_error = cudaGetErrorString(e); return nullptr; }
  zq_ctx* c = new zq_ctx();
  c->device = device;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  c->num_sms = prop.multiProcessorCount;
  // a wave's scratch (work tables, tokens, LZ streams) comes to ~1.6x wave_bytes; 1/16 of the device keeps the four
  // contexts of a zq_pipe of depth 4 within 40 % of an 80 GB H100 (5 GB: ~3 400 blocks of 64 KiB per wave)
  c->wave_bytes = std::max<size_t>(prop.totalGlobalMem / 16, (size_t)64 << 20);
  if (cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess) { g_create_error = "stream creation failed"; delete c; return nullptr; }
  c->stream = c->own_stream;
  for (int k = 0; k < 16; ++k) { cudaEventCreate(&c->tm[k].a); cudaEventCreate(&c->tm[k].b); }
  for (int k = 0; k < 4; ++k) cudaEventCreate(&c->ev[k]);
  if (const char* s = getenv("ZQ_MODEL_BUDGET")) { size_t v = strtoull(s, nullptr, 10); if (v >= 1024) c->model_budget = v; }
  if (const char* s = getenv("ZQ_FRAG_SEG")) { uint64_t v = strtoull(s, nullptr, 10); if (v >= 64) c->frag_seg = v; }
  if (const char* s = getenv("ZQ_CM_PREFETCH")) c->cm_prefetch = atoi(s);
  if (const char* s = getenv("ZQ_CM_FAST")) c->cm_fast = atoi(s);
  if (const char* s = getenv("ZQ_CM_JIT")) { c->cm_jit = atoi(s); c->cm_jit_auto = false; }
  if (const char* s = getenv("ZQ_LZ_OLD")) c->lz_old = atoi(s) ? 1 : 0;
  if (const char* s = getenv("ZQ_SORT16")) c->sort16 = atoi(s);
  if (const char* s = getenv("ZQ_SORT_NT")) c->sort_nt = atoi(s);
  if (const char* s = getenv("ZQ_SORT_MINB")) c->sort_minb = atoi(s);
  if (c->sort_nt != 1024 && c->sort_nt != 512 && c->sort_nt != 256 && c->sort_nt != 128) c->sort_nt = 256;
  if (c->sort_nt == 1024) c->sort_minb = 1;
  else if (c->sort_nt == 512) c->sort_minb = c->sort_minb >= 4 ? 4 : 2;
  else if (c->sort_nt == 256) c->sort_minb = c->sort_minb >= 8 ? 8 : 4;
  else c->sort_minb = c->sort_minb >= 16 ? 16 : 8;
  if (const char* s = getenv("ZQ_WAVE_BYTES")) { size_t v = strtoull(s, nullptr, 10); if (v >= 1024) c->wave_bytes = v; }
  return c;
}

void zq_destroy(zq_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  DevBuf* bufs[] = {&c->d_in, &c->d_out, &c->d_units, &c->d_plans, &c->d_blob, &c->d_todo, &c->d_outoff, &c->d_work, &c->d_ht, &c->d_todo2, &c->d_todo3, &c->d_todo4, &c->d_todo5, &c->d_dec, &c->d_tok, &c->d_bitpos, &c->d_tables, &c->d_cmplans, &c->d_fills, &c->d_model, &c->d_coded, &c->d_codedlen, &c->d_lz, &c->d_lzlen, &c->d_sha, &c->d_kbuf, &c->d_vbuf, &c->d_err, &c->d_misc};
  for (DevBuf* b : bufs) b->release();
  c->d_ctx.release(); c->d_ctxoff.release(); c->d_ctxargs.release();
  for (auto& kv : c->jit_cache) if (kv.second.lib) cudaLibraryUnload(kv.second.lib);
  for (int k = 0; k < 16; ++k) { cudaEventDestroy(c->tm[k].a); cudaEventDestroy(c->tm[k].b); }
  for (int k = 0; k < 4; ++k) cudaEventDestroy(c->ev[k]);
  cudaStreamDestroy(c->own_stream);
  delete c;
}

int zq_set_compute_gate(zq_ctx* c, void (*fn)(void*, int), void* arg) {
  if (!c) return ZQ_E_NODEVICE;
  c->gate_fn = fn; c->gate_arg = arg;
  return ZQ_OK;
}

int zq_set_stream(zq_ctx* c, void* s) {
  if (!c) return ZQ_E_NODEVICE;
  cudaStreamSynchronize(c->stream);
  c->stream = s ? (cudaStream_t)s : c->own_stream;
  return ZQ_OK;
}

const char* zq_last_error(zq_ctx* c) { return c ? c->err.c_str() : g_create_error.c_str(); }

uint64_t zq_compress_bound(uint32_t n) {
  // stored/LZ worst case: n + n/32 + 64 stream bytes, 4 per 64 KiB chunk, prefix <= 13+5+64 KiB header,
  // names <= 2*256, trailer 26. Generous and cheap.
  return (uint64_t)n + n / 16 + 70000;
}

int zq_plan_block(const char* method, const uint8_t* data, uint32_t n, char* expanded, size_t expanded_cap, int args9[9],
                  uint8_t* header, uint32_t* header_len, uint8_t* pcomp, uint32_t* pcomp_len, char* errbuf, size_t errcap) {
  try {
    if (!method || !*method) throw zq::Error("empty method");
    zq::BlockPlan p = zq::plan_block(method, data, n);
    if (expanded && expanded_cap) { strncpy(expanded, p.method.c_str(), expanded_cap - 1); expanded[expanded_cap - 1] = 0; }
    if (args9) memcpy(args9, p.args, 9 * sizeof(int));
    if (header_len) {
      if (header && *header_len >= p.code.header.size()) memcpy(header, p.code.header.data(), p.code.header.size());
      *header_len = (uint32_t)p.code.header.size();
    }
    if (pcomp_len) {
      if (pcomp && *pcomp_len >= p.code.pcomp.size() && !p.code.pcomp.empty()) memcpy(pcomp, p.code.pcomp.data(), p.code.pcomp.size());
      *pcomp_len = (uint32_t)p.code.pcomp.size();
    }
    return ZQ_OK;
  } catch (const zq::Error& e) {
    if (errbuf && errcap) { strncpy(errbuf, e.msg.c_str(), errcap - 1); errbuf[errcap - 1] = 0; }
    return ZQ_E_METHOD;
  }
}

int zq_compress_blocks_device(zq_ctx* c, int n, const uint8_t* d_in, const uint64_t* in_off, const uint32_t* in_len,
                              const char* const* method, const char* const* filename, const char* const* comment,
                              int uniform, int dosha1, uint8_t* d_out, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len) {
  if (!c) return ZQ_E_NODEVICE;
  cudaSetDevice(c->device);
  return compress_core(c, n, d_in, in_off, in_len, method, filename, comment, uniform, dosha1, d_out, out_cap, out_off, out_len, nullptr);
}

}  // extern "C"

namespace {
// host-pointer front end shared by zq_compress_blocks and zq_compress_segments
int compress_host(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                  const char* const* method, const char* const* filename, const char* const* comment,
                  int uniform, int dosha1, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len,
                  const RawModel* raw) {
  if (!c) return ZQ_E_NODEVICE;
  if (n < 0 || (n > 0 && (!in_base || !in_off || !in_len || !out_base))) return fail(c, ZQ_E_ARG, "bad argument");
  if (n == 0) return ZQ_OK;
  cudaSetDevice(c->device);
  // stage the touched range of the arena
  uint64_t lo = ~0ull, hi = 0, bound = 0;
  for (int u = 0; u < n; ++u) {
    lo = std::min(lo, in_off[u]); hi = std::max(hi, in_off[u] + in_len[u]);
    bound += zq_compress_bound(in_len[u]);
  }
  if (hi < lo) hi = lo;
  const uint64_t span = hi - lo;
  ZQ_CUDA(c, c->d_in.ensure(span + 64));
  ZQ_CUDA(c, c->d_out.ensure(std::min<uint64_t>(bound, std::max<uint64_t>(out_cap, 1)) + 64));
  cudaEvent_t e0 = c->ev[0], e1 = c->ev[1], e2 = c->ev[2], e3 = c->ev[3];
  struct CopyTurn {   // several batches in flight copy their inputs one after the other, not all at once at a third of the rate
    zq_ctx* c;
    explicit CopyTurn(zq_ctx* c_) : c(c_) { if (c->gate_fn) { c->gate_fn(c->gate_arg, 2); c->copy_held = true; } }
    ~CopyTurn() { if (c->copy_held) { c->gate_fn(c->gate_arg, 3); c->copy_held = false; } }
  } turn(c);
  cudaEventRecord(e0, c->stream);
  if (span) ZQ_CUDA(c, cudaMemcpyAsync(c->d_in.p, in_base + lo, span, cudaMemcpyHostToDevice, c->stream));
  cudaEventRecord(e1, c->stream);
  std::vector<uint64_t> roff(n);
  for (int u = 0; u < n; ++u) roff[u] = in_off[u] - lo;
  int rc = compress_core(c, n, c->d_in.as<uint8_t>(), roff.data(), in_len, method, filename, comment, uniform, dosha1,
                         c->d_out.as<uint8_t>(), std::min<uint64_t>(c->d_out.cap, out_cap), out_off, out_len, raw);
  if (rc == ZQ_OK) {
    const uint64_t total = out_off[n - 1] + out_len[n - 1];
    cudaEventRecord(e2, c->stream);
    cudaError_t e = cudaMemcpyAsync(out_base, c->d_out.p, total, cudaMemcpyDeviceToHost, c->stream);
    cudaEventRecord(e3, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) rc = fail(c, ZQ_E_NODEVICE, std::string("CUDA error: ") + cudaGetErrorString(e));
    else { cudaEventElapsedTime(&c->last_ms[6], e0, e1); cudaEventElapsedTime(&c->last_ms[7], e2, e3); }
  }
  return rc;
}
}  // namespace

extern "C" {

int zq_compress_blocks(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                       const char* const* method, const char* const* filename, const char* const* comment,
                       int uniform, int dosha1, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len) {
  return compress_host(c, n, in_base, in_off, in_len, method, filename, comment, uniform, dosha1, out_base, out_cap, out_off, out_len, nullptr);
}

int zq_compress_segments(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                         const uint8_t* header, uint32_t header_len, const uint8_t* pcomp, uint32_t pcomp_len,
                         const char* const* filename, const char* const* comment, int uniform,
                         const uint8_t* sha1_digests, int write_tag,
                         uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len) {
  if (!c) return ZQ_E_NODEVICE;
  if (!header || header_len < 8) return fail(c, ZQ_E_ARG, "bad argument");
  RawModel raw;
  try {
    size_t used = 0;
    raw.code = zq::parse_block_header(header, header_len, &used);
  } catch (const zq::Error& e) { return fail(c, ZQ_E_METHOD, e.msg); }
  if (pcomp_len > 65535) return fail(c, ZQ_E_METHOD, "PCOMP too long");
  if (pcomp && pcomp_len) raw.pcomp.assign(pcomp, pcomp + pcomp_len);
  raw.tag = write_tag != 0;
  raw.digests = sha1_digests;
  return compress_host(c, n, in_base, in_off, in_len, nullptr, filename, comment, uniform, sha1_digests != nullptr,
                       out_base, out_cap, out_off, out_len, &raw);
}

const char* zq_model_config(int level) {
  // The two small standard models of the ZPAQ distribution as ZPAQL source (min.cfg, mid.cfg). The reference
  // keeps their assembled bytes in a table (Compressor::startBlock(int), Z:15992-16026); assembling these
  // sources reproduces those bytes (tests/test_oracle_pinned.py).
  static const char* kMin =
      "comp 1 2 0 0 2 0 icm 16 1 isse 19 0 "
      "hcomp *b=a a=0 d=0 hash b-- hash *d=a d++ b-- hash b-- hash *d=a halt end ";
  static const char* kMid =
      "comp 3 3 0 0 8 0 icm 5 1 isse 13 0 2 isse 17 1 3 isse 18 2 4 isse 18 3 5 isse 19 4 "
      "6 match 22 24 7 mix 16 0 7 24 255 "
      "hcomp c++ *c=a b=c a=0 d= 1 hash *d=a b-- d++ hash *d=a b-- d++ hash *d=a b-- d++ hash *d=a "
      "b-- d++ hash *d=a b-- d++ hash b-- hash *d=a d++ a=*c a<<= 8 *d=a halt end ";
  return level == 1 ? kMin : level == 2 ? kMid : nullptr;
}

int zq_assemble_config(const char* config, const int args9[9], uint8_t* header, uint32_t* header_len,
                       uint8_t* pcomp, uint32_t* pcomp_len, char* pcomp_cmd, size_t pcomp_cmd_cap, char* errbuf, size_t errcap) {
  try {
    if (!config) throw zq::Error("no config");
    int args[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (args9) memcpy(args, args9, sizeof args);
    zq::Assembled a = zq::assemble(config, args);
    if (header_len) {
      if (header && *header_len >= a.header.size()) memcpy(header, a.header.data(), a.header.size());
      *header_len = (uint32_t)a.header.size();
    }
    if (pcomp_len) {
      if (pcomp && *pcomp_len >= a.pcomp.size() && !a.pcomp.empty()) memcpy(pcomp, a.pcomp.data(), a.pcomp.size());
      *pcomp_len = (uint32_t)a.pcomp.size();
    }
    if (pcomp_cmd && pcomp_cmd_cap) { strncpy(pcomp_cmd, a.pcomp_cmd.c_str(), pcomp_cmd_cap - 1); pcomp_cmd[pcomp_cmd_cap - 1] = 0; }
    return ZQ_OK;
  } catch (const zq::Error& e) {
    if (errbuf && errcap) { strncpy(errbuf, e.msg.c_str(), errcap - 1); errbuf[errcap - 1] = 0; }
    return ZQ_E_METHOD;
  }
}

// ---- block decompression ---------------------------------------------------------------------------
int zq_decompress_blocks(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                         const uint32_t* expect_len, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len) {
  return zq_decompress_blocks_ex(c, n, in_base, in_off, in_len, expect_len, out_base, out_cap, out_off, out_len, nullptr, nullptr);
}

static int decompress_impl(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                           const uint32_t* expect_len, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len,
                           uint32_t* in_used, uint8_t* sha1_out, bool prefix) {
  using namespace zqdev;
  if (!c) return ZQ_E_NODEVICE;
  if (n < 0 || (n > 0 && (!in_base || !in_off || !in_len || !out_base || !out_off || !out_len))) return fail(c, ZQ_E_ARG, "bad argument");
  if (n == 0) return ZQ_OK;
  cudaSetDevice(c->device);
  static const unsigned char tag[13] = {0x37, 0x6b, 0x53, 0x74, 0xa0, 0x31, 0x83, 0xd3, 0x8c, 0xb2, 0x28, 0xb0, 0xd3};
  std::vector<ZqDecUnit> units(n);
  std::vector<ZqCmPlan> cmplans;
  std::vector<ZqCmFill> fills;
  std::vector<uint8_t> blob;
  std::map<std::string, int> plan_idx;
  uint64_t lo = ~0ull, hi = 0;
  for (int u = 0; u < n; ++u) { lo = std::min(lo, in_off[u]); hi = std::max(hi, in_off[u] + in_len[u]); }
  if (hi < lo) hi = lo;
  uint64_t out_pos = 0;
  try {
    for (int u = 0; u < n; ++u) {
      const uint8_t* b = in_base + in_off[u];
      size_t len = in_len[u], p = 0;
      if (len >= 13 && memcmp(b, tag, 13) == 0) p = 13;
      if (len < p + 5 || b[p] != 'z' || b[p + 1] != 'P' || b[p + 2] != 'Q') return fail(c, ZQ_E_METHOD, "block does not start with a ZPAQ block header");
      const int level = b[p + 3];
      if (level != 1 && level != 2) return fail(c, ZQ_E_METHOD, "unsupported ZPAQ level");
      if (b[p + 4] != 1) return fail(c, ZQ_E_METHOD, "unsupported ZPAQL type");
      p += 5;
      size_t used = 0;
      zq::Assembled code = zq::parse_block_header(b + p, len - p, &used);
      if (level == 1 && code.ncomp == 0) return fail(c, ZQ_E_METHOD, "ZPAQ level 1 requires at least 1 component");
      const std::string key((const char*)b + p, used);
      p += used;
      int pi;
      auto it = plan_idx.find(key);
      if (it != plan_idx.end()) pi = it->second;
      else {
        ZqCmPlan cp = zq::make_cm_plan(code, fills);
        zq::add_pcomp_region(cp, code.ph, code.pm, fills);
        cp.hcomp_off = (u32)blob.size(); cp.hcomp_len = (u32)code.hcomp.size();
        blob.insert(blob.end(), code.hcomp.begin(), code.hcomp.end());
        pi = (int)cmplans.size();
        cmplans.push_back(cp);
        plan_idx[key] = pi;
      }
      if (p >= len || b[p] != 1) return fail(c, ZQ_E_METHOD, "missing segment or end of block");
      ++p;
      while (p < len && b[p]) ++p;   // filename
      if (p >= len) return fail(c, ZQ_E_METHOD, "unexpected EOF");
      ++p;
      const size_t cstart = p;
      while (p < len && b[p]) ++p;   // comment
      if (p + 1 >= len) return fail(c, ZQ_E_METHOD, "unexpected EOF");
      uint64_t expect = 0; bool have = false;
      if (expect_len) { expect = expect_len[u]; have = true; }
      else { size_t q = cstart; while (q < p && isdigit(b[q])) { expect = expect * 10 + (b[q] - '0'); ++q; have = true; } }
      if (!have || expect > 0xfffffff0ull) return fail(c, ZQ_E_ARG, "block size unknown: pass expect_len (segment comment carries no size)");
      ++p;
      if (b[p] != 0) return fail(c, ZQ_E_METHOD, "missing reserved byte");
      ++p;
      ZqDecUnit& du = units[u];
      du.data_off = in_off[u] - lo + p; du.data_len = len - p; du.out_off = out_pos; du.out_cap = (u32)expect; du.plan = (u32)pi; du.model_off = 0;
      out_off[u] = out_pos; out_pos += expect;
    }
  } catch (const zq::Error& e) { return fail(c, ZQ_E_METHOD, e.msg); }
  if (out_pos > out_cap) return fail(c, ZQ_E_OUTPUT, "output buffer too small");
  if (!c->d_tables.p) {
    try {
      const zq::CmTables& t = zq::cm_tables();
      ZQ_CUDA(c, c->d_tables.ensure(sizeof(zq::CmTables)));
      ZQ_CUDA(c, cudaMemcpyAsync(c->d_tables.p, &t, sizeof t, cudaMemcpyHostToDevice, c->stream));
    } catch (const zq::Error& e) { return fail(c, ZQ_E_METHOD, e.msg); }
  }
  ZQ_CUDA(c, c->d_in.ensure(hi - lo + 64));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_in.p, in_base + lo, hi - lo, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, c->d_out.ensure(out_pos + 64));
  ZQ_CUDA(c, c->d_blob.ensure(blob.size() + 16));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_blob.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, c->d_cmplans.ensure(cmplans.size() * sizeof(ZqCmPlan)));
  ZQ_CUDA(c, c->d_fills.ensure(fills.size() * sizeof(ZqCmFill)));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_cmplans.p, cmplans.data(), cmplans.size() * sizeof(ZqCmPlan), cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_fills.p, fills.data(), fills.size() * sizeof(ZqCmFill), cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, c->d_err.ensure(64));
  size_t budget = c->model_budget;
  { size_t fr = 0, tot = 0; cudaMemGetInfo(&fr, &tot); fr += c->d_model.cap; budget = std::min<size_t>(budget, fr > ((size_t)6 << 30) ? fr - ((size_t)6 << 30) : fr / 2); }
  std::vector<ZqDecResult> res(n);
  // segments that are followed by another one in their block are reported through a table (most blocks have none)
  const u32 segcap = (u32)std::min<uint64_t>((uint64_t)n + 65536, 1u << 24);
  ZQ_CUDA(c, c->d_kbuf.ensure(16 + (size_t)segcap * sizeof(ZqDecSeg)));
  u32* d_nseg = c->d_kbuf.as<u32>(); ZqDecSeg* d_segs = (ZqDecSeg*)(c->d_kbuf.as<u8>() + 16);
  ZQ_CUDA(c, cudaMemsetAsync(d_nseg, 0, 16, c->stream));
  const size_t dec_smem = sizeof(CmSmem) + 16 * sizeof(CmUnitSmem);
  if (!c->attr_cm_dec) {
    cudaFuncSetAttribute(k_cm_decode<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dec_smem);
    c->attr_cm_dec = true;
  }
  auto cmd = k_cm_decode<0>;
  int w0 = 0;
  while (w0 < n) {
    size_t model = 0; int w1 = w0, maxjobs = 1;
    std::vector<uint64_t> moff; std::vector<uint32_t> pof;
    while (w1 < n) {
      const ZqCmPlan& cp = cmplans[units[w1].plan];
      if (w1 > w0 && model + cp.model_bytes > budget) break;
      units[w1].model_off = model; model += cp.model_bytes;
      moff.push_back(units[w1].model_off); pof.push_back(units[w1].plan);
      maxjobs = std::max(maxjobs, (int)cp.fill_count);
      ++w1;
    }
    const int wn = w1 - w0;
    ZQ_CUDA(c, c->d_model.ensure(model));
    ZQ_CUDA(c, c->d_units.ensure((size_t)wn * sizeof(ZqDecUnit)));
    ZQ_CUDA(c, c->d_misc.ensure((size_t)wn * 12 + (size_t)wn * sizeof(ZqDecResult) + 256));
    u64* d_moff = c->d_misc.as<u64>(); u32* d_pof = (u32*)(d_moff + wn); ZqDecResult* d_res = (ZqDecResult*)(c->d_misc.as<u8>() + align_up((size_t)wn * 12, 16));
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_units.p, units.data() + w0, (size_t)wn * sizeof(ZqDecUnit), cudaMemcpyHostToDevice, c->stream));
    ZQ_CUDA(c, cudaMemcpyAsync(d_moff, moff.data(), (size_t)wn * 8, cudaMemcpyHostToDevice, c->stream));
    ZQ_CUDA(c, cudaMemcpyAsync(d_pof, pof.data(), (size_t)wn * 4, cudaMemcpyHostToDevice, c->stream));
    u32* ctr = c->d_err.as<u32>() + 10;
    ZQ_CUDA(c, cudaMemsetAsync(ctr, 0, 4, c->stream));
    k_cm_init_pairs<<<wn * maxjobs, 256, 0, c->stream>>>(d_moff, d_pof, c->d_cmplans.as<ZqCmPlan>(), c->d_fills.as<ZqCmFill>(), wn, maxjobs,
                                                        c->d_tables.as<CmTablesDev>(), c->d_model.as<u8>());
    ++c->launches;
    cmd<<<std::min((wn + 15) / 16, c->num_sms), 512, dec_smem, c->stream>>>(
        c->d_in.as<u8>(), c->d_units.as<ZqDecUnit>(), c->d_cmplans.as<ZqCmPlan>(), wn, c->d_tables.as<CmTablesDev>(), c->d_blob.as<u8>(),
        c->d_model.as<u8>(), c->d_out.as<u8>(), d_res, ctr, c->cm_fast, d_segs, d_nseg, segcap, (u32)w0);
    ++c->launches;
    ZQ_CUDA(c, cudaMemcpyAsync(res.data() + w0, d_res, (size_t)wn * sizeof(ZqDecResult), cudaMemcpyDeviceToHost, c->stream));
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
    ZQ_CUDA(c, cudaGetLastError());
    w0 = w1;
  }
  // results, trailers, checksums
  u32 nseg = 0;
  ZQ_CUDA(c, cudaMemcpyAsync(&nseg, d_nseg, 4, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  std::vector<ZqDecSeg> inner(std::min(nseg, segcap));
  if (!inner.empty()) {
    ZQ_CUDA(c, cudaMemcpyAsync(inner.data(), d_segs, inner.size() * sizeof(ZqDecSeg), cudaMemcpyDeviceToHost, c->stream));
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
    std::sort(inner.begin(), inner.end(), [](const ZqDecSeg& a, const ZqDecSeg& b) { return a.unit != b.unit ? a.unit < b.unit : a.trailer < b.trailer; });
  }
  c->last_segs.clear();
  std::vector<uint64_t> soff; std::vector<uint64_t> slen; std::vector<const uint8_t*> swant;
  size_t ip = 0;
  for (int u = 0; u < n; ++u) {
    const ZqDecResult& r = res[u];
    static const char* msg[] = {"", "archive corrupted", "unexpected end of file", "decoded size exceeds the expected size", "ZPAQL execution error", "unknown post processing type", "too many segments in one call"};
    const uint8_t* b = in_base + in_off[u];
    const size_t data0 = (size_t)(units[u].data_off + lo - in_off[u]);     // offset of the first coded byte in the block
    uint32_t seg_begin = 0;
    for (; ip < inner.size() && inner[ip].unit == (u32)u; ++ip) {          // the segments before the last one
      const ZqDecSeg& sg = inner[ip];
      const size_t p = data0 + sg.trailer;
      zq_segment zs; zs.block = (uint32_t)u; zs.out_begin = seg_begin; zs.out_end = sg.out_end; zs.trailer = (uint32_t)p;
      c->last_segs.push_back(zs);
      if (b[p] == 253) { soff.push_back(units[u].out_off + seg_begin); slen.push_back(sg.out_end - seg_begin); swant.push_back(b + p + 1); }
      seg_begin = sg.out_end;
    }
    if (prefix && (r.error == 3 || r.error == 0)) {   // Decompresser::decompress(n): stop after n bytes, no trailer is looked at
      out_len[u] = std::min<uint32_t>(r.out_len, units[u].out_cap);   // (the writer counts the byte that did not fit)
      if (in_used) in_used[u] = 0;
      if (sha1_out) sha1_out[(size_t)u * 21] = 0;
      continue;
    }
    if (r.error) return fail(c, r.error == 3 ? ZQ_E_OUTPUT : r.error == 6 ? ZQ_E_UNSUPPORTED : ZQ_E_METHOD, msg[r.error < 7 ? r.error : 1]);
    out_len[u] = r.out_len;
    const size_t p = data0 + r.consumed;
    if (p >= in_len[u]) return fail(c, ZQ_E_METHOD, "missing end of segment marker");
    if (b[p] == 253) {
      if (p + 21 > in_len[u]) return fail(c, ZQ_E_METHOD, "unexpected EOF");
      soff.push_back(units[u].out_off + seg_begin); slen.push_back(r.out_len - seg_begin); swant.push_back(b + p + 1);
    } else if (b[p] != 254) return fail(c, ZQ_E_METHOD, "missing end of segment marker");
    { zq_segment zs; zs.block = (uint32_t)u; zs.out_begin = seg_begin; zs.out_end = r.out_len; zs.trailer = (uint32_t)p; c->last_segs.push_back(zs); }
    const size_t e = p + (b[p] == 253 ? 21 : 1);
    if (e < in_len[u] && b[e] == 1) return fail(c, ZQ_E_METHOD, "segment header corrupted");
    if (in_used) in_used[u] = (uint32_t)e;       // offset of the end-of-block byte (255)
    if (sha1_out) { sha1_out[(size_t)u * 21] = b[p] == 253; if (b[p] == 253) memcpy(sha1_out + (size_t)u * 21 + 1, b + p + 1, 20); }
  }
  if (!soff.empty()) {
    const int k = (int)soff.size();
    ZQ_CUDA(c, c->d_misc.ensure((size_t)k * 16));
    ZQ_CUDA(c, c->d_sha.ensure((size_t)k * 20));
    u64* d_off = c->d_misc.as<u64>(); u64* d_len = d_off + k;
    ZQ_CUDA(c, cudaMemcpyAsync(d_off, soff.data(), (size_t)k * 8, cudaMemcpyHostToDevice, c->stream));
    ZQ_CUDA(c, cudaMemcpyAsync(d_len, slen.data(), (size_t)k * 8, cudaMemcpyHostToDevice, c->stream));
    k_sha1_many<<<(k + 127) / 128, 128, 0, c->stream>>>(c->d_out.as<u8>(), d_off, nullptr, d_len, k, c->d_sha.as<u8>());
    ++c->launches;
    std::vector<uint8_t> dg((size_t)k * 20);
    ZQ_CUDA(c, cudaMemcpyAsync(dg.data(), c->d_sha.p, dg.size(), cudaMemcpyDeviceToHost, c->stream));
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
    for (int i = 0; i < k; ++i)
      if (memcmp(swant[i], dg.data() + (size_t)i * 20, 20) != 0) return fail(c, ZQ_E_METHOD, "SHA-1 checksum mismatch after decompression");
  }
  if (out_pos) ZQ_CUDA(c, cudaMemcpy(out_base, c->d_out.p, out_pos, cudaMemcpyDeviceToHost));
  return ZQ_OK;
}

int zq_decompress_blocks_ex(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                            const uint32_t* expect_len, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len,
                            uint32_t* in_used, uint8_t* sha1_out) {
  return decompress_impl(c, n, in_base, in_off, in_len, expect_len, out_base, out_cap, out_off, out_len, in_used, sha1_out, false);
}

int zq_decompress_last_segments(zq_ctx* c, const zq_segment** segs, uint64_t* nsegs) {
  if (!c) return ZQ_E_NODEVICE;
  if (!segs || !nsegs) return fail(c, ZQ_E_ARG, "bad argument");
  *segs = c->last_segs.data(); *nsegs = c->last_segs.size();
  return ZQ_OK;
}

int zq_decompress_prefix(zq_ctx* c, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                         const uint32_t* max_out, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len) {
  if (c && n > 0 && !max_out) return fail(c, ZQ_E_ARG, "bad argument");
  return decompress_impl(c, n, in_base, in_off, in_len, max_out, out_base, out_cap, out_off, out_len, nullptr, nullptr, true);
}

// ---- hashes --------------------------------------------------------------------------------------
int zq_sha1_device(zq_ctx* c, int n, const uint8_t* d_base, const uint64_t* off, const uint64_t* len, uint8_t* d_digests) {
  if (!c) return ZQ_E_NODEVICE;
  if (n <= 0) return n == 0 ? ZQ_OK : fail(c, ZQ_E_ARG, "bad argument");
  cudaSetDevice(c->device);
  ZQ_CUDA(c, c->d_misc.ensure((size_t)n * 16));
  u64* d_off = c->d_misc.as<u64>(); u64* d_len = d_off + n;
  ZQ_CUDA(c, cudaMemcpyAsync(d_off, off, (size_t)n * 8, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(d_len, len, (size_t)n * 8, cudaMemcpyHostToDevice, c->stream));
  zqdev::k_sha1_many<<<(n + 127) / 128, 128, 0, c->stream>>>(d_base, d_off, nullptr, d_len, n, d_digests);
  ++c->launches;
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  ZQ_CUDA(c, cudaGetLastError());
  return ZQ_OK;
}

int zq_sha1(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  if (!c) return ZQ_E_NODEVICE;
  if (n <= 0) return n == 0 ? ZQ_OK : fail(c, ZQ_E_ARG, "bad argument");
  cudaSetDevice(c->device);
  std::vector<uint64_t> roff;
  int rc = stage_buffers(c, n, base, off, len, roff);
  if (rc) return rc;
  ZQ_CUDA(c, c->d_sha.ensure((size_t)n * 20));
  rc = zq_sha1_device(c, n, c->d_in.as<uint8_t>(), roff.data(), len, c->d_sha.as<uint8_t>());
  if (rc) return rc;
  ZQ_CUDA(c, cudaMemcpy(digests, c->d_sha.p, (size_t)n * 20, cudaMemcpyDeviceToHost));
  return ZQ_OK;
}

int zq_sha256(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 32, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) {
    zqdev::k_sha256_many<<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, n, c->d_sha.as<u8>());
    ++c->launches;
    return ZQ_OK;
  });
}

int zq_xxh3_128(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 16, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) {
    zqdev::k_xxh3_128_many<<<(n + 3) / 4, 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, n, c->d_sha.as<u8>());
    ++c->launches;
    return ZQ_OK;
  });
}

int zq_blake3(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 32, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) -> int {
    std::vector<uint64_t> first(n + 1);
    std::vector<int> multi;
    uint64_t tot = 0;
    for (int i = 0; i < n; ++i) {
      first[i] = tot;
      const uint64_t k = len[i] ? (len[i] + 1023) / 1024 : 1;
      if (k > 1) multi.push_back(i);
      tot += k;
    }
    first[n] = tot;
    ZQ_CUDA(c, c->d_work.ensure(tot * 64 + (size_t)(n + 1) * 8 + multi.size() * 4 + 1024));
    u8* W = c->d_work.as<u8>();
    u32* cvA = (u32*)W; u32* cvB = (u32*)(W + tot * 32);
    u64* d_first = (u64*)(W + tot * 64); int* d_multi = (int*)(W + tot * 64 + (size_t)(n + 1) * 8);
    ZQ_CUDA(c, cudaMemcpyAsync(d_first, first.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    if (!multi.empty()) ZQ_CUDA(c, cudaMemcpyAsync(d_multi, multi.data(), multi.size() * 4, cudaMemcpyHostToDevice, c->stream));
    zqdev::k_blake3_chunks<<<(unsigned)((tot + 127) / 128), 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, d_first, n, tot, cvA, c->d_sha.as<u8>());
    ++c->launches;
    if (!multi.empty()) {
      zqdev::k_blake3_tree<<<(int)std::min<size_t>(multi.size(), (size_t)c->num_sms * 8), 256, 0, c->stream>>>(d_first, d_multi, (int)multi.size(), cvA, cvB, c->d_sha.as<u8>());
      ++c->launches;
    }
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));   // host vectors go out of scope
    return ZQ_OK;
  });
}

// CRC-32 slice tables and the "advance through 4 KiB of zeros" operator (see zq_hashes2.cuh)
static const zqdev::CrcTables& crc_tables() {
  // built once, by whichever thread comes first (C++11 magic static: contexts on several host threads may race here)
  static const zqdev::CrcTables t = [] {
    zqdev::CrcTables t;
    for (uint32_t v = 0; v < 256; ++v) {
      uint32_t c = v;
      for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
      t.T[0][v] = c;
    }
    for (uint32_t v = 0; v < 256; ++v)
      for (int k = 1; k < 4; ++k) t.T[k][v] = (t.T[k - 1][v] >> 8) ^ t.T[0][t.T[k - 1][v] & 255];
    for (int k = 0; k < 4; ++k)
      for (uint32_t v = 0; v < 256; ++v) {
        uint32_t s = v << (8 * k);
        for (uint32_t z = 0; z < zqdev::CRC_CHUNK; ++z) s = t.T[0][s & 255] ^ (s >> 8);
        t.Z[k][v] = s;
      }
    return t;
  }();
  return t;
}

int zq_crc32(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 4, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) -> int {
    std::vector<uint64_t> first(n + 1);
    uint64_t tot = 0;
    for (int i = 0; i < n; ++i) { first[i] = tot; tot += (len[i] + zqdev::CRC_CHUNK - 1) / zqdev::CRC_CHUNK; }
    first[n] = tot;
    ZQ_CUDA(c, c->d_work.ensure(tot * 4 + (size_t)(n + 1) * 8 + sizeof(zqdev::CrcTables) + 1024));
    u8* W = c->d_work.as<u8>();
    zqdev::CrcTables* d_tab = (zqdev::CrcTables*)W;
    u64* d_first = (u64*)(W + sizeof(zqdev::CrcTables)); u32* d_part = (u32*)(d_first + n + 1);
    const zqdev::CrcTables& t = crc_tables();
    ZQ_CUDA(c, cudaMemcpyAsync(d_tab, &t, sizeof t, cudaMemcpyHostToDevice, c->stream));
    ZQ_CUDA(c, cudaMemcpyAsync(d_first, first.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    if (tot) {
      zqdev::k_crc32_chunks<<<(unsigned)((tot + 127) / 128), 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, d_first, n, tot, d_tab, d_part);
      ++c->launches;
    }
    zqdev::k_crc32_fold<<<(n + 127) / 128, 128, 0, c->stream>>>(d_len, d_first, n, d_tab, d_part, c->d_sha.as<u32>());
    ++c->launches;
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));   // host vectors go out of scope
    return ZQ_OK;
  });
}

int zq_xxh64(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 8, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) {
    zqdev::k_xxh64_many<<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, n, c->d_sha.as<u64>());
    ++c->launches;
    return ZQ_OK;
  });
}

// MD5 / SHA3-256 of n buffers (Jidac::updatehash with -md5 / -sha3: MD5::add Z:21616, SHA3::add Z:21337)
int zq_md5(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 16, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) -> int {
    static const zqdev::Md5Consts K = [] {      // floor(2^32 |sin(i+1)|), RFC 1321 section 3.4
      zqdev::Md5Consts k;
      for (int i = 0; i < 64; ++i) k.K[i] = (uint32_t)(long long)floor(fabs(sin((double)(i + 1))) * 4294967296.0);
      return k;
    }();
    ZQ_CUDA(c, c->d_tok.ensure(sizeof K));
    ZQ_CUDA(c, cudaMemcpyAsync(c->d_tok.p, &K, sizeof K, cudaMemcpyHostToDevice, c->stream));
    zqdev::k_md5_many<<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, n, c->d_tok.as<zqdev::Md5Consts>(), c->d_sha.as<u8>());
    ++c->launches;
    return ZQ_OK;
  });
}

int zq_sha3_256(zq_ctx* c, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests) {
  return hash_many(c, n, base, off, len, digests, 32, [&](u64* d_off, u64* d_len, std::vector<uint64_t>&) {
    zqdev::k_sha3_256_many<<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_in.as<u8>(), d_off, d_len, n, c->d_sha.as<u8>());
    ++c->launches;
    return ZQ_OK;
  });
}

// state: 5 (SHA-1) or 8 (SHA-256) chaining words, host; data: nblocks * 64 bytes, host
static int hash_continue(zq_ctx* c, int words, uint32_t* state, const uint8_t* data, uint64_t nblocks) {
  using namespace zqdev;
  if (!c) return ZQ_E_NODEVICE;
  if (!state || (nblocks && !data)) return fail(c, ZQ_E_ARG, "bad argument");
  if (nblocks == 0) return ZQ_OK;
  cudaSetDevice(c->device);
  ZQ_CUDA(c, c->d_in.ensure(nblocks * 64 + 64));
  ZQ_CUDA(c, c->d_sha.ensure(64));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_in.p, data, nblocks * 64, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_sha.p, state, (size_t)words * 4, cudaMemcpyHostToDevice, c->stream));
  if (words == 5) k_sha1_continue<<<1, 1, 0, c->stream>>>(c->d_in.as<u8>(), nblocks, c->d_sha.as<u32>());
  else k_sha256_continue<<<1, 1, 0, c->stream>>>(c->d_in.as<u8>(), nblocks, c->d_sha.as<u32>());
  ++c->launches;
  ZQ_CUDA(c, cudaMemcpyAsync(state, c->d_sha.p, (size_t)words * 4, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  return ZQ_OK;
}
int zq_sha1_continue(zq_ctx* c, uint32_t state[5], const uint8_t* data, uint64_t nblocks) { return hash_continue(c, 5, state, data, nblocks); }
int zq_sha256_continue(zq_ctx* c, uint32_t state[8], const uint8_t* data, uint64_t nblocks) { return hash_continue(c, 8, state, data, nblocks); }

int zq_dedup_first(zq_ctx* c, uint64_t n, const uint8_t* sha1, uint32_t* first) {
  using namespace zqdev;
  if (!c) return ZQ_E_NODEVICE;
  if (n > 0x7fffffffu || (n > 0 && (!sha1 || !first))) return fail(c, ZQ_E_ARG, "bad argument");
  if (n == 0) return ZQ_OK;
  cudaSetDevice(c->device);
  u32 slots = 1024;
  while (slots < 2 * n) slots <<= 1;
  ZQ_CUDA(c, c->d_sha.ensure(n * 20));
  ZQ_CUDA(c, c->d_ht.ensure((size_t)slots * 4));
  ZQ_CUDA(c, c->d_tok.ensure(n * 4));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_sha.p, sha1, n * 20, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemsetAsync(c->d_ht.p, 0xff, (size_t)slots * 4, c->stream));
  const u32 grid = (u32)((n + 255) / 256);
  k_dedup_insert<<<grid, 256, 0, c->stream>>>(c->d_sha.as<u32>(), (u32)n, c->d_ht.as<u32>(), slots - 1);
  k_dedup_lookup<<<grid, 256, 0, c->stream>>>(c->d_sha.as<u32>(), (u32)n, c->d_ht.as<u32>(), slots - 1, c->d_tok.as<u32>());
  c->launches += 2;
  ZQ_CUDA(c, cudaMemcpyAsync(first, c->d_tok.p, n * 4, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  return ZQ_OK;
}

int zq_fragment(zq_ctx* c, int nfiles, const uint8_t* base, const uint64_t* off, const uint64_t* len, int fragment,
                uint32_t blocksize, uint32_t* frag_len, uint32_t* frag_hits, uint8_t* frag_sha1, uint64_t frag_cap,
                uint64_t* frag_first) {
  return zq_fragment_ex(c, nfiles, base, off, len, fragment, blocksize, frag_len, frag_hits, frag_sha1, nullptr, frag_cap, frag_first);
}

int zq_fragment_ex(zq_ctx* c, int nfiles, const uint8_t* base, const uint64_t* off, const uint64_t* len, int fragment,
                   uint32_t blocksize, uint32_t* frag_len, uint32_t* frag_hits, uint8_t* frag_sha1, uint8_t* frag_o1,
                   uint64_t frag_cap, uint64_t* frag_first) {
  using namespace zqdev;
  if (!c) return ZQ_E_NODEVICE;
  if (nfiles < 0 || (nfiles > 0 && (!base || !off || !len)) || !frag_first || fragment < 0 || blocksize < 64)
    return fail(c, ZQ_E_ARG, "bad argument");
  cudaSetDevice(c->device);
  // constants exactly as Jidac::add derives them (Z:121626-121631)
  uint64_t maxf64 = fragment <= 19 ? ((uint64_t)8128 << fragment) : (uint64_t)blocksize - 12;
  if (maxf64 > (uint64_t)blocksize - 12) maxf64 = blocksize - 12;
  uint64_t minf64 = fragment <= 25 ? ((uint64_t)64 << fragment) : maxf64;
  if (minf64 > maxf64) minf64 = maxf64;
  const uint32_t maxf = (uint32_t)maxf64, minf = (uint32_t)minf64;
  const uint32_t thresh = fragment <= 22 ? (1u << (22 - fragment)) : 0u;
  frag_first[0] = 0;
  if (nfiles == 0) return ZQ_OK;
  std::vector<uint64_t> roff;
  int rc = stage_buffers(c, nfiles, base, off, len, roff);
  if (rc) return rc;
  // segments
  uint64_t seg = c->frag_seg;
  if (seg < minf) seg = minf;
  std::vector<ZqSeg> segs;
  std::vector<uint32_t> seg_first_of_file(nfiles + 1, 0);
  for (int f = 0; f < nfiles; ++f) {
    seg_first_of_file[f] = (uint32_t)segs.size();
    for (uint64_t p = 0; p < len[f]; p += seg) {
      ZqSeg sg; sg.begin = roff[f] + p; sg.end = roff[f] + std::min<uint64_t>(len[f], p + seg); sg.file_end = roff[f] + len[f];
      sg.first = p == 0; sg.pad = 0;
      segs.push_back(sg);
    }
  }
  seg_first_of_file[nfiles] = (uint32_t)segs.size();
  const int nseg = (int)segs.size();
  if (nseg == 0) { for (int f = 0; f <= nfiles; ++f) frag_first[f] = 0; return ZQ_OK; }
  const uint32_t cap = (uint32_t)((seg + maxf) / std::max<uint32_t>(minf, 1) + 3);
  const size_t per = (size_t)nseg * cap;
  // layout in d_work: segs | exitA exitB entry | bndA bndB | hitsA hitsB | cntA cntB | flags
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  const size_t o_segs = take(sizeof(ZqSeg) * nseg), o_exA = take(8 * (size_t)nseg), o_exB = take(8 * (size_t)nseg), o_ent = take(8 * (size_t)nseg);
  const size_t o_bA = take(8 * per), o_bB = take(8 * per), o_hA = take(4 * per), o_hB = take(4 * per);
  const size_t o_cA = take(4 * (size_t)nseg), o_cB = take(4 * (size_t)nseg), o_fl = take(64), o_first = take(8 * (size_t)nseg);
  const size_t o_cv = take(4 * (size_t)nseg), o_ce = take(8 * (size_t)nseg), o_lv = take(4 * 256), o_hv = take(4 * 256), o_rf = take(4 * (size_t)nseg);
  ZQ_CUDA(c, c->d_work.ensure(o));
  u8* W = c->d_work.as<u8>();
  ZQ_CUDA(c, cudaMemcpyAsync(W + o_segs, segs.data(), sizeof(ZqSeg) * nseg, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemsetAsync(W + o_fl, 0, 64, c->stream));
  int cur = 0;
  for (int round = 0; round <= nseg; ++round) {
    ZQ_CUDA(c, cudaMemsetAsync(W + o_fl, 0, 4, c->stream));
    const size_t exP = cur ? o_exB : o_exA, exN = cur ? o_exA : o_exB, bP = cur ? o_bB : o_bA, bN = cur ? o_bA : o_bB;
    const size_t hP = cur ? o_hB : o_hA, hN = cur ? o_hA : o_hB, cP = cur ? o_cB : o_cA, cN = cur ? o_cA : o_cB;
    k_fragment_round<<<(nseg + FRAG_THREADS - 1) / FRAG_THREADS, FRAG_THREADS, 0, c->stream>>>(
        c->d_in.as<u8>(), (const ZqSeg*)(W + o_segs), nseg, round, minf, maxf, thresh, cap, (const u64*)(W + exP), (u64*)(W + exN),
        (u64*)(W + o_ent), (const u64*)(W + bP), (const u32*)(W + hP), (const u32*)(W + cP), (u64*)(W + bN), (u32*)(W + hN),
        (u32*)(W + cN), (u32*)(W + o_fl), (u32*)(W + o_fl + 4), (u32*)(W + o_cv), (const u64*)(W + o_ce), (const u32*)(W + o_rf),
        (const u32*)(W + o_lv), (const u32*)(W + o_hv));
    ++c->launches;
    cur ^= 1;
    if (round == 0) {   // constant segments -> end of the constant run they belong to (same value, same file)
      std::vector<uint32_t> cv(nseg);
      ZQ_CUDA(c, cudaMemcpyAsync(cv.data(), W + o_cv, 4 * (size_t)nseg, cudaMemcpyDeviceToHost, c->stream));
      ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
      std::vector<uint64_t> ce(nseg, 0);
      std::vector<uint32_t> rf(nseg);
      for (int k = nseg - 1; k >= 0; --k)
        if (cv[k] < 256) ce[k] = (k + 1 < nseg && !segs[k + 1].first && cv[k + 1] == cv[k]) ? ce[k + 1] : segs[k].end;
      for (int k = 0; k < nseg; ++k)
        rf[k] = (cv[k] < 256 && k > 0 && !segs[k].first && cv[k - 1] == cv[k]) ? rf[k - 1] : (uint32_t)k;
      ZQ_CUDA(c, cudaMemcpyAsync(W + o_ce, ce.data(), 8 * (size_t)nseg, cudaMemcpyHostToDevice, c->stream));
      ZQ_CUDA(c, cudaMemcpyAsync(W + o_rf, rf.data(), 4 * (size_t)nseg, cudaMemcpyHostToDevice, c->stream));
      bool any = false;
      for (int k = 0; k < nseg && !any; ++k) any = cv[k] < 256;
      if (any) {   // the fragment a fresh machine cuts from an endless run of each byte value
        k_fragment_const_table<<<1, 256, 0, c->stream>>>(minf, maxf, thresh, (u32*)(W + o_lv), (u32*)(W + o_hv));
        ++c->launches;
      }
    }
    uint32_t flags[2] = {0, 0};
    ZQ_CUDA(c, cudaMemcpyAsync(flags, W + o_fl, 8, cudaMemcpyDeviceToHost, c->stream));
    ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
    if (flags[1]) return fail(c, ZQ_E_OUTPUT, "internal: fragment table overflow");
    if (!flags[0]) break;
  }
  // current chains are in the buffers last written ("next" of the final round) == index cur^1 ... after the flip: prev set
  const size_t bF = cur ? o_bB : o_bA, hF = cur ? o_hB : o_hA, cF = cur ? o_cB : o_cA;
  std::vector<uint32_t> cnt(nseg);
  ZQ_CUDA(c, cudaMemcpyAsync(cnt.data(), W + cF, 4 * (size_t)nseg, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  std::vector<uint64_t> first(nseg);
  uint64_t total = 0;
  for (int f = 0; f < nfiles; ++f) {
    frag_first[f] = total;
    for (uint32_t k = seg_first_of_file[f]; k < seg_first_of_file[f + 1]; ++k) { first[k] = total; total += cnt[k]; }
  }
  frag_first[nfiles] = total;
  if (total > frag_cap) return fail(c, ZQ_E_OUTPUT, "fragment arrays too small");
  if (total == 0) return ZQ_OK;
  ZQ_CUDA(c, cudaMemcpyAsync(W + o_first, first.data(), 8 * (size_t)nseg, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, c->d_misc.ensure(total * 16));
  u32* d_fl = c->d_misc.as<u32>(); u32* d_fh = d_fl + total; u64* d_fo = (u64*)(d_fh + total);
  k_fragment_gather<<<(nseg + 127) / 128, 128, 0, c->stream>>>((const ZqSeg*)(W + o_segs), nseg, cap, (const u64*)(W + bF), (const u32*)(W + hF),
                                                               (const u32*)(W + cF), (const u64*)(W + o_first), (const u64*)(W + o_ent), d_fl, d_fh, d_fo);
  ++c->launches;
  if (frag_len) ZQ_CUDA(c, cudaMemcpyAsync(frag_len, d_fl, total * 4, cudaMemcpyDeviceToHost, c->stream));
  if (frag_hits) ZQ_CUDA(c, cudaMemcpyAsync(frag_hits, d_fh, total * 4, cudaMemcpyDeviceToHost, c->stream));
  if (frag_sha1) {
    ZQ_CUDA(c, c->d_sha.ensure(total * 20));
    k_sha1_many<<<(int)((total + 127) / 128), 128, 0, c->stream>>>(c->d_in.as<u8>(), d_fo, d_fl, nullptr, (int)total, c->d_sha.as<u8>());
    ++c->launches;
    ZQ_CUDA(c, cudaMemcpyAsync(frag_sha1, c->d_sha.p, total * 20, cudaMemcpyDeviceToHost, c->stream));
  }
  if (frag_o1) {
    ZQ_CUDA(c, c->d_out.ensure(total * 256));
    k_fragment_o1<<<(int)std::min<uint64_t>(total, (uint64_t)c->num_sms * 8), 256, 0, c->stream>>>(c->d_in.as<u8>(), d_fo, d_fl, (int)total, c->d_out.as<u8>());
    ++c->launches;
    ZQ_CUDA(c, cudaMemcpyAsync(frag_o1, c->d_out.p, total * 256, cudaMemcpyDeviceToHost, c->stream));
  }
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  ZQ_CUDA(c, cudaGetLastError());
  return ZQ_OK;
}

#ifdef ZQ_SORT_PROF
// tuning builds only (ZQ_EXTRA_FLAGS=-DZQ_SORT_PROF): read and clear the suffix sort's phase counters
int zq_debug_sort_profile(unsigned long long out[8]) {
  unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out, zqdev::g_sort_prof, sizeof z);
  cudaMemcpyToSymbol(zqdev::g_sort_prof, z, sizeof z);
  return 0;
}
#endif

// ---- introspection -------------------------------------------------------------------------------
uint64_t zq_launch_count(zq_ctx* c) { return c ? c->launches : 0; }
int zq_last_timings(zq_ctx* c, float ms[8]) {
  if (!c) return ZQ_E_NODEVICE;
  memcpy(ms, c->last_ms, 8 * sizeof(float));
  return ZQ_OK;
}

int zq_last_timings_ex(zq_ctx* c, float* ms, int n) {
  if (!c) return ZQ_E_NODEVICE;
  for (int k = 0; k < n; ++k) ms[k] = k < 16 ? c->last_ms[k] : 0.f;
  return ZQ_OK;
}

int zq_suffix_array(zq_ctx* c, const uint8_t* data, uint32_t n, uint32_t* sa_out) {
  using namespace zqdev;
  if (!c) return ZQ_E_NODEVICE;
  if (n == 0) return ZQ_OK;
  cudaSetDevice(c->device);
  const size_t scr = align_up((size_t)n + 1, 64);
  ZQ_CUDA(c, c->d_in.ensure(n + 64));
  ZQ_CUDA(c, c->d_work.ensure(zq_work_bytes(n, 4)));
  ZQ_CUDA(c, c->d_kbuf.ensure(2 * scr * 8)); ZQ_CUDA(c, c->d_vbuf.ensure(6 * scr * 4));
  ZQ_CUDA(c, c->d_units.ensure(sizeof(ZqUnit))); ZQ_CUDA(c, c->d_todo.ensure(4));
  ZqUnit u; memset(&u, 0, sizeof u); u.n = n;
  int zero = 0;
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_in.p, data, n, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_units.p, &u, sizeof u, cudaMemcpyHostToDevice, c->stream));
  ZQ_CUDA(c, cudaMemcpyAsync(c->d_todo.p, &zero, 4, cudaMemcpyHostToDevice, c->stream));
  k_suffix_sort<256, 4><<<1, 256, sizeof(SortSmem<256>), c->stream>>>(c->d_in.as<u8>(), c->d_units.as<ZqUnit>(), c->d_todo.as<int>(), 1,
                                                                 c->d_work.as<u8>(), c->d_kbuf.as<u64>(), c->d_vbuf.as<u32>(), scr);
  ++c->launches;
  ZQ_CUDA(c, cudaMemcpyAsync(sa_out, c->d_work.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  ZQ_CUDA(c, cudaStreamSynchronize(c->stream));
  ZQ_CUDA(c, cudaGetLastError());
  return ZQ_OK;
}

}  // extern "C"
