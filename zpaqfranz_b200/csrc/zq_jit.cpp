// zq_jit.cpp -- see zq_jit.h.
#include "zq_jit.h"

#include <dlfcn.h>

#include <cstdarg>
#include <cstdio>
#include <set>

namespace zq {
namespace {

int op_len(unsigned op) { return 1 + ((op & 7) == 7) + (op == 255); }

std::string num(unsigned v) { return std::to_string(v) + "u"; }

// the value of operand `src` of a two-operand instruction
std::string operand(unsigned src, unsigned imm) {
  switch (src) {
    case 0: return "a"; case 1: return "b"; case 2: return "c"; case 3: return "d";
    case 4: return "(unsigned)M[b & MM]"; case 5: return "(unsigned)M[c & MM]"; case 6: return "H[d & HM]";
    default: return num(imm);
  }
}

}  // namespace

bool jit_translate(const uint8_t* code, size_t len, bool with_out, std::string& body, std::string& why) {
  // pass 1: instruction starts and jump targets
  std::set<long> starts, targets;
  for (size_t pc = 0; pc < len; pc += op_len(code[pc])) starts.insert((long)pc);
  for (size_t pc = 0; pc < len; pc += op_len(code[pc])) {
    const unsigned op = code[pc];
    if (pc + op_len(op) > len + 1) break;
    long t = -1;
    if (op == 39 || op == 47 || op == 63) t = (long)pc + 2 + (long)(int8_t)code[pc + 1];   // ((N+128)&255)-127 from the operand byte
    else if (op == 255 && pc + 2 < len) t = (long)code[pc + 1] + 256L * code[pc + 2];
    else continue;
    if (t < 0 || t > (long)len) { targets.insert(-1); continue; }   // leaves the program: a ZPAQL error at run time
    if (t < (long)len && !starts.count(t)) { why = "jump into the middle of an instruction"; return false; }
    targets.insert(t);
  }
  auto label = [&](long t) { return t < 0 || t >= (long)len ? std::string("Lerr") : "L" + std::to_string(t); };
  // pass 2: statements
  std::string s;
  char buf[64];
  for (size_t pc = 0; pc < len; pc += op_len(code[pc])) {
    const unsigned op = code[pc], n = pc + 1 < len ? code[pc + 1] : 0;
    if (targets.count((long)pc)) { snprintf(buf, sizeof buf, "L%ld:;\n", (long)pc); s += buf; }
    s += "  ";
    if (op >= 64) {
      const unsigned src = op & 7, grp = op >> 3;
      const std::string x = operand(src, n);
      switch (grp) {
        case 8: s += "a = " + x + ";"; break; case 9: s += "b = " + x + ";"; break;
        case 10: s += "c = " + x + ";"; break; case 11: s += "d = " + x + ";"; break;
        case 12: s += "M[b & MM] = (unsigned char)(" + x + ");"; break;
        case 13: s += "M[c & MM] = (unsigned char)(" + x + ");"; break;
        case 14: s += "H[d & HM] = " + x + ";"; break;
        case 16: s += "a += " + x + ";"; break; case 17: s += "a -= " + x + ";"; break; case 18: s += "a *= " + x + ";"; break;
        case 19: s += "{ const unsigned x = " + x + "; a = x ? a / x : 0u; }"; break;
        case 20: s += "{ const unsigned x = " + x + "; a = x ? a % x : 0u; }"; break;
        case 21: s += "a &= " + x + ";"; break; case 22: s += "a &= ~(" + x + ");"; break;
        case 23: s += "a |= " + x + ";"; break; case 24: s += "a ^= " + x + ";"; break;
        case 25: s += "a <<= ((" + x + ") & 31u);"; break; case 26: s += "a >>= ((" + x + ") & 31u);"; break;
        case 27: s += "f = a == " + x + ";"; break; case 28: s += "f = a < " + x + ";"; break; case 29: s += "f = a > " + x + ";"; break;
        default:
          if (op == 255) s += "goto " + label(pc + 2 < len ? (long)code[pc + 1] + 256L * code[pc + 2] : -1) + ";";
          else s += "goto Lerr;";
      }
    } else {
      const long rel = (long)pc + 2 + (long)(int8_t)n;
      switch (op) {
        case 1: s += "++a;"; break; case 2: s += "--a;"; break; case 3: s += "a = ~a;"; break; case 4: s += "a = 0u;"; break;
        case 7: s += "a = R[" + num(n) + "];"; break;
        case 8: s += "{ const unsigned t = a; a = b; b = t; }"; break;
        case 9: s += "++b;"; break; case 10: s += "--b;"; break; case 11: s += "b = ~b;"; break; case 12: s += "b = 0u;"; break;
        case 15: s += "b = R[" + num(n) + "];"; break;
        case 16: s += "{ const unsigned t = a; a = c; c = t; }"; break;
        case 17: s += "++c;"; break; case 18: s += "--c;"; break; case 19: s += "c = ~c;"; break; case 20: s += "c = 0u;"; break;
        case 23: s += "c = R[" + num(n) + "];"; break;
        case 24: s += "{ const unsigned t = a; a = d; d = t; }"; break;
        case 25: s += "++d;"; break; case 26: s += "--d;"; break; case 27: s += "d = ~d;"; break; case 28: s += "d = 0u;"; break;
        case 31: s += "d = R[" + num(n) + "];"; break;
        case 32: s += "{ const unsigned t = M[b & MM]; M[b & MM] = (unsigned char)a; a = (a & ~255u) | t; }"; break;
        case 33: s += "M[b & MM] = (unsigned char)(M[b & MM] + 1);"; break; case 34: s += "M[b & MM] = (unsigned char)(M[b & MM] - 1);"; break;
        case 35: s += "M[b & MM] = (unsigned char)~M[b & MM];"; break; case 36: s += "M[b & MM] = 0;"; break;
        case 39: s += "if (f) goto " + label(rel) + ";"; break;
        case 40: s += "{ const unsigned t = M[c & MM]; M[c & MM] = (unsigned char)a; a = (a & ~255u) | t; }"; break;
        case 41: s += "M[c & MM] = (unsigned char)(M[c & MM] + 1);"; break; case 42: s += "M[c & MM] = (unsigned char)(M[c & MM] - 1);"; break;
        case 43: s += "M[c & MM] = (unsigned char)~M[c & MM];"; break; case 44: s += "M[c & MM] = 0;"; break;
        case 47: s += "if (!f) goto " + label(rel) + ";"; break;
        case 48: s += "{ const unsigned t = H[d & HM]; H[d & HM] = a; a = t; }"; break;
        case 49: s += "H[d & HM] = H[d & HM] + 1u;"; break; case 50: s += "H[d & HM] = H[d & HM] - 1u;"; break;
        case 51: s += "H[d & HM] = ~H[d & HM];"; break; case 52: s += "H[d & HM] = 0u;"; break;
        case 55: s += "R[" + num(n) + "] = a;"; break;
        case 56: s += "goto Lend;"; break;
        case 57: s += with_out ? "ZQ_JIT_OUT(a);" : ";"; break;
        case 59: s += "a = (a + M[b & MM] + 512u) * 773u;"; break;
        case 60: s += "H[d & HM] = (H[d & HM] + a + 512u) * 773u;"; break;
        case 63: s += "goto " + label(rel) + ";"; break;
        default: s += "goto Lerr;";
      }
    }
    snprintf(buf, sizeof buf, "   /* %zu: %u */\n", pc, op);
    s += buf;
  }
  s += "Lerr: err = 1;\nLend:;\n";   // running past the last instruction is a ZPAQL error too
  body = s;
  return true;
}

bool jit_context_source(const uint8_t* hcomp, size_t len, int hh, int hm, int ncomp, std::string& src, std::string& why) {
  std::string body;
  if (!jit_translate(hcomp, len, false, body, why)) return false;
  std::string s;
  s += "// generated by zq_jit (ZPAQL -> CUDA C); do not edit\n";
  s += "#ifndef ZQ_JIT_FN\n#define ZQ_JIT_FN static __device__ __forceinline__\n#endif\n";
  s += "#define MM " + num(hm >= 32 ? 0xffffffffu : ((1u << hm) - 1u)) + "\n";
  s += "#define HM " + num(hh >= 32 ? 0xffffffffu : ((1u << hh) - 1u)) + "\n";
  s += "#define ZQ_JIT_NCOMP " + std::to_string(ncomp) + "\n";
  s += "struct ZqJitVm { unsigned a, b, c, d, f; };\n";
  s += "ZQ_JIT_FN void zq_hcomp(ZqJitVm& v, unsigned char* M, unsigned* H, unsigned* R, unsigned input, int& err) {\n";
  s += "  unsigned a = input, b = v.b, c = v.c, d = v.d, f = v.f;\n";
  s += body;
  s += "  v.a = a; v.b = b; v.c = c; v.d = d; v.f = f;\n}\n";
  s += "#undef MM\n#undef HM\n";
  s +=
      "#ifdef __CUDACC__\n"
      "// one thread per block: the block's coded bytes are head[0..hlen) then stream; M, H, R live in the block's model\n"
      "// region (zeroed by k_cm_init); ctx receives H[0..ncomp) after every byte but the last, byte-major\n"
      "extern \"C\" __global__ void zq_ctx_kernel(const unsigned char* head, unsigned hlen, const unsigned char* sbase,\n"
      "                                         const unsigned long long* soff, const unsigned* slen, int nunits,\n"
      "                                         unsigned char* model_base, const unsigned long long* model_off,\n"
      "                                         unsigned long long m_off, unsigned long long h_off, unsigned long long r_off,\n"
      "                                         unsigned* ctx_base, const unsigned long long* ctx_off, unsigned* err_flag) {\n"
      "  const int t = blockIdx.x * blockDim.x + threadIdx.x;\n"
      "  if (t >= nunits) return;\n"
      "  unsigned char* model = model_base + model_off[t];\n"
      "  unsigned char* M = model + m_off;\n"
      "  unsigned* H = (unsigned*)(model + h_off);\n"
      "  unsigned* R = (unsigned*)(model + r_off);\n"
      "  const unsigned char* s = sbase + soff[t];\n"
      "  unsigned* out = ctx_base + ctx_off[t];\n"
      "  ZqJitVm v; v.a = v.b = v.c = v.d = v.f = 0;\n"
      "  int err = 0;\n"
      "  const unsigned K = hlen + slen[t];\n"
      "  for (unsigned k = 0; k + 1 < K; ++k) {\n"
      "    zq_hcomp(v, M, H, R, k < hlen ? head[k] : s[k - hlen], err);\n"
      "    for (int i = 0; i < ZQ_JIT_NCOMP; ++i) out[(unsigned long long)k * ZQ_JIT_NCOMP + i] = H[i & " + num(hh >= 32 ? 0xffffffffu : ((1u << hh) - 1u)) + "];\n"
      "  }\n"
      "  if (err) atomicOr(err_flag, 2u);\n"
      "}\n"
      "#endif\n";
  src = s;
  return true;
}

int jit_compile(const std::string& src, std::vector<char>& cubin, std::string& log) {
  typedef int (*create_t)(void**, const char*, const char*, int, const char* const*, const char* const*);
  typedef int (*compile_t)(void*, int, const char* const*);
  typedef int (*size_t_fn)(void*, size_t*);
  typedef int (*get_t)(void*, char*);
  typedef int (*destroy_t)(void**);
  static void* lib = nullptr;
  if (!lib) {
    const char* names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"};
    for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_LOCAL); if (lib) break; }
  }
  if (!lib) { log = "libnvrtc not found"; return -1; }
  create_t create = (create_t)dlsym(lib, "nvrtcCreateProgram");
  compile_t compile = (compile_t)dlsym(lib, "nvrtcCompileProgram");
  size_t_fn logsize = (size_t_fn)dlsym(lib, "nvrtcGetProgramLogSize");
  get_t getlog = (get_t)dlsym(lib, "nvrtcGetProgramLog");
  size_t_fn binsize = (size_t_fn)dlsym(lib, "nvrtcGetCUBINSize");
  get_t getbin = (get_t)dlsym(lib, "nvrtcGetCUBIN");
  destroy_t destroy = (destroy_t)dlsym(lib, "nvrtcDestroyProgram");
  if (!create || !compile || !logsize || !getlog || !binsize || !getbin || !destroy) { log = "libnvrtc lacks the expected entry points"; return -1; }
  void* prog = nullptr;
  if (create(&prog, src.c_str(), "zq_jit.cu", 0, nullptr, nullptr) != 0) { log = "nvrtcCreateProgram failed"; return -2; }
  const char* opts[] = {"--gpu-architecture=sm_90a", "-lineinfo", "--std=c++17"};
  const int rc = compile(prog, 3, opts);
  size_t ls = 0;
  if (logsize(prog, &ls) == 0 && ls > 1) { log.resize(ls); getlog(prog, &log[0]); }
  if (rc != 0) { destroy(&prog); return -3; }
  size_t bs = 0;
  if (binsize(prog, &bs) != 0 || bs == 0) { destroy(&prog); log += " (no cubin)"; return -4; }
  cubin.resize(bs);
  getbin(prog, cubin.data());
  destroy(&prog);
  return 0;
}

}  // namespace zq

// ---- C ABI (include/zq_b200.h) ------------------------------------------------------------------------------
#include <cstring>

#include "../../include/zq_b200.h"
#include "zq_cm_host.h"

extern "C" int zq_jit_context_source(const uint8_t* header, uint32_t header_len, char* src, uint32_t src_cap, uint32_t* src_len,
                                     char* errbuf, size_t errcap) {
  auto fail = [&](int rc, const std::string& m) {
    if (errbuf && errcap) snprintf(errbuf, errcap, "%s", m.c_str());
    return rc;
  };
  if (!header || !src_len) return fail(ZQ_E_ARG, "bad argument");
  try {
    size_t used = 0;
    zq::Assembled code = zq::parse_block_header(header, header_len, &used);
    std::string s, why;
    if (!zq::jit_context_source(code.hcomp.data(), code.hcomp.size(), code.hh, code.hm, code.ncomp, s, why))
      return fail(ZQ_E_UNSUPPORTED, why);
    *src_len = (uint32_t)s.size();
    if (src) {
      if (src_cap < s.size() + 1) return fail(ZQ_E_OUTPUT, "source buffer too small");
      memcpy(src, s.c_str(), s.size() + 1);
    }
    return ZQ_OK;
  } catch (const zq::Error& e) {
    return fail(ZQ_E_METHOD, e.msg);
  }
}

extern "C" int zq_jit_compile(const char* src, uint32_t* cubin_size, char* log, size_t logcap) {
  if (!src) return ZQ_E_ARG;
  std::vector<char> cubin;
  std::string l;
  const int rc = zq::jit_compile(src, cubin, l);
  if (log && logcap) snprintf(log, logcap, "%s", l.c_str());
  if (cubin_size) *cubin_size = (uint32_t)cubin.size();
  return rc == 0 ? ZQ_OK : rc == -1 ? ZQ_E_UNSUPPORTED : ZQ_E_METHOD;
}

// ---- model -> straight-line coder ---------------------------------------------------------------------------
#include "zq_cm_types.h"

namespace zq {
namespace {

std::string S(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
std::string S(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  return buf;
}

const char* kCoderPrelude = R"GEN(
// ---- generated coder: helpers -------------------------------------------------------------------------------
struct ZqGenCoder { unsigned low, high; unsigned char* out; unsigned char* end; int overflow; };
ZQ_JIT_FN void zq_gen_encode(ZqGenCoder& E, unsigned y, unsigned p16) {            // Encoder::encode, Z:15557
  const unsigned mid = E.low + (unsigned)(((unsigned long long)(E.high - E.low) * p16) >> 16);
  if (y) E.high = mid; else E.low = mid + 1;
  while ((E.high ^ E.low) < 0x1000000u) {
    if (E.out < E.end) *E.out = (unsigned char)(E.high >> 24); else E.overflow = 1;
    ++E.out;
    E.high = E.high << 8 | 255; E.low = E.low << 8; E.low += (E.low == 0);
  }
}
ZQ_JIT_FN int zq_gen_clamp2k(int x) { return x < -2048 ? -2048 : x > 2047 ? 2047 : x; }
ZQ_JIT_FN int zq_gen_clamp512k(int x) { return x < -(1 << 19) ? -(1 << 19) : x > (1 << 19) - 1 ? (1 << 19) - 1 : x; }
struct ZqGenRow { unsigned w[4]; unsigned pos, ok; };
ZQ_JIT_FN unsigned zq_gen_get(const ZqGenRow& r, unsigned idx) { return (r.w[idx >> 2] >> ((idx & 3) * 8)) & 255u; }
ZQ_JIT_FN void zq_gen_put(ZqGenRow& r, unsigned idx, unsigned v) {
  const unsigned sh = (idx & 3) * 8;
  r.w[idx >> 2] = (r.w[idx >> 2] & ~(255u << sh)) | (v << sh);
}
// Predictor::find (Z:15254) with the row held in variables; the previous row goes back to the table first
ZQ_JIT_FN void zq_gen_find(ZqGenRow& r, unsigned char* ht, unsigned ht_mask, unsigned chkshift, unsigned cxt) {
  if (r.ok) { unsigned* d = (unsigned*)(ht + r.pos); d[0] = r.w[0]; d[1] = r.w[1]; d[2] = r.w[2]; d[3] = r.w[3]; }
  const unsigned chk = (cxt >> chkshift) & 255u;
  const unsigned h0 = (cxt * 16u) & (ht_mask - 15u), h1 = h0 ^ 16u, h2 = h0 ^ 32u;
  const unsigned* q0 = (const unsigned*)(ht + h0); const unsigned* q1 = (const unsigned*)(ht + h1); const unsigned* q2 = (const unsigned*)(ht + h2);
  const unsigned a0 = q0[0], a1 = q1[0], a2 = q2[0];
  const unsigned* q; unsigned pos; int fresh = 0;
  if ((a0 & 255u) == chk) { q = q0; pos = h0; }
  else if ((a1 & 255u) == chk) { q = q1; pos = h1; }
  else if ((a2 & 255u) == chk) { q = q2; pos = h2; }
  else {
    const unsigned p0 = (a0 >> 8) & 255u, p1 = (a1 >> 8) & 255u, p2 = (a2 >> 8) & 255u;
    if (p0 <= p1 && p0 <= p2) { q = q0; pos = h0; } else if (p1 < p2) { q = q1; pos = h1; } else { q = q2; pos = h2; }
    fresh = 1;
  }
  if (fresh) { r.w[0] = chk; r.w[1] = r.w[2] = r.w[3] = 0; } else { r.w[0] = q[0]; r.w[1] = q[1]; r.w[2] = q[2]; r.w[3] = q[3]; }
  r.pos = pos; r.ok = 1;
}
)GEN";

}  // namespace

bool jit_coder_source(const void* plan_ptr, std::string& src, std::string& why) {
  const ZqCmPlan& cp = *(const ZqCmPlan*)plan_ptr;
  const int n = cp.n;
  if (n < 1) { why = "no components"; return false; }
  std::string decl, pred, upd, byteend;
  auto off = [](uint64_t o) { return std::to_string((unsigned long long)o) + "ull"; };
  for (int i = 0; i < n; ++i) {
    const ZqCmComp& c = cp.comp[i];
    const std::string I = std::to_string(i);
    const std::string cm = "((unsigned*)(model + " + off(c.cm_off) + "))", ht = "(model + " + off(c.ht_off) + ")";
    switch (c.type) {
      case ZQ_CONS:
        decl += S("  const int p%d = %d;\n", i, ((int)c.a1 - 128) * 4);
        break;
      case ZQ_CM:
        decl += S("  unsigned cx%d = 0, pn%d = 0; int p%d = 0;\n", i, i, i);
        pred += S("      cx%d = (h%d ^ hmap4) & %uu; pn%d = %s[cx%d]; p%d = STRETCH[pn%d >> 17];\n", i, i, c.cm_mask, i, cm.c_str(), i, i, i);
        upd += S("      { const unsigned cnt = pn%d & 0x3ffu; const int er = (int)(y * 32767u) - (int)(pn%d >> 17);\n"
                 "        pn%d += (unsigned)((er * DT[cnt]) & -1024) + (cnt < %uu ? 1u : 0u); %s[cx%d] = pn%d; }\n",
                 i, i, i, (unsigned)c.a2 * 4u, cm.c_str(), i, i);
        break;
      case ZQ_ICM:
        decl += S("  ZqGenRow r%d; r%d.ok = 0; r%d.pos = 0; unsigned s%d = 0, pn%d = 0; int p%d = 0;\n", i, i, i, i, i, i);
        pred += S("      if (nib) zq_gen_find(r%d, %s, %uu, %uu, h%d + 16u * c8);\n", i, ht.c_str(), c.ht_mask, (unsigned)c.a1 + 2u, i);
        pred += S("      s%d = zq_gen_get(r%d, hmap4 & 15u); pn%d = %s[s%d]; p%d = STRETCH[pn%d >> 8];\n", i, i, i, cm.c_str(), i, i, i);
        upd += S("      zq_gen_put(r%d, hmap4 & 15u, NS[s%d * 4 + y]); pn%d += (unsigned)(((int)(y * 32767u) - (int)(pn%d >> 8)) >> 2); %s[s%d] = pn%d;\n",
                 i, i, i, i, cm.c_str(), i, i);
        break;
      case ZQ_ISSE:
        decl += S("  ZqGenRow r%d; r%d.ok = 0; r%d.pos = 0; unsigned s%d = 0; int w0_%d = 0, w1_%d = 0, p%d = 0;\n", i, i, i, i, i, i, i);
        pred += S("      if (nib) zq_gen_find(r%d, %s, %uu, %uu, h%d + 16u * c8);\n", i, ht.c_str(), c.ht_mask, (unsigned)c.a1 + 2u, i);
        pred += S("      s%d = zq_gen_get(r%d, hmap4 & 15u); w0_%d = (int)%s[s%d * 2]; w1_%d = (int)%s[s%d * 2 + 1];\n", i, i, i, cm.c_str(), i, i, cm.c_str(), i);
        pred += S("      p%d = zq_gen_clamp2k((w0_%d * p%d + w1_%d * 64) >> 16);\n", i, i, (int)c.a2, i);
        upd += S("      { const int er = (int)(y * 32767u) - (int)SQUASH[p%d + 2048];\n"
                 "        %s[s%d * 2] = (unsigned)zq_gen_clamp512k(w0_%d + ((er * p%d + (1 << 12)) >> 13));\n"
                 "        %s[s%d * 2 + 1] = (unsigned)zq_gen_clamp512k(w1_%d + ((er + 16) >> 5));\n"
                 "        zq_gen_put(r%d, hmap4 & 15u, NS[s%d * 4 + y]); }\n",
                 i, cm.c_str(), i, i, (int)c.a2, cm.c_str(), i, i, i, i);
        break;
      case ZQ_MATCH:
        decl += S("  unsigned ml%d = 0, mp%d = 0, mb%d = 0, mc%d = 0, lim%d = 0; int p%d = 0;\n", i, i, i, i, i, i);
        pred += S("      if (ml%d == 0) p%d = 0; else { mb%d = (%s[(lim%d - mp%d) & %uu] >> (7 - mc%d)) & 1u;\n"
                  "        p%d = STRETCH[(DT2K[ml%d] * (mb%d ? -1 : 1)) & 32767]; }\n",
                  i, i, i, ht.c_str(), i, i, c.ht_mask, i, i, i, i);
        upd += S("      if (mb%d != y) ml%d = 0;\n", i, i);
        upd += S("      if (++mc%d == 8) { %s[lim%d & %uu] = (unsigned char)(c8 * 2 + y); mc%d = 0; lim%d = (lim%d + 1) & %uu;\n"
                 "        if (ml%d == 0) { mp%d = lim%d - %s[h%d & %uu];\n"
                 "          if (mp%d & %uu) while (ml%d < 255 && %s[(lim%d - ml%d - 1) & %uu] == %s[(lim%d - ml%d - mp%d - 1) & %uu]) ++ml%d; }\n"
                 "        else ml%d += ml%d < 255;\n"
                 "        %s[h%d & %uu] = lim%d; }\n",
                 i, ht.c_str(), i, c.ht_mask, i, i, i, c.ht_mask,
                 i, i, i, cm.c_str(), i, c.cm_mask,
                 i, c.ht_mask, i, ht.c_str(), i, i, c.ht_mask, ht.c_str(), i, i, i, c.ht_mask, i,
                 i, i,
                 cm.c_str(), i, c.cm_mask, i);
        break;
      case ZQ_AVG:
        decl += S("  int p%d = 0;\n", i);
        pred += S("      p%d = (p%d * %d + p%d * %d) >> 8;\n", i, (int)c.a1, (int)c.a3, (int)c.a2, 256 - (int)c.a3);
        break;
      case ZQ_MIX2:
        decl += S("  unsigned cx%d = 0; int w%d = 0, p%d = 0;\n", i, i, i);
        pred += S("      cx%d = (h%d + (c8 & %uu)) & %uu; w%d = ((unsigned short*)%s)[cx%d];\n", i, i, (unsigned)c.a5, c.cm_mask, i, cm.c_str(), i);
        pred += S("      p%d = (w%d * p%d + (65536 - w%d) * p%d) >> 16;\n", i, i, (int)c.a2, i, (int)c.a3);
        upd += S("      { const int er = (((int)(y * 32767u) - (int)SQUASH[p%d + 2048]) * %d) >> 5;\n"
                 "        int w = w%d + ((er * (p%d - p%d) + (1 << 12)) >> 13); w = w < 0 ? 0 : w > 65535 ? 65535 : w;\n"
                 "        ((unsigned short*)%s)[cx%d] = (unsigned short)w; }\n",
                 i, (int)c.a4, i, (int)c.a2, (int)c.a3, cm.c_str(), i);
        break;
      case ZQ_MIX: {
        const int m = c.a3, j0 = c.a2;
        decl += S("  unsigned row%d = 0; int p%d = 0;", i, i);
        for (int k = 0; k < m; ++k) decl += S(" int wt%d_%d = 0;", i, k);
        decl += "\n";
        pred += S("      row%d = ((h%d + (c8 & %uu)) & %uu) * %uu;\n      { int* wp = (int*)%s + row%d; int sum = 0;\n", i, i, (unsigned)c.a5, c.cm_mask, (unsigned)m, cm.c_str(), i);
        for (int k = 0; k < m; ++k) pred += S("        wt%d_%d = wp[%d]; sum += (wt%d_%d >> 8) * p%d;\n", i, k, k, i, k, j0 + k);
        pred += S("        p%d = zq_gen_clamp2k(sum >> 8); }\n", i);
        upd += S("      { int* wp = (int*)%s + row%d; const int er = (((int)(y * 32767u) - (int)SQUASH[p%d + 2048]) * %d) >> 4;\n", cm.c_str(), i, i, (int)c.a4);
        for (int k = 0; k < m; ++k) upd += S("        wp[%d] = zq_gen_clamp512k(wt%d_%d + ((er * p%d + (1 << 12)) >> 13));\n", k, i, k, j0 + k);
        upd += "      }\n";
        break;
      }
      case ZQ_SSE:
        decl += S("  unsigned cx%d = 0, pn%d = 0; int p%d = 0;\n", i, i, i);
        pred += S("      { unsigned cx = (h%d + c8) * 32u; int pq = p%d + 992; pq = pq < 0 ? 0 : pq > 1983 ? 1983 : pq; const int wt = pq & 63; pq >>= 6; cx += (unsigned)pq;\n"
                  "        const unsigned e0 = %s[cx & %uu], e1 = %s[(cx + 1) & %uu];\n"
                  "        p%d = STRETCH[((e0 >> 10) * (unsigned)(64 - wt) + (e1 >> 10) * (unsigned)wt) >> 13];\n"
                  "        cx += (unsigned)(wt >> 5); cx%d = cx & %uu; pn%d = (wt >> 5) ? e1 : e0; }\n",
                  i, (int)c.a2, cm.c_str(), c.cm_mask, cm.c_str(), c.cm_mask, i, i, c.cm_mask, i);
        upd += S("      { const unsigned cnt = pn%d & 0x3ffu; const int er = (int)(y * 32767u) - (int)(pn%d >> 17);\n"
                 "        pn%d += (unsigned)((er * DT[cnt]) & -1024) + (cnt < %uu ? 1u : 0u); %s[cx%d] = pn%d; }\n",
                 i, i, i, (unsigned)c.a4 * 4u, cm.c_str(), i, i);
        break;
      default: why = "unknown component type"; return false;
    }
  }
  std::string s = kCoderPrelude;
  s += S("// model: %d components; mixer updates come first, as in Predictor::update0 (Z:15139): they use every p as predicted\n", n);
  s += "ZQ_JIT_FN unsigned zq_encode_block(const unsigned char* head, unsigned hlen, const unsigned char* stream, unsigned slen,\n"
       "                                   const unsigned* ctx, unsigned char* model, const short* STRETCH, const unsigned short* SQUASH,\n"
       "                                   const int* DT, const int* DT2K, const unsigned char* NS, unsigned char* out, unsigned cap, int* overflow) {\n";
  s += "  ZqGenCoder E; E.low = 1; E.high = 0xffffffffu; E.out = out; E.end = out + cap; E.overflow = 0;\n";
  s += decl;
  for (int i = 0; i < n; ++i) s += S("  unsigned h%d = 0;\n", i);
  s += "  const unsigned K = hlen + slen;\n  for (unsigned k = 0; k < K; ++k) {\n";
  s += S("    if (k > 0) { const unsigned* cv = ctx + (unsigned long long)(k - 1) * %d;", n);
  for (int i = 0; i < n; ++i) s += S(" h%d = cv[%d];", i, i);
  s += " }\n";
  s += "    const unsigned c = k < hlen ? head[k] : stream[k - hlen];\n    zq_gen_encode(E, 0, 0);\n    unsigned c8 = 1, hmap4 = 1;\n";
  s += "    for (int bit = 7; bit >= 0; --bit) {\n      const unsigned y = (c >> bit) & 1u;\n      const int nib = c8 == 1 || (c8 & 0xf0u) == 16u;\n";
  s += pred;
  s += S("      zq_gen_encode(E, y, (unsigned)SQUASH[p%d + 2048] * 2 + 1);\n", n - 1);
  // updates: no component's update reads another one's state (inputs are the p's of the prediction), so index order
  s += upd;
  s += "      c8 += c8 + y;\n"
       "      if (c8 >= 256) { c8 = 1; hmap4 = 1; }\n"
       "      else if (c8 >= 16 && c8 < 32) hmap4 = (hmap4 & 0xf) << 5 | y << 4 | 1;\n"
       "      else hmap4 = (hmap4 & 0x1f0) | (((hmap4 & 0xf) * 2 + y) & 0xf);\n";
  s += "    }\n  }\n  zq_gen_encode(E, 1, 0);\n  *overflow = E.overflow;\n  return (unsigned)(E.out - out);\n}\n";
  s +=
      "#ifdef __CUDACC__\n"
      "// One block per `stride` threads (stride 32: lane 0 of every warp codes a block, the chain fast path's mapping;\n"
      "// stride 1: one block per thread).  `tab` is the device copy of zq::CmTables (stretch, squash, dt, dt2k, ns in that\n"
      "// order), read through L1; contexts come from zq_ctx_kernel's buffer; ids[t] is the unit the t-th block belongs to.\n"
      "extern \"C\" __global__ void zq_code_kernel(const unsigned char* head, unsigned hlen, const unsigned char* sbase,\n"
      "                                          const unsigned long long* soff, const unsigned* slen, int nunits, int stride,\n"
      "                                          unsigned char* model_base, const unsigned long long* model_off,\n"
      "                                          const unsigned* ctx_base, const unsigned long long* ctx_off, const unsigned char* tab,\n"
      "                                          unsigned char* coded_base, const unsigned long long* coded_off, const unsigned* coded_cap,\n"
      "                                          const int* ids, unsigned* coded_len, unsigned* err_flag) {\n"
      "  const int g = blockIdx.x * blockDim.x + threadIdx.x;\n"
      "  if (g % stride) return;\n"
      "  const int t = g / stride;\n"
      "  if (t >= nunits) return;\n"
      "  int overflow = 0;\n"
      "  coded_len[ids[t]] = zq_encode_block(head, hlen, sbase + soff[t], slen[t], ctx_base + ctx_off[t], model_base + model_off[t],\n"
      "                                      (const short*)tab, (const unsigned short*)(tab + 65536), (const int*)(tab + 73728),\n"
      "                                      (const int*)(tab + 77824), tab + 78848, coded_base + coded_off[t], coded_cap[t], &overflow);\n"
      "  if (overflow) atomicOr(err_flag, 1u);\n"
      "}\n"
      "#endif\n";
  src += s;
  return true;
}

}  // namespace zq

extern "C" int zq_jit_coder_source(const uint8_t* header, uint32_t header_len, char* src, uint32_t src_cap, uint32_t* src_len,
                                   char* errbuf, size_t errcap) {
  auto fail = [&](int rc, const std::string& m) {
    if (errbuf && errcap) snprintf(errbuf, errcap, "%s", m.c_str());
    return rc;
  };
  if (!header || !src_len) return fail(ZQ_E_ARG, "bad argument");
  try {
    size_t used = 0;
    zq::Assembled code = zq::parse_block_header(header, header_len, &used);
    std::vector<ZqCmFill> fills;
    ZqCmPlan cp = zq::make_cm_plan(code, fills);
    std::string s, why;
    if (!zq::jit_context_source(code.hcomp.data(), code.hcomp.size(), code.hh, code.hm, code.ncomp, s, why)) return fail(ZQ_E_UNSUPPORTED, why);
    if (!zq::jit_coder_source(&cp, s, why)) return fail(ZQ_E_UNSUPPORTED, why);
    *src_len = (uint32_t)s.size();
    if (src) {
      if (src_cap < s.size() + 1) return fail(ZQ_E_OUTPUT, "source buffer too small");
      memcpy(src, s.c_str(), s.size() + 1);
    }
    return ZQ_OK;
  } catch (const zq::Error& e) {
    return fail(ZQ_E_METHOD, e.msg);
  }
}
