// zq_jit.h -- ZPAQL -> CUDA C translation of a block's context program (HCOMP), and run-time compilation with NVRTC.
//
// The reference does not interpret ZPAQL on its hot path either: libzpaq translates HCOMP/PCOMP to x86 machine code
// when a block starts (ZPAQL::assemble, Z:16358, called from ZPAQL::run Z:17677; interpreter only under `flagnojit`).  The device counterpart is
// source-to-source: one labelled C statement per ZPAQL instruction, jumps become gotos, M/H sizes are baked in as
// constants, then NVRTC -> cubin for sm_90a.  ncu (profiles/r01j) has the interpreted context machine as the critical
// path of the chain models (~380 cycles per ZPAQL instruction against a handful of SASS instructions translated).
//
// Status: on the compress path (zq_api.cu loads the module per model, cached; default for models of <= 8 components,
// ZQ_CM_JIT forces a form).  The CPU tests compile the generated code for the host and step it against the
// interpreter, NVRTC compiles it for sm_90a without a GPU, the GPU tests run all three forms bit for bit
// (tests/test_gpu_compress.py::test_context_program_forms_over_several_waves).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace zq {

// C statements for one run of the program (registers a,b,c,d,f; memories M,H,R; masks MM,HM; `err` set on ZPAQL
// errors).  Returns false (with `why`) for programs the translator does not cover: jumps into the middle of an
// instruction.  `with_out`: PCOMP's OUT calls ZQ_JIT_OUT(a); HCOMP ignores it.
bool jit_translate(const uint8_t* code, size_t len, bool with_out, std::string& body, std::string& why);

// Complete translation unit: `zq_hcomp` (one run) and the kernel `zq_ctx_kernel` (one thread per block: runs the
// program over the block's coded bytes and stores H[0..ncomp) after every byte but the last).
bool jit_context_source(const uint8_t* hcomp, size_t len, int hh, int hm, int ncomp, std::string& src, std::string& why);

// The model itself as straight-line code: `zq_encode_block` codes a block's bytes with the component chain of `plan`
// written out component by component (index order is a valid evaluation order: inputs always have lower indices),
// every size, mask, limit, rate and table offset a literal, hash rows and mixer weights in local variables.  This is
// the chain fast path of zq_cm.cuh generalised to any model; `plan` supplies the table offsets inside a block's
// model region (make_cm_plan), so k_cm_init's initialisation applies unchanged.  Appended to `src`.
struct ZqCmPlanRef;   // (ZqCmPlan from zq_cm_types.h; declared in the .cpp to keep this header light)
bool jit_coder_source(const void* zq_cm_plan, std::string& src, std::string& why);

// NVRTC (dlopen'ed, no link-time dependency): source -> cubin for sm_90a.  Returns 0 or a negative code with `log`.
int jit_compile(const std::string& src, std::vector<char>& cubin, std::string& log);

}  // namespace zq
