// zq_config.h -- host side of the block compressor: method expansion, ZPAQ config generation and
// the ZPAQL assembler. Everything here is tiny, runs once per (method, block size) and only has to
// produce the exact header / PCOMP bytes the reference would write (SURVEY.md §8 a1-a3).
//
// Reference behaviour restated (not copied) from the reference's zpaqfranz.cpp:
//   compressBlock digit-level table  Z:20289-20390
//   makeConfig                       Z:19615-20247
//   Compiler (ZPAQL assembler)       Z:15602-15969
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace zq {

// Thrown for every condition the reference reports through libzpaq::error().
struct Error {
  std::string msg;
  explicit Error(const std::string& m) : msg(m) {}
};

// floor(log2(x))+1, 0 for x==0  (== reference lg(), Z:19269)
inline int bitlen(uint32_t x) { return x ? 32 - __builtin_clz(x) : 0; }

// Result of assembling one config.
struct Assembled {
  std::vector<uint8_t> header;  // bytes exactly as ZPAQL::write(out,false) emits them (Z:14084)
  std::vector<uint8_t> pcomp;   // PCOMP bytecode incl. trailing 0 (empty if none)
  std::string pcomp_cmd;        // text between "pcomp" and ";"
  int hh = 0, hm = 0, ph = 0, pm = 0, ncomp = 0;
  std::vector<uint8_t> comp;    // raw component descriptor bytes (type, args...) x ncomp
  std::vector<uint8_t> hcomp;   // HCOMP bytecode incl. trailing 0
};

// Digit methods ("0".."9" + optional block-size digit + ",R,t") -> explicit "x..."/"0..." method.
// `data`/`n` are only inspected for levels >= 5 (byte-gap period analysis, Z:20355-20388).
// Non-digit methods are returned unchanged.
std::string expand_method(const std::string& method, const uint8_t* data, uint32_t n);
// Same for levels >= 5 when the two byte-gap periods were already found (e.g. on the device):
// periods[k] == 0 means "none" (and stops, like the reference's loop).
std::string expand_method_periods(const std::string& method, uint32_t n, const int periods[2]);
// The period analysis alone (Z:20355-20388): fills periods[2].
void gap_periods(const uint8_t* data, uint32_t n, int periods[2]);

// Explicit method string -> ZPAQL config source text; fills args[0..8].
std::string make_config(const std::string& method, int args[9]);

// ZPAQL source -> bytes.
Assembled assemble(const std::string& config, const int args[9]);

// Everything compressBlock needs to know before touching the data.
struct BlockPlan {
  std::string method;   // explicit method
  int args[9];
  Assembled code;
  int lz_level;         // args[1]&3 : 0 none, 1 var-length LZ77, 2 byte LZ77, 3 BWT
  bool e8e9;            // args[1] in 4..7
  bool use_sa;          // LZ77 searches a suffix array (args[5]-args[0] >= 21) or BWT
  bool stored;          // type '0' method: config "comp 0 0 0 0 0"
};
BlockPlan plan_block(const std::string& method, const uint8_t* data, uint32_t n);

}  // namespace zq
