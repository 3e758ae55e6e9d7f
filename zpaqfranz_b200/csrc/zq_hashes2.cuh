// zq_hashes2.cuh -- the two per-file checks the archiver computes by default (SURVEY §8f rank 4): CRC-32 (always on in
// Jidac::updatehash, crc32_16bytes Z:30299: IEEE 802.3, reflected polynomial 0xEDB88320) and XXH64 (the default file
// hash, XXH64 Z:24688, seed 0).
//
// CRC-32 is linear over GF(2): raw(A||B, x) = raw(B, 0) ^ Z_|B|(raw(A, x)), Z_n = "advance the register through n zero
// bytes".  So a buffer is cut into 4 KiB chunks coded independently from a zero register by one thread each (slice by
// four, tables in shared memory), and one thread per buffer folds the partial values with the fixed operator Z_4096
// (as four 256-entry tables built on the host) -- the same algebra as the reference's crc32_combine (Z:30382).
// XXH64 is a sequential recurrence over 32-byte stripes: one thread per buffer.
// Checked bit for bit against zlib and the reference's own XXH64 under the SIMT emulator (tests/test_hash_emu.py) and on
// the GPU (tests/test_gpu_hashes.py).
#pragma once
#include "zq_common.cuh"

namespace zqdev {

constexpr u32 CRC_CHUNK = 4096;

struct CrcTables {      // built on the host (zq_api.cu): T[k][v] slice tables, Z[k][v] = Z_4096(v << 8k)
  u32 T[4][256];
  u32 Z[4][256];
};

// partial[c] = raw CRC register of chunk c starting from 0
__global__ void __launch_bounds__(128)
k_crc32_chunks(const u8* __restrict__ base, const u64* __restrict__ off, const u64* __restrict__ len, const u64* __restrict__ chunk_first,
               int nbuf, u64 nchunks, const CrcTables* __restrict__ tab, u32* __restrict__ partial) {
  __shared__ u32 T[4][256];
  for (u32 k = threadIdx.x; k < 1024; k += blockDim.x) T[k >> 8][k & 255] = tab->T[k >> 8][k & 255];
  __syncthreads();
  const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nchunks) return;
  int lo = 0, hi = nbuf - 1;   // last b with chunk_first[b] <= t
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (chunk_first[mid] <= t) lo = mid; else hi = mid - 1; }
  const u64 start = (t - chunk_first[lo]) * CRC_CHUNK;
  const u64 L = len[lo];
  const u32 n = (u32)(L - start < CRC_CHUNK ? L - start : CRC_CHUNK);
  const u8* __restrict__ p = base + off[lo] + start;
  u32 crc = 0, i = 0;
  for (; i < n && ((uintptr_t)(p + i) & 3); ++i) crc = T[0][(crc ^ p[i]) & 255] ^ (crc >> 8);
  for (; i + 4 <= n; i += 4) {
    const u32 w = crc ^ *(const u32*)(p + i);
    crc = T[3][w & 255] ^ T[2][(w >> 8) & 255] ^ T[1][(w >> 16) & 255] ^ T[0][w >> 24];
  }
  for (; i < n; ++i) crc = T[0][(crc ^ p[i]) & 255] ^ (crc >> 8);
  partial[t] = crc;
}

// out[b] = CRC-32 of buffer b (little-endian u32): fold the chunk values left to right
__global__ void __launch_bounds__(128)
k_crc32_fold(const u64* __restrict__ len, const u64* __restrict__ chunk_first, int nbuf, const CrcTables* __restrict__ tab,
             const u32* __restrict__ partial, u32* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nbuf) return;
  const u64 L = len[b], first = chunk_first[b];
  const u64 full = L / CRC_CHUNK;
  u32 s = 0xffffffffu;
  for (u64 c = 0; c < full; ++c)
    s = tab->Z[0][s & 255] ^ tab->Z[1][(s >> 8) & 255] ^ tab->Z[2][(s >> 16) & 255] ^ tab->Z[3][s >> 24] ^ partial[first + c];
  const u32 tail = (u32)(L - full * CRC_CHUNK);
  if (tail) {
    for (u32 k = 0; k < tail; ++k) s = tab->T[0][s & 255] ^ (s >> 8);   // Z_tail
    s ^= partial[first + full];
  }
  out[b] = ~s;
}

__device__ __forceinline__ u64 xxh_rotl(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ u64 xxh_read64(const u8* p) {
  u64 v = 0;
  for (int k = 7; k >= 0; --k) v = v << 8 | p[k];
  return v;
}
__device__ __forceinline__ u64 xxh64_round(u64 acc, u64 in) {
  acc += in * 0xC2B2AE3D27D4EB4FULL;
  return xxh_rotl(acc, 31) * 0x9E3779B185EBCA87ULL;
}
__device__ __forceinline__ u64 xxh64_merge(u64 h, u64 v) {
  h ^= xxh64_round(0, v);
  return h * 0x9E3779B185EBCA87ULL + 0x85EBCA77C2B2AE63ULL;
}

// out[b] = XXH64(buffer b, seed 0) as a little-endian u64
__global__ void __launch_bounds__(128)
k_xxh64_many(const u8* __restrict__ base, const u64* __restrict__ off, const u64* __restrict__ len, int n, u64* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 P1 = 0x9E3779B185EBCA87ULL, P2 = 0xC2B2AE3D27D4EB4FULL, P3 = 0x165667B19E3779F9ULL, P4 = 0x85EBCA77C2B2AE63ULL,
            P5 = 0x27D4EB2F165667C5ULL;
  const u8* __restrict__ p = base + off[i];
  const u64 L = len[i];
  u64 pos = 0, h;
  if (L >= 32) {
    u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
    for (; pos + 32 <= L; pos += 32) {
      v1 = xxh64_round(v1, xxh_read64(p + pos)); v2 = xxh64_round(v2, xxh_read64(p + pos + 8));
      v3 = xxh64_round(v3, xxh_read64(p + pos + 16)); v4 = xxh64_round(v4, xxh_read64(p + pos + 24));
    }
    h = xxh_rotl(v1, 1) + xxh_rotl(v2, 7) + xxh_rotl(v3, 12) + xxh_rotl(v4, 18);
    h = xxh64_merge(h, v1); h = xxh64_merge(h, v2); h = xxh64_merge(h, v3); h = xxh64_merge(h, v4);
  } else h = P5;
  h += L;
  for (; pos + 8 <= L; pos += 8) { h ^= xxh64_round(0, xxh_read64(p + pos)); h = xxh_rotl(h, 27) * P1 + P4; }
  if (pos + 4 <= L) {
    const u64 w = (u64)p[pos] | (u64)p[pos + 1] << 8 | (u64)p[pos + 2] << 16 | (u64)p[pos + 3] << 24;
    h ^= w * P1; h = xxh_rotl(h, 23) * P2 + P3; pos += 4;
  }
  for (; pos < L; ++pos) { h ^= p[pos] * P5; h = xxh_rotl(h, 11) * P1; }
  h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
  out[i] = h;
}

}  // namespace zqdev
