// crc32.cuh — CRC-32 (the gzip / zlib polynomial) on the device: the byte table, and zlib's crc32_combine algebra
// (multiplication by x^(8 len) mod P in GF(2)), so slices computed in parallel can be joined.  Used by the BGZF
// compressor and inflater (bgzf_device.cu, bgzf_inflate.cu).
#pragma once
#include <cstdint>

namespace gb {

constexpr uint32_t CRC_POLY = 0xedb88320u;

__device__ inline uint32_t multmodp(uint32_t a, uint32_t b) {          // a * b mod P, bit-reflected (a != 0)
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}
__device__ inline uint32_t x8nmodp(uint64_t n, const uint32_t* x2n) {  // x^(8n) mod P; x2n[k] = x^(2^k)
    uint32_t p = 1u << 31;
    for (uint32_t k = 3; n; n >>= 1, k++)
        if (n & 1) p = multmodp(x2n[k & 31], p);
    return p;
}
// crc(A || B) from crc(A), crc(B) and len(B) (zlib's crc32_combine)
__device__ inline uint32_t crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b, const uint32_t* x2n) {
    return len_b ? multmodp(x8nmodp(len_b, x2n), crc_a) ^ crc_b : crc_a;
}

// The byte table and x^(2^k) mod P, built by the threads t = 0..nt-1 of a CTA (the caller synchronises after).
__device__ inline void crc32_tables(uint32_t* tab, uint32_t* x2n, uint32_t t, uint32_t nt) {
    for (uint32_t i = t; i < 256; i += nt) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
        tab[i] = c;
    }
    if (t == 0) {
        x2n[0] = 1u << 30;
        for (int k = 1; k < 32; k++) x2n[k] = multmodp(x2n[k - 1], x2n[k - 1]);
    }
}

} // namespace gb
