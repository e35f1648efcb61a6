// geno_expand.cuh - 2-bit genotype -> int8 operand expansion shared by every tensor-path kernel.
//
// A 32-bit word holds 16 consecutive samples of ONE variant (PgrGet layout).  For a plane whose
// value depends only on the genotype code, the 16 output bytes come from four PRMT (byte permute)
// instructions whose selector nibbles are the genotype codes themselves and whose source register
// is the plane's 4-entry table {value(code0), value(code1), value(code2), value(code3)}.
// Even and odd samples are handled separately (their codes are already nibble-aligned after one
// mask), so byte position p of the 16-byte result holds sample PosToSample(p) (common.cuh).
#pragma once
#include <cstdint>

namespace pl2 {

struct Sel4 {
  uint32_t e_lo, e_hi, o_lo, o_hi;  // selectors: samples {0,2,4,6}, {8,10,12,14}, {1,3,5,7}, {9,..,15}
};

__device__ __forceinline__ Sel4 make_selectors(uint32_t w) {
  const uint32_t ev = w & 0x33333333u;
  const uint32_t od = (w >> 2) & 0x33333333u;
  Sel4 s;
  s.e_lo = ev;
  s.e_hi = ev >> 16;
  s.o_lo = od;
  s.o_hi = od >> 16;
  return s;
}

__device__ __forceinline__ uint4 expand16(uint32_t table, const Sel4& s) {
  uint4 r;
  r.x = __byte_perm(table, 0u, s.e_lo);
  r.y = __byte_perm(table, 0u, s.e_hi);
  r.z = __byte_perm(table, 0u, s.o_lo);
  r.w = __byte_perm(table, 0u, s.o_hi);
  return r;
}

// Plane tables, byte c = value for genotype code c (0 hom-REF, 1 het, 2 hom-ALT, 3 missing).
constexpr uint32_t kTabHet = 0x00000100u;     // T: het indicator
constexpr uint32_t kTabHom = 0x00010001u;     // H: hom indicator (the reference's `hom` plane)
constexpr uint32_t kTabSgn = 0x00FF0001u;     // S: +1 hom-REF, -1 hom-ALT, 0 otherwise
constexpr uint32_t kTabDosage = 0x00020100u;  // g: ALT dosage 0/1/2, missing -> 0
constexpr uint32_t kTabNonmiss = 0x00010101u; // m: non-missing indicator
constexpr uint32_t kTabMiss = 0x01000000u;    // mu: missing indicator

// A plane table as a PER-THREAD register.  PRMT needs its table operand in a vector register; a
// compile-time constant gets hoisted into a uniform register and re-materialised with one extra
// IMAD.U32 in front of EVERY PRMT.  OR-ing in
// `thread_zero` - a value that is 0 at run time but that ptxas can prove neither constant nor
// warp-uniform (callers pass threadIdx.x * (a kernel argument >> 31)) - keeps each table in one
// vector register for the whole kernel.
__device__ __forceinline__ uint32_t table_reg(uint32_t table, uint32_t thread_zero) { return table | thread_zero; }

// Bytes of one no-swizzle core matrix of a wgmma operand in shared memory: 8 rows x 16 K-bytes.
constexpr uint32_t kCoreBytes = 128;

}  // namespace pl2
