// exact_sum.cuh -- an exact, order-independent sum of fp32 values (the accumulator of the deterministic mode, DESIGN.md 3.10).
//
// A finite fp32 value is m 2^e with |m| < 2^24 and e in [-149, 104]: every one of them is an integer multiple of 2^-149 below
// 2^128.  An ExactSum holds the sum of the values deposited into it as that integer, in nine int64 words; word i holds (after
// the carries have been propagated) the 32-bit digit of weight 2^(32 i - 149).  A deposit adds the value's two 32-bit-aligned
// pieces to two adjacent words with two integer additions; integer addition is associative, so the words -- and the value
// ExactFinalize rounds from them -- do not depend on the order of the deposits.  Each deposit adds less than 2^32 in magnitude
// to a word, so fewer than 2^31 deposits per ExactSum cannot overflow one.  Non-finite values set sticky flags instead, which give
// the IEEE sum: NaN if a NaN or both infinities were deposited, else the infinity that was.
//
// The same code runs on the host (bba_host_exact_sum) and on the device (atomic deposits).
#pragma once

#include <stdint.h>
#include <string.h>

namespace bba {

constexpr int kExactWords = 9;
constexpr unsigned long long kExactPosInf = 1ull, kExactNegInf = 2ull, kExactNaN = 4ull;

struct ExactSum {
  unsigned long long w[kExactWords];   // int64 two's complement
  unsigned long long flags;            // kExactPosInf | kExactNegInf | kExactNaN
};
static_assert(sizeof(ExactSum) == 80, "ExactSum layout");

// The deposit of x: add lo to word `word` and hi to word `word` + 1.  Returns false for a non-finite x (*flag says which) and for
// zeros (*flag = 0).
__host__ __device__ __forceinline__ bool ExactSplit(float x, int* word, long long* lo, long long* hi, unsigned long long* flag) {
#ifdef __CUDA_ARCH__
  const uint32_t bits = __float_as_uint(x);
#else
  uint32_t bits;
  memcpy(&bits, &x, sizeof(bits));
#endif
  const uint32_t biased = (bits >> 23) & 0xffu, frac = bits & 0x7fffffu;
  const bool neg = (bits >> 31) != 0;
  *flag = 0;
  if (biased == 0xffu) {
    *flag = frac ? kExactNaN : (neg ? kExactNegInf : kExactPosInf);
    return false;
  }
  if (biased == 0 && frac == 0) return false;
  // x = m 2^(o - 149): subnormals have o = 0, normals o = biased - 1 and the implicit bit
  const int o = biased == 0 ? 0 : static_cast<int>(biased) - 1;
  const long long m = static_cast<long long>(biased == 0 ? frac : (frac | 0x800000u));
  const long long v = (neg ? -m : m) * (1ll << (o & 31));   // |v| < 2^55
  *word = o >> 5;                                          // 0 .. 7
  *lo = v & 0xffffffffll;
  *hi = v >> 32;                                           // arithmetic shift: floor(v / 2^32)
  return true;
}

__host__ __device__ __forceinline__ int ExactClz32(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __clz(static_cast<int>(x));
#else
  return x ? __builtin_clz(x) : 32;
#endif
}

__host__ __device__ __forceinline__ double ExactBitsToDouble(unsigned long long bits) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(static_cast<long long>(bits));
#else
  double r;
  memcpy(&r, &bits, sizeof(r));
  return r;
#endif
}

// Propagates the carries of w[0..8] (in place): afterwards w[0..7] lie in [0, 2^32) and w[8] carries the sign.
__host__ __device__ __forceinline__ void ExactCarry(long long (&w)[kExactWords]) {
  for (int i = 0; i + 1 < kExactWords; ++i) {
    const long long carry = w[i] >> 32;
    w[i] -= carry * (1ll << 32);
    w[i + 1] += carry;
  }
}

// The sum of the deposits rounded to fp64, to nearest with ties to even; an exact zero gives +0.0.
__host__ __device__ inline double ExactFinalize(const unsigned long long (&words)[kExactWords], unsigned long long flags) {
  if ((flags & kExactNaN) || (flags & (kExactPosInf | kExactNegInf)) == (kExactPosInf | kExactNegInf)) return ExactBitsToDouble(0x7ff8000000000000ull);
  if (flags & kExactPosInf) return ExactBitsToDouble(0x7ff0000000000000ull);
  if (flags & kExactNegInf) return ExactBitsToDouble(0xfff0000000000000ull);
  long long w[kExactWords];
  for (int i = 0; i < kExactWords; ++i) w[i] = static_cast<long long>(words[i]);
  ExactCarry(w);
  const bool neg = w[kExactWords - 1] < 0;
  if (neg) {
    for (int i = 0; i < kExactWords; ++i) w[i] = -w[i];
    ExactCarry(w);
  }
  // magnitude as ten 32-bit digits (the top word may exceed 32 bits: 2^31 deposits below 2^128 sum to less than 2^159)
  uint32_t d[kExactWords + 1];
  for (int i = 0; i + 1 < kExactWords; ++i) d[i] = static_cast<uint32_t>(w[i]);
  d[kExactWords - 1] = static_cast<uint32_t>(w[kExactWords - 1] & 0xffffffffll);
  d[kExactWords] = static_cast<uint32_t>(w[kExactWords - 1] >> 32);
  int k = kExactWords;
  while (k >= 0 && d[k] == 0) --k;
  if (k < 0) return 0.0;
  // the top 96 bits from digit k down, shifted so that the leading one is bit 95
  const int lz = ExactClz32(d[k]);
  const uint32_t d1 = k >= 1 ? d[k - 1] : 0u, d2 = k >= 2 ? d[k - 2] : 0u;
  bool sticky = false;
  for (int i = 0; i < k - 2; ++i) sticky |= d[i] != 0;
  unsigned long long top = (static_cast<unsigned long long>(d[k]) << 32) | d1;   // bits 95..32 before the shift
  uint32_t low = d2;
  if (lz) {
    top = (top << lz) | (low >> (32 - lz));
    low <<= lz;
  }
  sticky |= low != 0;
  // 53 bits of mantissa, then the rounding bit and the bits below it
  unsigned long long mant = top >> 11;
  const unsigned long long rest = top & 0x7ffull;
  const int lead = 32 * k + 31 - lz;   // bit index of the leading one in units of 2^-149
  int exp = lead - 52 - 149;
  if ((rest & 0x400ull) && ((rest & 0x3ffull) || sticky || (mant & 1ull))) {
    ++mant;
    if (mant == (1ull << 53)) {
      mant >>= 1;
      ++exp;
    }
  }
  // mant < 2^53 and 2^-201 <= |result| < 2^160: the product is exact, no fp64 overflow or subnormal
  double r = static_cast<double>(mant);
  for (; exp > 0; exp -= exp < 32 ? exp : 32) r *= static_cast<double>(1ull << (exp < 32 ? exp : 32));
  for (; exp < 0; exp += -exp < 32 ? -exp : 32) r /= static_cast<double>(1ull << (-exp < 32 ? -exp : 32));
  return neg ? -r : r;
}
inline __host__ __device__ double ExactFinalize(const ExactSum& s) { return ExactFinalize(s.w, s.flags); }

#ifdef __CUDACC__
// Adds x to *s with two integer atomics (one atomicOr for a non-finite x).
__device__ __forceinline__ void ExactDeposit(ExactSum* s, float x) {
  int word;
  long long lo, hi;
  unsigned long long flag;
  if (!ExactSplit(x, &word, &lo, &hi, &flag)) {
    if (flag) atomicOr(&s->flags, flag);
    return;
  }
  if (lo) atomicAdd(&s->w[word], static_cast<unsigned long long>(lo));
  if (hi) atomicAdd(&s->w[word + 1], static_cast<unsigned long long>(hi));
}
#endif

}  // namespace bba
