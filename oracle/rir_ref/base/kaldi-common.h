// Minimal stand-ins for the Kaldi types rir-generator.{h,cc} uses, so that the reference's own
// generator compiles without Kaldi (oracle/rir_ref/build.sh).  TEST INFRASTRUCTURE ONLY.
#pragma once
#include <cmath>
#include <cstdint>
#include <iostream>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace kaldi {
typedef float BaseFloat;
typedef int32_t int32;
inline double Log(double x) { return std::log(x); }

struct ErrorThrower {   // KALDI_ERR << ...: throws when the statement ends
  std::ostringstream s;
  template <class T> ErrorThrower& operator<<(const T& v) { s << v; return *this; }
  ~ErrorThrower() noexcept(false) { throw std::runtime_error(s.str()); }
};

template <class T>
struct Matrix {
  int rows = 0, cols = 0;
  std::vector<T> data;
  void Resize(int r, int c) { rows = r; cols = c; data.assign((size_t)r * c, T(0)); }
  T& operator()(int r, int c) { return data[(size_t)r * cols + c]; }
};
}  // namespace kaldi

#define KALDI_ERR ::kaldi::ErrorThrower()
#define KALDI_ASSERT(cond) \
  do { if (!(cond)) throw std::runtime_error("assertion failed: " #cond); } while (0)
