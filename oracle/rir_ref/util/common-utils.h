// String splitting and option registration as rir-generator.h uses them (see base/kaldi-common.h).
#pragma once
#include <cstdlib>
#include <string>
#include <vector>

namespace kaldi {
inline void SplitStringToVector(const std::string& s, const char* delim, bool omit_empty,
                                std::vector<std::string>* out) {
  out->clear();
  size_t start = 0;
  while (true) {
    const size_t end = s.find_first_of(delim, start);
    const std::string piece = s.substr(start, end == std::string::npos ? std::string::npos : end - start);
    if (!(omit_empty && piece.empty())) out->push_back(piece);
    if (end == std::string::npos) break;
    start = end + 1;
  }
}

inline bool SplitStringToFloats(const std::string& s, const char* delim, bool omit_empty,
                                std::vector<float>* out) {
  std::vector<std::string> pieces;
  SplitStringToVector(s, delim, omit_empty, &pieces);
  out->clear();
  for (const std::string& p : pieces) {
    char* end = nullptr;
    out->push_back(std::strtof(p.c_str(), &end));
    if (p.empty() || *end != '\0') return false;
  }
  return true;
}

struct OptionsItf {
  template <class T> void Register(const std::string&, T*, const std::string&) {}
};
}  // namespace kaldi
