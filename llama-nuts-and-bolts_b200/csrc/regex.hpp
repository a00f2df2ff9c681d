// regex.hpp -- a regular expression over UTF-8 text -> a trimmed, minimal byte-level DFA, host-only C++ (DESIGN.md §9g).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace lnb {

// The language of `pattern` is re.fullmatch(pattern, s, re.ASCII) over the UTF-8 encodings of s.  On success: Q states,
// state 0 the start, trans[q * 256 + b] the state after byte b (-1: no string of the language continues that way) and
// accept[q]; every state reaches an accepting one.  Returns false with `err` set for unsupported syntax (the message gives
// the byte offset), for a pattern that matches no string, when an intermediate automaton passes its size bound, and when
// the minimal DFA has more than max_states states.  *n_states (if given): Q, also when Q is past max_states; else 0.
bool regex_dfa(const char* pattern, int64_t len, int max_states, std::vector<int32_t>& trans, std::vector<uint8_t>& accept,
               std::string& err, int* n_states = nullptr);

}  // namespace lnb
