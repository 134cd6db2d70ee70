// Text side of the collect recorder: the per-environment dataset files of collect_data.py:67-78, byte for byte.
// collect_data.py turns each float32 pred_info row into Python floats (.tolist()) and writes
//   str(frame) \t str(id) \t str(px) \t str(py) \n
// str() of a Python float is its shortest round-trip repr (float_repr_style 'short'): the shortest digit string that
// reads back as the same double, positional for decimal exponents -4 <= e < 16 (always with a '.', "12.0"), scientific
// otherwise ("3.0517578125e-05", "1e+16").  std::to_chars gives the same shortest digits; the layout follows CPython's
// format_float_short.
#include <charconv>
#include <errno.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>

#include "../../include/crowdnav_b200.h"
#include "cn_host_util.h"

namespace {

// repr(float(x)) into out (>= 32 bytes); returns the length.  x is finite.
int py_repr(double x, char* out) {
  char sci[40];
  const std::to_chars_result res = std::to_chars(sci, sci + sizeof(sci), x, std::chars_format::scientific);
  *res.ptr = 0;
  const char* q = sci;
  int n = 0;
  if (*q == '-') { out[n++] = '-'; ++q; }
  char digits[24];
  int nd = 0;
  for (; *q && *q != 'e'; ++q)
    if (*q != '.') digits[nd++] = *q;
  const int exp10 = atoi(q + 1);
  if (nd == 1 && digits[0] == '0') {                         // zero
    memcpy(out + n, "0.0", 3);
    return n + 3;
  }
  const int decpt = exp10 + 1;                               // value = 0.d1d2... x 10^decpt
  if (decpt <= -4 || decpt > 16) {
    out[n++] = digits[0];
    if (nd > 1) { out[n++] = '.'; memcpy(out + n, digits + 1, nd - 1); n += nd - 1; }
    n += snprintf(out + n, 8, "e%c%02d", exp10 < 0 ? '-' : '+', exp10 < 0 ? -exp10 : exp10);
    return n;
  }
  if (decpt <= 0) {
    out[n++] = '0'; out[n++] = '.';
    for (int i = 0; i < -decpt; ++i) out[n++] = '0';
    memcpy(out + n, digits, nd); n += nd;
  } else if (decpt >= nd) {
    memcpy(out + n, digits, nd); n += nd;
    for (int i = nd; i < decpt; ++i) out[n++] = '0';
    out[n++] = '.'; out[n++] = '0';
  } else {
    memcpy(out + n, digits, decpt); n += decpt;
    out[n++] = '.';
    memcpy(out + n, digits + decpt, nd - decpt); n += nd - decpt;
  }
  return n;
}

void append_rows(std::string& s, const float* rows, int64_t n) {
  char buf[40];
  for (int64_t r = 0; r < n; ++r) {
    for (int c = 0; c < 4; ++c) {
      s.append(buf, py_repr((double)rows[4 * r + c], buf));
      s.push_back(c == 3 ? '\n' : '\t');
    }
  }
}

}  // namespace

extern "C" {

int64_t cn_format_rows(const float* h_rows, int64_t n, char* out, int64_t cap) {
  if (!h_rows || n < 0) return -1;
  std::string s;
  append_rows(s, h_rows, n);
  if (out && (int64_t)s.size() <= cap) memcpy(out, s.data(), s.size());
  return (int64_t)s.size();
}

int cn_write_rows_txt(const char* dir, const float* h_rows, const int64_t* h_env_rows, int num_envs, int env_base,
                      int append) {
  if (!dir || (!h_rows && num_envs > 0) || !h_env_rows) return cn_set_error("cn_write_rows_txt: null argument");
  std::string s;
  int64_t at = 0;
  for (int e = 0; e < num_envs; ++e) {
    s.clear();
    append_rows(s, h_rows + 4 * at, h_env_rows[e]);
    at += h_env_rows[e];
    const std::string path = std::string(dir) + "/" + std::to_string(env_base + e) + ".txt";
    FILE* f = fopen(path.c_str(), append ? "ab" : "wb");
    if (!f) return cn_set_error("cn_write_rows_txt: cannot open %s: %s", path.c_str(), strerror(errno));
    const size_t w = s.empty() ? 0 : fwrite(s.data(), 1, s.size(), f);
    const int rc = fclose(f);
    if (w != s.size() || rc != 0) return cn_set_error("cn_write_rows_txt: write to %s failed", path.c_str());
  }
  return 0;
}

}  // extern "C"
