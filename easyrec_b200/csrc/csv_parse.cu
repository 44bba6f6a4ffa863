// Host-side text reader for the CSV input path (input/csv_input.py:78-175 -> tf.decode_csv with per-field
// record_defaults; input/input.py:537-675 for what the fields become): one pass over a byte buffer of
// delimiter-separated lines straight into the column arrays the packed batch is made of -- int64 ids,
// Fingerprint64 of string ids, fp32 dense values / fixed-width vectors, CSR lists for Tag / Sequence fields.
// No CUDA: the result is what the trainer copies to the device.  Lines are split across std::threads.
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"

extern "C" uint64_t er_fingerprint64_host(const char* s, size_t len);

namespace er {
namespace {

inline bool is_kv(int kind) { return kind == ER_CSV_I64_KV_LIST || kind == ER_CSV_HASH_KV_LIST; }
inline bool is_steps(int kind) { return kind == ER_CSV_I64_STEP_LIST || kind == ER_CSV_HASH_STEP_LIST; }
inline bool is_list(int kind) {
  return kind == ER_CSV_I64_LIST || kind == ER_CSV_HASH_LIST || kind == ER_CSV_F32_LIST || is_kv(kind) || is_steps(kind);
}

struct Span {
  const char* p;
  size_t n;
};

// decimal int64 with optional sign; surrounding blanks allowed (tf.decode_csv strips them for numbers)
inline bool parse_i64(Span s, int64_t* out) {
  const char* p = s.p;
  const char* e = s.p + s.n;
  while (p < e && (*p == ' ' || *p == '\t')) ++p;
  while (e > p && (e[-1] == ' ' || e[-1] == '\t')) --e;
  if (p == e) return false;
  bool neg = false;
  if (*p == '-' || *p == '+') {
    neg = *p == '-';
    ++p;
  }
  if (p == e) return false;
  while (p + 1 < e && *p == '0') ++p;            // leading zeros do not count towards the 19 digits
  if (e - p > 19) return false;                  // cannot fit int64 (and would wrap the accumulator)
  uint64_t v = 0;
  for (; p < e; ++p) {
    const unsigned d = (unsigned)(*p - '0');
    if (d > 9) return false;
    v = v * 10 + d;
  }
  if (v > (neg ? (uint64_t)1 << 63 : ((uint64_t)1 << 63) - 1)) return false;   // out of range, like decode_csv
  *out = neg ? (int64_t)(0 - v) : (int64_t)v;
  return true;
}

// Correctly rounded decimal -> float.  Fast path (Clinger): at most 7-8 significant digits (mantissa < 2^24)
// and a power of ten that is exact in binary32 (10^0..10^10): one exact int->float conversion and ONE rounded
// multiply or divide, i.e. the same value strtof returns.  Everything else (long mantissas, big exponents,
// inf / nan spellings, hex floats) goes to strtof itself.
inline bool parse_f32(Span s, float* out) {
  static const float kPow10[11] = {1e0f, 1e1f, 1e2f, 1e3f, 1e4f, 1e5f, 1e6f, 1e7f, 1e8f, 1e9f, 1e10f};
  const char* p = s.p;
  const char* e = s.p + s.n;
  while (p < e && (*p == ' ' || *p == '\t')) ++p;
  while (e > p && (e[-1] == ' ' || e[-1] == '\t')) --e;
  if (p == e) return false;
  const char* q = p;
  bool neg = false;
  if (*q == '-' || *q == '+') {
    neg = *q == '-';
    ++q;
  }
  uint32_t m = 0;
  int digits = 0, exp10 = 0;
  bool ok = q < e, seen = false;
  for (; q < e && (unsigned)(*q - '0') <= 9; ++q) {
    seen = true;
    if (m || *q != '0') {
      if (++digits > 7) ok = false;
      m = m * 10 + (unsigned)(*q - '0');
    }
  }
  if (q < e && *q == '.') {
    for (++q; q < e && (unsigned)(*q - '0') <= 9; ++q) {
      seen = true;
      --exp10;
      if (m || *q != '0') {
        if (++digits > 7) ok = false;
      }
      if (ok) m = m * 10 + (unsigned)(*q - '0');
    }
  }
  if (ok && seen && q < e && (*q == 'e' || *q == 'E')) {
    ++q;
    bool eneg = false;
    if (q < e && (*q == '-' || *q == '+')) {
      eneg = *q == '-';
      ++q;
    }
    int ex = 0, nd = 0;
    for (; q < e && (unsigned)(*q - '0') <= 9 && nd < 4; ++q, ++nd) ex = ex * 10 + (*q - '0');
    if (nd == 0 || nd == 4) ok = false;
    exp10 += eneg ? -ex : ex;
  }
  if (ok && seen && q == e && exp10 >= -10 && exp10 <= 10) {
    float v = (float)m;                       // exact: m < 10^7 < 2^24
    v = exp10 < 0 ? v / kPow10[-exp10] : v * kPow10[exp10];
    *out = neg ? -v : v;
    return true;
  }
  char tmp[64];
  const size_t n = (size_t)(e - p);
  if (n >= sizeof(tmp)) return false;
  std::memcpy(tmp, p, n);
  tmp[n] = 0;
  char* end = nullptr;
  const float v = std::strtof(tmp, &end);
  if (end == tmp || *end != 0) return false;
  *out = v;
  return true;
}

// Correctly rounded decimal -> double (strtod), for ExprFeature inputs.  Hex floats are not decimal numbers.
inline bool parse_f64(const char* p, size_t n, double* out) {
  while (n && (*p == ' ' || *p == '\t')) ++p, --n;
  while (n && (p[n - 1] == ' ' || p[n - 1] == '\t')) --n;
  char tmp[128];
  if (n == 0 || n >= sizeof(tmp)) return false;
  std::memcpy(tmp, p, n);
  tmp[n] = 0;
  if (std::strpbrk(tmp, "xX")) return false;
  char* end = nullptr;
  const double v = std::strtod(tmp, &end);
  if (end == tmp || *end != 0) return false;
  *out = v;
  return true;
}

// Fingerprint64 of a string id; with hash_mod the hash bucket (uint64 mod, StringToHashBucketFast) and an
// empty string -> -1, the "no value" id the lookup drops (feature_column_v2.py:2566-2585 ignores '').
inline int64_t hashed(const er_csv_col_t& k, const char* p, size_t n) {
  if (k.hash_mod) {
    if (!n) return -1;
    return (int64_t)(er_fingerprint64_host(p, n) % k.hash_mod);
  }
  return (int64_t)er_fingerprint64_host(p, n);
}

struct LineErr {
  int64_t row = -1;
  int col = 0;
};

}  // namespace
}  // namespace er

extern "C" int er_fingerprint64_i64(const int64_t* values, int64_t n, uint64_t* out) {
  using namespace er;
  ER_REQUIRE((values && out) || n == 0, "null argument");
  char buf[32];
  for (int64_t i = 0; i < n; ++i) {
    const int len = std::snprintf(buf, sizeof(buf), "%lld", (long long)values[i]);   // tf.as_string of an int64
    out[i] = er_fingerprint64_host(buf, (size_t)len);
  }
  return ER_OK;
}

// er_csv_parse_lines: line j of the buffer (0-based) is parsed when j >= line_phase and (j - line_phase) is a
// multiple of line_stride -- rank r of N reads lines r::N of a file this way (dataset.shard(N, r), input/input.py:
// 1018-1023).  Every newline is scanned, only the kept lines are split into fields.  Stops after max_rows kept lines;
// *lines_seen = complete lines passed over (kept or not) up to *consumed, so the caller carries the file's line index.
extern "C" int er_csv_parse_lines(const char* buf, size_t len, char sep, er_csv_col_t* cols, int32_t n_cols,
                                  int64_t max_rows, int32_t n_threads, int64_t line_stride, int64_t line_phase,
                                  int64_t* n_rows, size_t* consumed, int64_t* lines_seen) {
  using namespace er;
  ER_REQUIRE(buf && cols && n_rows && consumed && lines_seen, "null argument");
  ER_REQUIRE(n_cols > 0 && max_rows >= 0, "bad n_cols / max_rows");
  ER_REQUIRE(line_stride >= 1 && line_phase >= 0 && line_phase < line_stride, "bad line_stride / line_phase");
  for (int c = 0; c < n_cols; ++c) {
    const er_csv_col_t& k = cols[c];
    ER_REQUIRE(k.kind >= ER_CSV_SKIP && k.kind <= ER_CSV_F64, "unknown column kind");
    ER_REQUIRE(!is_steps(k.kind) || (k.step_lens && k.width > 0 && k.kv_sep), "step-list column needs step_lens, width and the value separator");
    ER_REQUIRE(k.kind == ER_CSV_SKIP || k.out, "column without an output array");
    ER_REQUIRE(!is_list(k.kind) || (k.lens && k.list_cap >= 0), "list column needs lens and list_cap");
    ER_REQUIRE(!is_kv(k.kind) || (k.weights && k.kv_sep), "key:weight list column needs weights and kv_sep");
    ER_REQUIRE(k.kind != ER_CSV_F32_VEC || k.width > 0, "vector column needs width");
    cols[c].n_vals = 0;
  }
  // ---- the kept complete lines of the buffer: [starts[r], ends[r]) with ends[r] at the '\n' (the tail without '\n' is
  // left to the caller) ----
  std::vector<size_t> starts, ends;
  starts.reserve((size_t)std::min<int64_t>(max_rows, 1 << 20));
  ends.reserve(starts.capacity());
  size_t pos = 0;
  int64_t seen = 0;
  while ((int64_t)starts.size() < max_rows && pos < len) {
    const char* nl = (const char*)std::memchr(buf + pos, '\n', len - pos);
    if (!nl) break;
    if (seen >= line_phase && (seen - line_phase) % line_stride == 0) {
      starts.push_back(pos);
      ends.push_back((size_t)(nl - buf));
    }
    ++seen;
    pos = (size_t)(nl - buf) + 1;
  }
  const int64_t rows = (int64_t)starts.size();
  *n_rows = rows;
  *consumed = pos;
  *lines_seen = seen;
  if (rows == 0) return ER_OK;
  const int T = (int)std::max<int64_t>(1, std::min<int64_t>(n_threads > 0 ? n_threads : 1, (rows + 255) / 256));
  std::vector<LineErr> errs(T);

  // field c of line r; missing trailing fields read as empty (-> the column default)
  auto for_rows = [&](auto&& body) {
    std::vector<std::thread> th;
    for (int t = 0; t < T; ++t) {
      const int64_t r0 = rows * t / T, r1 = rows * (t + 1) / T;
      th.emplace_back([&, t, r0, r1] {
        std::vector<Span> f((size_t)n_cols);
        for (int64_t r = r0; r < r1 && errs[t].row < 0; ++r) {
          const char* p = buf + starts[r];
          const char* e = buf + ends[r];                    // the '\n'
          if (e > p && e[-1] == '\r') --e;
          int c = 0;
          while (c < n_cols) {
            const char* q = (const char*)std::memchr(p, sep, (size_t)(e - p));
            const char* fe = q ? q : e;
            f[c++] = Span{p, (size_t)(fe - p)};
            if (!q) break;
            p = q + 1;
          }
          for (; c < n_cols; ++c) f[c] = Span{e, 0};
          const int bad = body(r, f.data());
          if (bad >= 0) {
            errs[t].row = r;
            errs[t].col = bad;
          }
        }
      });
    }
    for (auto& x : th) x.join();
    for (int t = 0; t < T; ++t)
      if (errs[t].row >= 0) return t;
    return -1;
  };
  auto report = [&](int t) {
    const er_csv_col_t& k = cols[errs[t].col];
    return fail(ER_ERR_INVALID_ARG, "er_csv_parse: line " + std::to_string(line_phase + errs[t].row * line_stride + 1) + ", field " +
                                        std::to_string(errs[t].col + 1) + " is not a valid " +
                                        (k.kind == ER_CSV_F32 || k.kind == ER_CSV_F32_VEC || k.kind == ER_CSV_F32_LIST || k.kind == ER_CSV_F64 ? "float"
                                         : is_kv(k.kind)                                  ? "key:weight list"
                                                                                          : "integer"));
  };

  // ---- pass 1: scalar kinds, and the list lengths ----
  bool any_list = false;
  for (int c = 0; c < n_cols; ++c) any_list |= is_list(cols[c].kind);
  int bad = for_rows([&](int64_t r, const Span* f) -> int {
    for (int c = 0; c < n_cols; ++c) {
      const er_csv_col_t& k = cols[c];
      const Span s = f[c];
      switch (k.kind) {
        case ER_CSV_I64: {
          int64_t v = k.default_i64;
          if (s.n && !parse_i64(s, &v)) return c;
          ((int64_t*)k.out)[r] = v;
          break;
        }
        case ER_CSV_F32: {
          float v = k.default_f32;
          if (s.n && !parse_f32(s, &v)) return c;
          ((float*)k.out)[r] = v;
          break;
        }
        case ER_CSV_F64: {
          const bool dflt = s.n == 0;
          if (!parse_f64(dflt ? k.default_str : s.p, dflt ? (k.default_str ? std::strlen(k.default_str) : 0) : s.n,
                         (double*)k.out + r))
            return c;
          break;
        }
        case ER_CSV_HASH: {
          const char* p = s.p;
          size_t n = s.n;
          if (!n && k.default_str) {
            p = k.default_str;
            n = std::strlen(k.default_str);
          }
          ((int64_t*)k.out)[r] = hashed(k, p, n);
          break;
        }
        case ER_CSV_F32_VEC: {
          float* o = (float*)k.out + r * k.width;
          for (int j = 0; j < k.width; ++j) o[j] = 0.f;
          const char* p = s.p;
          const char* e = s.p + s.n;
          for (int j = 0; j < k.width && p <= e && s.n; ++j) {
            const char* q = (const char*)std::memchr(p, k.inner_sep, (size_t)(e - p));
            const char* fe = q ? q : e;
            float v = k.default_f32;
            if (fe > p && !parse_f32(Span{p, (size_t)(fe - p)}, &v)) return c;
            o[j] = v;
            if (!q) break;
            p = q + 1;
          }
          if (!s.n) o[0] = k.default_f32;
          break;
        }
        case ER_CSV_I64_STEP_LIST:
        case ER_CSV_HASH_STEP_LIST: {   // steps split by inner_sep, the values of a step by kv_sep; empty tokens dropped
          int32_t* sl = k.step_lens + r * k.width;
          for (int j = 0; j < k.width; ++j) sl[j] = 0;
          int32_t steps = 0;
          const char* p = s.p;
          const char* e = s.p + s.n;
          while (p < e && steps < k.width) {   // keep the FIRST width steps
            const char* q = (const char*)std::memchr(p, k.inner_sep, (size_t)(e - p));
            const char* fe = q ? q : e;
            if (fe > p) {
              int32_t cnt = 0;
              const char* vp = p;
              while (vp < fe) {
                const char* vq = (const char*)std::memchr(vp, k.kv_sep, (size_t)(fe - vp));
                const char* ve = vq ? vq : fe;
                cnt += ve > vp;
                vp = ve + 1;
              }
              sl[steps++] = cnt;
            }
            p = fe + 1;
          }
          k.lens[r] = steps;
          break;
        }
        case ER_CSV_HASH_LIST:
        case ER_CSV_I64_KV_LIST:
        case ER_CSV_HASH_KV_LIST:
        case ER_CSV_F32_LIST:
        case ER_CSV_I64_LIST: {   // count the non-empty tokens
          int32_t cnt = 0;
          const char* p = s.p;
          const char* e = s.p + s.n;
          while (p < e) {
            const char* q = (const char*)std::memchr(p, k.inner_sep, (size_t)(e - p));
            const char* fe = q ? q : e;
            cnt += fe > p;
            p = fe + 1;
          }
          if (k.width > 0 && cnt > k.width) cnt = k.width;   // keep the FIRST width tokens
          k.lens[r] = cnt;
          break;
        }
        default:
          break;
      }
    }
    return -1;
  });
  if (bad >= 0) return report(bad);
  if (!any_list) return ER_OK;

  // ---- pass 2: list values at their CSR offsets ----
  std::vector<std::vector<int64_t>> offs((size_t)n_cols);
  for (int c = 0; c < n_cols; ++c) {
    er_csv_col_t& k = cols[c];
    if (!is_list(k.kind)) continue;
    offs[c].resize((size_t)rows + 1);
    int64_t acc = 0;
    for (int64_t r = 0; r < rows; ++r) {
      offs[c][r] = acc;
      if (is_steps(k.kind)) {
        for (int j = 0; j < k.lens[r]; ++j) acc += k.step_lens[r * k.width + j];
      } else {
        acc += k.lens[r];
      }
    }
    offs[c][rows] = acc;
    k.n_vals = acc;
    if (acc > k.list_cap)
      return fail(ER_ERR_WORKSPACE, "er_csv_parse: list column " + std::to_string(c + 1) + " holds " +
                                        std::to_string(acc) + " values, capacity " + std::to_string(k.list_cap));
  }
  bad = for_rows([&](int64_t r, const Span* f) -> int {
    for (int c = 0; c < n_cols; ++c) {
      const er_csv_col_t& k = cols[c];
      if (!is_list(k.kind)) continue;
      int32_t left = k.lens[r];
      const char* p = f[c].p;
      const char* e = p + f[c].n;
      if (is_steps(k.kind)) {                      // the values of the first lens[r] non-empty steps, step by step
        int64_t* ov = (int64_t*)k.out + offs[c][r];
        int32_t steps = 0;
        while (p < e && steps < left) {
          const char* q = (const char*)std::memchr(p, k.inner_sep, (size_t)(e - p));
          const char* fe = q ? q : e;
          if (fe > p) {
            const char* vp = p;
            while (vp < fe) {
              const char* vq = (const char*)std::memchr(vp, k.kv_sep, (size_t)(fe - vp));
              const char* ve = vq ? vq : fe;
              if (ve > vp) {
                if (k.kind == ER_CSV_HASH_STEP_LIST)
                  *ov = hashed(k, vp, (size_t)(ve - vp));
                else if (!parse_i64(Span{vp, (size_t)(ve - vp)}, ov))
                  return c;
                ++ov;
              }
              vp = ve + 1;
            }
            ++steps;
          }
          p = fe + 1;
        }
        continue;
      }
      if (k.kind == ER_CSV_F32_LIST) {             // a ragged float list (the weight input of a TagFeature)
        float* of = (float*)k.out + offs[c][r];
        while (p < e && left > 0) {
          const char* q = (const char*)std::memchr(p, k.inner_sep, (size_t)(e - p));
          const char* fe = q ? q : e;
          if (fe > p) {
            if (!parse_f32(Span{p, (size_t)(fe - p)}, of)) return c;
            ++of;
            --left;
          }
          p = fe + 1;
        }
        continue;
      }
      int64_t* o = (int64_t*)k.out + offs[c][r];
      while (p < e && left > 0) {
        const char* q = (const char*)std::memchr(p, k.inner_sep, (size_t)(e - p));
        const char* fe = q ? q : e;
        if (fe > p) {
          const char* ke = fe;                       // end of the key part of the token
          if (is_kv(k.kind)) {                       // "key<kv_sep>weight": both parts are mandatory (input.py:447-458)
            const char* kv = (const char*)std::memchr(p, k.kv_sep, (size_t)(fe - p));
            float* w = k.weights + (o - (int64_t*)k.out);
            if (!kv || !parse_f32(Span{kv + 1, (size_t)(fe - kv - 1)}, w)) return c;
            ke = kv;
          }
          if (k.kind == ER_CSV_HASH_LIST || k.kind == ER_CSV_HASH_KV_LIST)
            *o = hashed(k, p, (size_t)(ke - p));
          else if (!parse_i64(Span{p, (size_t)(ke - p)}, o))
            return c;
          ++o;
          --left;
        }
        p = fe + 1;
      }
    }
    return -1;
  });
  if (bad >= 0) return report(bad);
  return ER_OK;
}

// every line of the buffer: the stride-1 case of er_csv_parse_lines
extern "C" int er_csv_parse(const char* buf, size_t len, char sep, er_csv_col_t* cols, int32_t n_cols,
                            int64_t max_rows, int32_t n_threads, int64_t* n_rows, size_t* consumed) {
  int64_t seen = 0;
  return er_csv_parse_lines(buf, len, sep, cols, n_cols, max_rows, n_threads, 1, 0, n_rows, consumed, &seen);
}
