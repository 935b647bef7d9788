// Request ingestion (SURVEY.md §8(f)3): a serialized api.v1.beta1.GetSuggestionsRequest goes straight from wire bytes to
// flat arrays — trial names (spans + 64-bit hashes), conditions, the objective metric and one double per (trial, parameter) —
// without building a message tree.  Katib resends EVERY finished trial as strings on every call (8192 trials × 32 parameters
// = 7.5 MB, 540k sub-messages at cfg3): protobuf-python (upb) parsing it and a Python walk over it cost far more than the GPU step
// when the experiment is new to the service; this scan hands NumPy the matrix directly.
//
// Host-only code (no device work): it lives in libkbo.so so the suggestion service has one native dependency.
// Field numbers are those of kubeflow_b200/suggestion/api_pb.py's SCHEMA table (UNVERIFIED against upstream's api.proto, as
// that file says); tests/test_reqparse.py checks this scan against protobuf's own parse of the same bytes, so the two can
// only be wrong together.  Semantics mirror suggestion/internal.py Trial.convert and base_service.py getSuggestions: a
// trial is usable when its condition is SUCCEEDED or EARLYSTOPPED and it carries the objective metric; with duplicates the
// LAST assignment of a name wins, the LAST metric matching a named objective wins, the FIRST metric when the name is empty.
// A value counts as numeric only if it is a plain decimal literal ([+-]digits[.digits][e[+-]digits]); anything else that
// Python's float()/int() might still accept (spaces, underscores, inf/nan) is flagged and the caller takes the slow path.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/kbo.h"

namespace {

struct Span {
  const uint8_t* p;
  size_t n;
};

inline bool read_varint(const uint8_t*& p, const uint8_t* end, uint64_t& v) {
  v = 0;
  for (int shift = 0; shift < 70 && p < end; shift += 7) {
    const uint8_t b = *p++;
    v |= (uint64_t)(b & 0x7f) << (shift < 64 ? shift : 63);
    if (!(b & 0x80)) return true;
  }
  return false;
}

// One field of a message: number, wire type, varint value (wt 0) or payload span (wt 2).  Returns false on malformed input.
struct Field {
  uint32_t num;
  uint32_t wt;
  uint64_t v;
  Span s;
};
inline bool next_field(const uint8_t*& p, const uint8_t* end, Field& f) {
  uint64_t tag;
  if (!read_varint(p, end, tag)) return false;
  f.num = (uint32_t)(tag >> 3);
  f.wt = (uint32_t)(tag & 7);
  f.v = 0;
  f.s = {nullptr, 0};
  if (f.num == 0) return false;
  switch (f.wt) {
    case 0: return read_varint(p, end, f.v);
    case 1:
      if (end - p < 8) return false;
      p += 8;
      return true;
    case 5:
      if (end - p < 4) return false;
      p += 4;
      return true;
    case 2: {
      uint64_t len;
      if (!read_varint(p, end, len) || len > (uint64_t)(end - p)) return false;
      f.s = {p, (size_t)len};
      p += len;
      return true;
    }
    default: return false;  // groups are not used by proto3 messages
  }
}

inline uint64_t fnv1a(Span s) {
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < s.n; i++) h = (h ^ s.p[i]) * 1099511628211ull;
  return h;
}
inline bool span_eq(Span a, Span b) { return a.n == b.n && (a.n == 0 || memcmp(a.p, b.p, a.n) == 0); }

// plain decimal literal?  bit0: float literal, bit1: integer literal of at most 15 digits (exact in a double)
inline int classify_number(Span s) {
  size_t i = 0;
  const uint8_t* c = s.p;
  if (i < s.n && (c[i] == '+' || c[i] == '-')) i++;
  size_t d0 = i;
  while (i < s.n && c[i] >= '0' && c[i] <= '9') i++;
  const size_t int_digits = i - d0;
  if (i == s.n) return int_digits == 0 ? 0 : (int_digits <= 15 ? 3 : 1);
  size_t frac_digits = 0;
  if (c[i] == '.') {
    i++;
    const size_t f0 = i;
    while (i < s.n && c[i] >= '0' && c[i] <= '9') i++;
    frac_digits = i - f0;
  }
  if (int_digits + frac_digits == 0) return 0;
  if (i < s.n && (c[i] == 'e' || c[i] == 'E')) {
    i++;
    if (i < s.n && (c[i] == '+' || c[i] == '-')) i++;
    const size_t e0 = i;
    while (i < s.n && c[i] >= '0' && c[i] <= '9') i++;
    if (i == e0) return 0;
  }
  return i == s.n ? 1 : 0;
}
inline double parse_double(Span s) {
  char tmp[64];
  if (s.n < sizeof tmp) {
    memcpy(tmp, s.p, s.n);
    tmp[s.n] = 0;
    return strtod(tmp, nullptr);
  }
  return strtod(std::string((const char*)s.p, s.n).c_str(), nullptr);  // correctly rounded, like Python's float()
}

}  // namespace

struct kbo_req {
  const uint8_t* base = nullptr;
  size_t len = 0;
  Span experiment{nullptr, 0};
  bool has_experiment = false;
  int32_t current_request_number = 0, total_request_number = 0;
  std::vector<Span> trials;
};

extern "C" {

int kbo_req_open(const void* bytes, uint64_t len, kbo_req** out) {
  if (!out || (!bytes && len)) return KBO_ERR_INVALID;
  *out = nullptr;
  kbo_req* r = new (std::nothrow) kbo_req;
  if (!r) return KBO_ERR_NOMEM;
  r->base = (const uint8_t*)bytes;
  r->len = (size_t)len;
  const uint8_t* p = r->base;
  const uint8_t* end = p + len;
  Field f;
  while (p < end) {
    if (!next_field(p, end, f)) {
      delete r;
      return KBO_ERR_INVALID;
    }
    if (f.num == 1 && f.wt == 2) {   // experiment (a repeated occurrence would merge; Katib sends one — keep the last, flag nothing)
      r->experiment = f.s;
      r->has_experiment = true;
    } else if (f.num == 2 && f.wt == 2) {
      r->trials.push_back(f.s);
    } else if (f.num == 4 && f.wt == 0) {
      r->current_request_number = (int32_t)f.v;
    } else if (f.num == 5 && f.wt == 0) {
      r->total_request_number = (int32_t)f.v;
    }
  }
  *out = r;
  return KBO_OK;
}

void kbo_req_close(kbo_req* r) { delete r; }

int kbo_req_header(const kbo_req* r, uint64_t* exp_off, uint64_t* exp_len, int32_t* current_request_number, int32_t* total_request_number,
                   int32_t* n_trials) {
  if (!r) return KBO_ERR_INVALID;
  if (exp_off) *exp_off = r->has_experiment ? (uint64_t)(r->experiment.p - r->base) : 0;
  if (exp_len) *exp_len = r->has_experiment ? r->experiment.n : 0;
  if (current_request_number) *current_request_number = r->current_request_number;
  if (total_request_number) *total_request_number = r->total_request_number;
  if (n_trials) *n_trials = (int32_t)r->trials.size();
  return KBO_OK;
}

uint64_t kbo_hash64(const void* bytes, uint64_t len) { return fnv1a({(const uint8_t*)bytes, (size_t)len}); }

int kbo_req_trials(const kbo_req* r, int32_t n_params, const char* const* param_names, uint64_t* name_off, uint32_t* name_len,
                   uint64_t* name_hash, int32_t* condition, uint8_t* usable, double* objective, uint8_t* objective_flags,
                   uint64_t* objective_off, uint32_t* objective_len, double* values, uint8_t* value_flags, uint64_t* value_off,
                   uint32_t* value_len, const uint8_t* select) {
  if (!r || n_params < 0 || (n_params && !param_names)) return KBO_ERR_INVALID;
  std::vector<Span> pn((size_t)n_params);
  for (int j = 0; j < n_params; j++) pn[j] = {(const uint8_t*)param_names[j], strlen(param_names[j])};
  const size_t T = r->trials.size();
  const double nan = std::nan("");
  for (size_t t = 0; t < T; t++) {
    Span name{r->base, 0}, obj_name{nullptr, 0}, target{nullptr, 0};
    bool have_target = false;
    int32_t cond = 0;
    std::vector<Span> metrics_n, metrics_v;   // (name, value) in order; resolved after the objective name is known
    for (int j = 0; j < n_params; j++) {
      const size_t e = t * (size_t)n_params + j;
      if (values) values[e] = nan;
      if (value_flags) value_flags[e] = 0;
      if (value_off) value_off[e] = 0;
      if (value_len) value_len[e] = 0xFFFFFFFFu;   // missing
    }
    const uint8_t* p = r->trials[t].p;
    const uint8_t* end = p + r->trials[t].n;
    Field f;
    while (p < end) {
      if (!next_field(p, end, f)) return KBO_ERR_INVALID;
      if (f.num == 1 && f.wt == 2) {
        name = f.s;
      } else if (f.num == 2 && f.wt == 2) {   // TrialSpec
        const uint8_t* q = f.s.p;
        const uint8_t* qe = q + f.s.n;
        Field g;
        while (q < qe) {
          if (!next_field(q, qe, g)) return KBO_ERR_INVALID;
          if (g.num == 2 && g.wt == 2) {   // ObjectiveSpec -> objective_metric_name = 3
            const uint8_t* u = g.s.p;
            const uint8_t* ue = u + g.s.n;
            Field k;
            while (u < ue) {
              if (!next_field(u, ue, k)) return KBO_ERR_INVALID;
              if (k.num == 3 && k.wt == 2) obj_name = k.s;
            }
          } else if (g.num == 3 && g.wt == 2 && n_params > 0 && (!select || select[t])) {   // ParameterAssignments -> assignments = 1
            const uint8_t* u = g.s.p;
            const uint8_t* ue = u + g.s.n;
            Field k;
            int hint = 0;
            while (u < ue) {
              if (!next_field(u, ue, k)) return KBO_ERR_INVALID;
              if (k.num != 1 || k.wt != 2) continue;
              Span an{nullptr, 0}, av{r->base, 0};
              const uint8_t* w = k.s.p;
              const uint8_t* we = w + k.s.n;
              Field m;
              while (w < we) {
                if (!next_field(w, we, m)) return KBO_ERR_INVALID;
                if (m.num == 1 && m.wt == 2) an = m.s;
                else if (m.num == 2 && m.wt == 2) av = m.s;
              }
              int j = -1;   // assignments normally come in parameter order: try the next slot first
              if (hint < n_params && span_eq(pn[hint], an)) j = hint;
              else
                for (int c = 0; c < n_params; c++)
                  if (span_eq(pn[c], an)) {
                    j = c;
                    break;
                  }
              if (j < 0) continue;
              hint = j + 1;
              const size_t e = t * (size_t)n_params + j;
              const int cls = classify_number(av);
              if (values) values[e] = cls ? parse_double(av) : nan;
              if (value_flags) value_flags[e] = (uint8_t)cls;
              if (value_off) value_off[e] = (uint64_t)(av.p - r->base);
              if (value_len) value_len[e] = (uint32_t)av.n;
            }
          }
        }
      } else if (f.num == 3 && f.wt == 2) {   // TrialStatus
        const uint8_t* q = f.s.p;
        const uint8_t* qe = q + f.s.n;
        Field g;
        while (q < qe) {
          if (!next_field(q, qe, g)) return KBO_ERR_INVALID;
          if (g.num == 3 && g.wt == 0) cond = (int32_t)g.v;
          else if (g.num == 4 && g.wt == 2) {   // Observation -> repeated metrics = 1
            const uint8_t* u = g.s.p;
            const uint8_t* ue = u + g.s.n;
            Field k;
            while (u < ue) {
              if (!next_field(u, ue, k)) return KBO_ERR_INVALID;
              if (k.num != 1 || k.wt != 2) continue;
              Span mn{nullptr, 0}, mv{r->base, 0};
              const uint8_t* w = k.s.p;
              const uint8_t* we = w + k.s.n;
              Field m;
              while (w < we) {
                if (!next_field(w, we, m)) return KBO_ERR_INVALID;
                if (m.num == 1 && m.wt == 2) mn = m.s;
                else if (m.num == 2 && m.wt == 2) mv = m.s;
              }
              metrics_n.push_back(mn);
              metrics_v.push_back(mv);
            }
          }
        }
      }
    }
    // a repeated `observation` field would be merged by protobuf (metrics concatenated): the flat list above does the same
    for (size_t i = 0; i < metrics_n.size(); i++) {
      if (obj_name.n ? span_eq(metrics_n[i], obj_name) : !have_target) {
        target = metrics_v[i];
        have_target = true;
      }
    }
    if (name_off) name_off[t] = (uint64_t)(name.p - r->base);
    if (name_len) name_len[t] = (uint32_t)name.n;
    if (name_hash) name_hash[t] = fnv1a(name);
    if (condition) condition[t] = cond;
    if (usable) usable[t] = (uint8_t)((cond == 2 || cond == 6) && have_target);
    const int ocls = have_target ? classify_number(target) : 0;
    if (objective) objective[t] = ocls ? parse_double(target) : nan;
    if (objective_flags) objective_flags[t] = (uint8_t)ocls;
    if (objective_off) objective_off[t] = have_target ? (uint64_t)(target.p - r->base) : 0;
    if (objective_len) objective_len[t] = have_target ? (uint32_t)target.n : 0xFFFFFFFFu;
  }
  return KBO_OK;
}

}  // extern "C"
