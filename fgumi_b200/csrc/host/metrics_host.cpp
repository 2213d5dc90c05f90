// `fgumi duplex-metrics` / `fgumi simplex-metrics` from raw BAM records (src/lib/commands/{shared_metrics,
// duplex_metrics,simplex_metrics}.rs, crates/fgumi-metrics/src/{duplex,simplex,shared}.rs): the collector
// (fgb_metrics_*) and its host exports.  The host does the header-level work -- record checks, the consensus-input
// check, QNAME runs and Template::from_records order, the interval table -- and cuts each call into staged runs of
// whole templates; the template pass and the family counting run on the device (metrics_kernels.cuh behind
// metrics_device.h), the UMI consensus of the 100 % fraction and the tables on host threads.  Restated in
// tests/metrics_oracle.py.
#include <cuda_runtime.h>

#include <algorithm>
#include <charconv>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <new>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "bam.h"
#include "group_rules.h"
#include "metrics_device.h"
#include "metrics_rules.h"
#include "prep.h"
#include "record_link.h"
#include "umi_host.h"

namespace {

namespace mt = fgb::metrics;
namespace link = fgb::link;
using link::ms_since;
constexpr int kF = mt::kFractions;
constexpr uint64_t kDictBit = 1ull << 63;

// ---- intervals (parse_intervals, shared_metrics.rs:197-253) -----------------------------------------------------
struct Interval {
  std::string name;
  int64_t start, end;   // 0-based half-open
};

bool parse_i32(std::string_view s, int64_t* v) {   // Rust's i32::from_str: an optional sign, then decimal digits
  size_t i = 0;
  bool neg = false;
  if (i < s.size() && (s[i] == '+' || s[i] == '-')) neg = s[i++] == '-';
  if (i == s.size()) return false;
  int64_t x = 0;
  for (; i < s.size(); ++i) {
    if (s[i] < '0' || s[i] > '9') return false;
    x = x * 10 + (s[i] - '0');
    if (x > 2147483648ll) return false;
  }
  x = neg ? -x : x;
  if (x > 2147483647ll || x < -2147483648ll) return false;
  *v = x;
  return true;
}

bool is_ws(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\f' || c == '\v'; }

// "" or why the text is refused.  A line starting with '@' switches to the Picard interval list's 1-based starts.
std::string parse_intervals(std::string_view text, std::vector<Interval>* out) {
  bool picard = false;
  size_t p = 0;
  while (p < text.size()) {
    size_t e = text.find('\n', p);
    if (e == std::string_view::npos) e = text.size();
    std::string_view ln = text.substr(p, e - p);
    p = e + 1;
    while (!ln.empty() && is_ws(ln.front())) ln.remove_prefix(1);
    while (!ln.empty() && is_ws(ln.back())) ln.remove_suffix(1);
    if (ln.empty() || ln[0] == '#') continue;
    if (ln[0] == '@') { picard = true; continue; }
    std::string_view f[3];
    int nf = 0;
    size_t q = 0;
    while (nf < 3 && q <= ln.size()) {   // splitn(4, '\t'): the first three fields
      size_t t = ln.find('\t', q);
      if (t == std::string_view::npos) t = ln.size();
      f[nf++] = ln.substr(q, t - q);
      if (t == ln.size()) { q = ln.size() + 1; break; }
      q = t + 1;
    }
    if (nf < 3) return std::string("Invalid ") + (picard ? "interval list" : "BED") + " line (needs at least 3 fields): " +
                       std::string(ln);
    int64_t s, en;
    if (!parse_i32(f[1], &s)) return "Invalid start position: " + std::string(f[1]);
    if (!parse_i32(f[2], &en)) return "Invalid end position: " + std::string(f[2]);
    out->push_back({std::string(f[0]), picard ? s - 1 : s, en});
  }
  return "";
}

// The interval table of IvTable for the header's @SQ names: a contig's intervals by start with running maximum ends
struct IvHost {
  std::vector<uint32_t> sq_begin;
  std::vector<int64_t> start, maxend;
  bool active = false;
  mt::IvTable table() const {
    return mt::IvTable{sq_begin.data(), start.data(), maxend.data(), static_cast<uint32_t>(sq_begin.size() - 1), active};
  }
};

void build_iv(const std::vector<std::string>& sq, const std::vector<Interval>& ivs, IvHost* h) {
  std::unordered_map<std::string, std::vector<std::pair<int64_t, int64_t>>> by;
  for (const auto& v : ivs) by[v.name].push_back({v.start, v.end});
  h->active = !ivs.empty();   // an empty interval file filters nothing (overlaps_intervals, :272-274)
  h->sq_begin.assign(1, 0);
  for (const auto& name : sq) {
    auto it = by.find(name);
    if (it != by.end()) {
      auto v = it->second;
      std::sort(v.begin(), v.end());
      int64_t mx = INT64_MIN;
      for (const auto& x : v) {
        h->start.push_back(x.first);
        mx = std::max(mx, x.second);
        h->maxend.push_back(mx);
      }
    }
    h->sq_begin.push_back(static_cast<uint32_t>(h->start.size()));
  }
}

// ---- names: String::from_utf8_lossy then encode_utf16 (shared_metrics.rs:502, 130) ------------------------------
std::vector<uint16_t> lossy_utf16(const uint8_t* s, size_t n) {
  std::vector<uint16_t> u;
  u.reserve(n);
  auto push = [&](uint32_t cp) {
    if (cp < 0x10000) { u.push_back(static_cast<uint16_t>(cp)); return; }
    cp -= 0x10000;
    u.push_back(static_cast<uint16_t>(0xD800 + (cp >> 10)));
    u.push_back(static_cast<uint16_t>(0xDC00 + (cp & 0x3FF)));
  };
  size_t i = 0;
  while (i < n) {
    const uint8_t c = s[i];
    if (c < 0x80) { push(c); ++i; continue; }
    uint32_t need, cp;
    uint8_t lo = 0x80, hi = 0xBF;
    if (c >= 0xC2 && c <= 0xDF) { need = 1; cp = c & 0x1F; }
    else if (c >= 0xE0 && c <= 0xEF) { need = 2; cp = c & 0x0F; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { need = 3; cp = c & 0x07; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
    else { push(0xFFFD); ++i; continue; }
    size_t j = i + 1;
    bool ok = true;
    for (uint32_t k = 0; k < need; ++k, ++j) {   // one U+FFFD per maximal invalid prefix
      const uint8_t d = j < n ? s[j] : 0;
      const uint8_t l = k == 0 ? lo : 0x80, h = k == 0 ? hi : 0xBF;
      if (j >= n || d < l || d > h) { ok = false; break; }
      cp = (cp << 6) | (d & 0x3F);
    }
    if (!ok) { push(0xFFFD); i = j; continue; }
    push(cp);
    i = j;
  }
  return u;
}

int32_t name_hash(const uint8_t* s, size_t n) {
  const std::vector<uint16_t> u = lossy_utf16(s, n);
  return mt::murmur3_units([&](uint32_t i) { return u[i]; }, static_cast<uint32_t>(u.size()), 42);
}

// ---- the TSV text: csv 1.1 over serde, floats by ryu 1.0 (DESIGN.md section 13) -----------------------------------
// ryu's format64 layout over the shortest round-trip digits d (|d| = len) and exponent k (value = d * 10^k):
// kk = len + k; 0 <= k and kk <= 16: digits, zeros, ".0"; 0 < kk <= 16: a point inside; -5 < kk <= 0: "0." and
// zeros; otherwise d[0] [. rest] 'e' (kk - 1).  Zero is "0.0".
std::string fmt_f64(double v) {
  if (v == 0) return std::signbit(v) ? "-0.0" : "0.0";
  char buf[64];
  const auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::scientific);
  std::string s(buf, r.ptr);
  std::string out;
  if (s[0] == '-') { out = "-"; s.erase(0, 1); }
  const size_t ep = s.find('e');
  const int exp10 = std::atoi(s.c_str() + ep + 1);
  std::string d;
  for (size_t i = 0; i < ep; ++i)
    if (s[i] != '.') d.push_back(s[i]);
  const int len = static_cast<int>(d.size()), kk = exp10 + 1, k = kk - len;
  if (k >= 0 && kk <= 16) out += d + std::string(k, '0') + ".0";
  else if (kk > 0 && kk <= 16) out += d.substr(0, kk) + "." + d.substr(kk);
  else if (kk > -5 && kk <= 0) out += "0." + std::string(-kk, '0') + d;
  else if (len == 1) out += d + "e" + std::to_string(kk - 1);
  else out += d.substr(0, 1) + "." + d.substr(1) + "e" + std::to_string(kk - 1);
  return out;
}

double frac(uint64_t n, uint64_t d) { return d ? static_cast<double>(n) / static_cast<double>(d) : 0.0; }

// csv's necessary quoting: a field with the delimiter, a quote or a line end is quoted, quotes doubled
std::string field(const std::string& s) {
  if (s.find_first_of("\t\"\r\n") == std::string::npos) return s;
  std::string q = "\"";
  for (char c : s) { if (c == '"') q += '"'; q += c; }
  return q + "\"";
}

struct Table {   // header written before the first row only: no rows, no text
  const char* header;
  std::string text;
  void row(std::initializer_list<std::string> cells) {
    if (text.empty()) text = std::string(header) + "\n";
    bool first = true;
    for (const auto& c : cells) { if (!first) text += '\t'; text += c; first = false; }
    text += '\n';
  }
};
std::string u(uint64_t v) { return std::to_string(v); }

// ---- UMI counting (UmiCountTracker, fgumi-metrics shared.rs:64-135) ---------------------------------------------
struct UmiCount { uint64_t raw = 0, err = 0, unique = 0; };
using UmiMap = std::unordered_map<std::string, UmiCount>;
void record_umi(UmiMap& m, const std::string& umi, uint64_t raw, uint64_t err) {
  UmiCount& c = m[umi];
  c.raw += raw;
  c.err += err;
  c.unique += 1;
}

// SimpleUmiConsensusCaller::consensus (simple_umi.rs:170-193): one UMI as it is, unequal lengths the first UMI, else
// the column-wise call; false where the reference panics
bool umi_consensus(const fgb::prep::UmiBuilder& b, const std::vector<std::string>& umis, std::string* out) {
  if (umis.size() <= 1) { *out = umis.empty() ? std::string() : umis[0]; return true; }
  for (const auto& x : umis)
    if (x.size() != umis[0].size()) { *out = umis[0]; return true; }
  return fgb::prep::consensus_umis(b, umis, out);
}

std::vector<std::string> split_dash(std::string_view s) {
  std::vector<std::string> v;
  size_t p = 0;
  while (true) {
    const size_t e = s.find('-', p);
    v.emplace_back(s.substr(p, e == std::string_view::npos ? std::string_view::npos : e - p));
    if (e == std::string_view::npos) return v;
    p = e + 1;
  }
}

// P(lower <= A <= upper), A ~ Binomial(n, 0.5), lower <= upper <= n: every term relative to the mode's by the ratio
// pmf(k + 1) / pmf(k) = (n - k) / (k + 1), the interval's terms over all of them.  A term is off by about its distance
// from the mode in ulps, and no two CDFs near 0.5 are subtracted, so a short interval amid the mass (min-ab and
// min-ba near n / 2) keeps its relative accuracy; lgamma terms lose ~ n ulps of lgamma(n) at large n.
double binom_interval_half(uint64_t lower, uint64_t upper, uint64_t n) {
  const uint64_t m = n / 2;
  double all = 1.0, in = lower <= m && m <= upper ? 1.0 : 0.0, t = 1.0;
  for (uint64_t k = m; k < n && t > 0; ++k) {   // t = pmf(k + 1) / pmf(m)
    t *= static_cast<double>(n - k) / static_cast<double>(k + 1);
    all += t;
    if (k + 1 >= lower && k + 1 <= upper) in += t;
  }
  t = 1.0;
  for (uint64_t k = m; k > 0 && t > 0; --k) {   // t = pmf(k - 1) / pmf(m)
    t *= static_cast<double>(k) / static_cast<double>(n - k + 1);
    all += t;
    if (k - 1 >= lower && k - 1 <= upper) in += t;
  }
  return in / all;
}

}  // namespace

// ---- the collector ---------------------------------------------------------------------------------------------
struct fgb_metrics {
  fgb_metrics_options opt{};
  int device = -1;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  std::vector<std::string> sq;
  IvHost iv;
  mt::IvTable d_iv{};
  void* d_iv_mem = nullptr;
  std::string last_error;
  bool checked_consensus = false, poisoned = false, finished = false;
  uint64_t records_seen = 0;
  uint64_t stats[FGB_METRICS_NSTATS] = {};
  double timing[4] = {0, 0, 0, 0};
  // kept templates not yet counted: the open coordinate group and whatever precedes it
  std::vector<mt::FTpl> pend;
  std::vector<uint64_t> pend_rec;        // the template's first record (over every call)
  std::vector<uint8_t> pend_kind;
  std::string pend_rx;
  std::vector<uint64_t> pend_rx_off{0};
  std::unordered_map<std::string, uint64_t> dict;   // non-canonical MI bases
  // per fraction: size -> count (CS, SS, DS), (ab, ba) -> count, templates
  std::map<uint64_t, uint64_t> sizes[3][kF];
  std::map<std::pair<uint64_t, uint64_t>, uint64_t> pairs[kF];
  uint64_t templates[kF] = {};
  UmiMap umi, dumi;
  fgb::prep::UmiBuilder builder;
  std::string tables[5];
  bool has_table[5] = {false, false, false, false, false};
  ~fgb_metrics() {
    if (device >= 0) {
      cudaSetDevice(device);
      if (d_iv_mem) cudaFree(d_iv_mem);
      if (stream) cudaStreamDestroy(stream);
    }
  }
};

namespace {

fgb_status fail_at(fgb_metrics* m, fgb_status st, uint64_t rec, const std::string& why, uint64_t* bad) {
  m->poisoned = true;
  if (bad) *bad = rec;
  m->last_error = why;
  return st;
}

// The UMI metrics of DS runs [r0, r1) of `order` (indices into pend, in (group, base) order, stream order within a
// run; run r = order[rs[r] .. rs[r + 1])) on this thread: duplex_metrics.rs:515-602 / simplex_metrics.rs:262-293.
// *bad = the pend index of the first template of the first family whose consensus fails.
void umi_runs(const fgb_metrics& m, const std::vector<uint32_t>& order, const std::vector<uint32_t>& rs, uint64_t r0,
              uint64_t r1, UmiMap* um, UmiMap* dm, uint64_t* bad) {
  const bool duplex = m.opt.mode == FGB_METRICS_DUPLEX;
  std::vector<std::string> u1, u2, parts;
  std::vector<std::vector<std::string>> split;
  std::string c1, c2;
  for (uint64_t r = r0; r < r1; ++r) {
    const uint32_t b = rs[r], e = rs[r + 1];
    auto rx = [&](uint32_t i) {
      const uint32_t t = order[i];
      return std::string_view(m.pend_rx).substr(m.pend_rx_off[t], m.pend_rx_off[t + 1] - m.pend_rx_off[t]);
    };
    auto failed = [&]() { *bad = std::min<uint64_t>(*bad, order[b]); };
    if (duplex) {
      u1.clear();
      u2.clear();
      for (uint32_t i = b; i < e; ++i) {
        const uint8_t kind = m.pend_kind[order[i]];
        parts = split_dash(rx(i));
        if (parts.size() != 2 || parts[0].empty() || parts[1].empty() || kind == 0) continue;
        u1.push_back(kind == 1 ? parts[0] : parts[1]);
        u2.push_back(kind == 1 ? parts[1] : parts[0]);
      }
      int got = 0;
      if (!u1.empty()) {
        if (!umi_consensus(m.builder, u1, &c1)) { failed(); continue; }
        uint64_t err = 0;
        for (const auto& x : u1) err += x != c1;
        record_umi(*um, c1, u1.size(), err);
        ++got;
      }
      if (!u2.empty()) {
        if (!umi_consensus(m.builder, u2, &c2)) { failed(); continue; }
        uint64_t err = 0;
        for (const auto& x : u2) err += x != c2;
        record_umi(*um, c2, u2.size(), err);
        ++got;
      }
      if (m.opt.duplex_umi_counts && got == 2) {
        const std::string d1 = c1 + "-" + c2, d2 = c2 + "-" + c1;
        uint64_t err = 0;
        for (uint32_t i = b; i < e; ++i) err += rx(i) != d1 && rx(i) != d2;
        record_umi(*dm, d1, u1.size(), err);
      }
    } else {
      split.clear();
      for (uint32_t i = b; i < e; ++i) split.push_back(split_dash(rx(i)));
      const size_t nc = split.empty() ? 0 : split[0].size();
      for (size_t pos = 0; pos < nc; ++pos) {
        u1.clear();
        for (const auto& s : split)
          if (pos < s.size() && !s[pos].empty()) u1.push_back(s[pos]);
        if (u1.empty()) continue;
        if (!umi_consensus(m.builder, u1, &c1)) { failed(); break; }
        uint64_t err = 0;
        for (const auto& x : u1) err += x != c1;
        record_umi(*um, c1, u1.size(), err);
      }
    }
  }
}

// Counts the first n pending templates (whole coordinate groups) on the device, folds the histograms in and runs the
// UMI consensus; drops them from the pending lists.  *bad_tpl = the pend index of a failing UMI family's first
// template (UINT64_MAX: none).
fgb_status count_closed(fgb_metrics* m, uint64_t n, uint64_t* bad_tpl) {
  *bad_tpl = UINT64_MAX;
  if (!n) return FGB_OK;
  auto fail = [&](cudaError_t e, const char* what) { return link::fail(&m->last_error, "fgb_metrics", e, what); };
  auto t0 = std::chrono::steady_clock::now();
  link::Resources r(m->stream, m->opt.n_threads);
  const uint32_t nn = static_cast<uint32_t>(n);
  uint64_t maxb = 1;
  for (uint64_t i = 0; i < n; ++i) maxb = std::max(maxb, m->pend[i].base);
  int base_bits = 1;
  while (base_bits < 64 && (maxb >> base_bits)) ++base_bits;
  mt::FamilyBufs b{};
  mt::FTpl* d_t;
  unsigned long long *d_sizes, *d_pairs, *d_tpl, *d_nover;
  mt::Overflow* d_over;
  const uint64_t cap = 6 * n + 64;
  cudaError_t e;
  if ((e = mt::family_temp_bytes(nn, &b.temp_bytes))) return fail(e, "CUB temp storage");
  uint8_t* d_temp;
  const uint64_t n_sizes = 3ull * kF * mt::kSmall, n_pairs = 1ull * kF * mt::kPair * mt::kPair;
  if ((e = r.alloc(&d_t, n)) || (e = r.alloc(&b.flag, n)) || (e = r.alloc(&b.gid, n)) ||
      (e = r.alloc(&b.group_start, n)) || (e = r.alloc(&b.perm_a, n)) || (e = r.alloc(&b.perm_b, n)) ||
      (e = r.alloc(&b.key_a, n)) || (e = r.alloc(&b.key_b, n)) || (e = r.alloc(&b.run_start, n + 1)) ||
      (e = r.alloc(&b.counts, 2)) || (e = r.alloc(&b.base_a, n)) || (e = r.alloc(&b.base_b, n)) ||
      (e = r.alloc(&d_temp, b.temp_bytes + 16)) || (e = r.alloc(&d_sizes, n_sizes + n_pairs + kF + 1)) ||
      (e = r.alloc(&d_over, cap)))
    return fail(e, "cudaMalloc");
  b.temp = d_temp;
  d_pairs = d_sizes + n_sizes;
  d_tpl = d_pairs + n_pairs;
  d_nover = d_tpl + kF;
  const char* what;
  if ((e = r.open(std::min<uint64_t>(link::kStageBytes, std::max<uint64_t>(n * sizeof(mt::FTpl), 4096)), &what)))
    return fail(e, what);
  if ((e = r.upload(d_t, m->pend.data(), n * sizeof(mt::FTpl))) ||
      (e = cudaMemsetAsync(d_sizes, 0, (n_sizes + n_pairs + kF + 1) * 8, m->stream)))
    return fail(e, "upload");
  const mt::Hist h{d_sizes, d_pairs, d_tpl, d_over, d_nover, cap};
  if ((e = mt::family_pass(d_t, nn, base_bits, b, h, m->stream))) return fail(e, "family pass");
  std::vector<unsigned long long> hist(n_sizes + n_pairs + kF + 1);
  uint32_t counts[2];
  if ((e = cudaMemcpyAsync(hist.data(), d_sizes, hist.size() * 8, cudaMemcpyDeviceToHost, m->stream)) ||
      (e = cudaMemcpyAsync(counts, b.counts, 8, cudaMemcpyDeviceToHost, m->stream)) ||
      (e = cudaStreamSynchronize(m->stream)))
    return fail(e, "family pass");
  const uint64_t n_over = hist.back();
  if (n_over > cap) { m->last_error = "fgb_metrics: overflow list exceeded its bound"; return FGB_ERR_CUDA; }
  std::vector<mt::Overflow> over(n_over);
  std::vector<uint32_t> order(n), rs(counts[1] + 1);
  if ((e = r.download(over.data(), d_over, n_over * sizeof(mt::Overflow))) ||
      (e = r.download(order.data(), b.perm_a, n * 4)) || (e = r.download(rs.data(), b.run_start, counts[1] * 4ull)))
    return fail(e, "download");
  rs[counts[1]] = nn;
  m->timing[1] += ms_since(t0);
  auto t1 = std::chrono::steady_clock::now();
  for (int k = 0; k < 3; ++k)
    for (int f = 0; f < kF; ++f)
      for (int s = 0; s < mt::kSmall; ++s)
        if (const uint64_t c = hist[(k * kF + f) * mt::kSmall + s]) m->sizes[k][f][s] += c;
  for (int f = 0; f < kF; ++f) {
    for (int a = 0; a < mt::kPair; ++a)
      for (int c = 0; c < mt::kPair; ++c)
        if (const uint64_t v = hist[n_sizes + (f * mt::kPair + a) * mt::kPair + c]) m->pairs[f][{a, c}] += v;
    m->templates[f] += hist[n_sizes + n_pairs + f];
  }
  for (const auto& o : over) {
    const uint32_t k = o.code >> 8, f = o.code & 0xFF;
    if (k == mt::kDup) m->pairs[f][{o.a, o.b}] += 1;
    else m->sizes[k][f][o.a] += 1;
  }
  m->stats[FGB_MSTAT_GROUPS] += counts[0];
  m->stats[FGB_MSTAT_DS_FAMILIES] += counts[1];
  m->stats[FGB_MSTAT_OVERFLOW] += n_over;
  m->timing[3] += ms_since(t1);
  // the UMI consensus of the 100 % fraction (every kept template is in it), on host threads by DS runs
  t1 = std::chrono::steady_clock::now();
  const uint64_t nr = counts[1], nt = std::max<uint64_t>(1, std::min<uint64_t>(std::max<uint32_t>(m->opt.n_threads, 1),
                                                                                 nr / 64 + 1));
  std::vector<UmiMap> ums(nt), dms(nt);
  std::vector<uint64_t> bads(nt, UINT64_MAX);
  fgb_umi::parallel_for(nt, m->opt.n_threads, [&](uint64_t w) {
    umi_runs(*m, order, rs, nr * w / nt, nr * (w + 1) / nt, &ums[w], &dms[w], &bads[w]);
  });
  for (uint64_t w = 0; w < nt; ++w) {
    *bad_tpl = std::min(*bad_tpl, bads[w]);
    for (const auto& kv : ums[w]) {
      UmiCount& c = m->umi[kv.first];
      c.raw += kv.second.raw; c.err += kv.second.err; c.unique += kv.second.unique;
    }
    for (const auto& kv : dms[w]) {
      UmiCount& c = m->dumi[kv.first];
      c.raw += kv.second.raw; c.err += kv.second.err; c.unique += kv.second.unique;
    }
  }
  m->timing[2] += ms_since(t1);
  if (*bad_tpl != UINT64_MAX) return FGB_OK;
  // drop the counted templates
  m->pend.erase(m->pend.begin(), m->pend.begin() + n);
  m->pend_rec.erase(m->pend_rec.begin(), m->pend_rec.begin() + n);
  m->pend_kind.erase(m->pend_kind.begin(), m->pend_kind.begin() + n);
  const uint64_t cut = m->pend_rx_off[n];
  m->pend_rx.erase(0, cut);
  m->pend_rx_off.erase(m->pend_rx_off.begin(), m->pend_rx_off.begin() + n);
  for (auto& o : m->pend_rx_off) o -= cut;
  return FGB_OK;
}

bool same_key(const mt::FTpl& x, const mt::FTpl& y) {
  return x.ref1 == y.ref1 && x.start1 == y.start1 && x.strand1 == y.strand1 && x.ref2 == y.ref2 &&
         x.start2 == y.start2 && x.strand2 == y.strand2;
}

// The pending templates before the last coordinate group's first one
uint64_t closed_count(const fgb_metrics& m) {
  uint64_t n = m.pend.size();
  if (!n) return 0;
  while (n > 1 && same_key(m.pend[n - 1], m.pend[n - 2])) --n;
  return n - 1;
}

fgb_status umi_failure(fgb_metrics* m, uint64_t tpl, uint64_t* bad) {
  return fail_at(m, FGB_ERR_INVALID_ARG, m->pend_rec[tpl], "fgb_metrics: record " + std::to_string(m->pend_rec[tpl]) +
                 ": the UMI consensus of its tag family fails: its RX parts mix DNA and other characters", bad);
}

const char* status_text(uint8_t st) {
  switch (st) {
    case FGB_MT_ERR_MI_MISSING: return "is missing the required MI tag. Metrics commands require standard MI/RX tags.";
    case FGB_MT_ERR_MI_UTF8: return "has an MI tag that is not UTF-8";
    case FGB_MT_ERR_RX_MISSING: return "is missing the required RX tag. Metrics commands require standard MI/RX tags.";
    default: return "has an RX tag that is not UTF-8";
  }
}

// Templates of records [0, n): QNAME runs and their primary slots (template_order).  Returns the index of the first
// bad record (n: none) and sets *err / *st.
uint64_t templates_of(const uint8_t* records, const uint64_t* rec_off, uint64_t n, std::vector<uint64_t>* first,
                      std::vector<int64_t>* prim, std::string* err, fgb_status* st) {
  uint64_t hb = n;
  for (uint64_t i = 0; i < n; ++i)
    if (!fgb::grp::record_ok(records, rec_off, i)) {
      hb = i;
      *err = "is malformed: it is shorter than 32 bytes or its name, CIGAR or fields run past its end";
      *st = FGB_ERR_LAYOUT;
      break;
    }
  std::vector<uint64_t> lists[4], ord;
  first->assign(1, 0);
  for (uint64_t i = 0; i < hb;) {
    const fgb::bam::View vi(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
    const std::string_view name = fgb::grp::read_name(vi);
    uint64_t j = i + 1;
    while (j < hb && fgb::grp::read_name(fgb::bam::View(records + rec_off[j], rec_off[j + 1] - rec_off[j])) == name) ++j;
    if (j == hb && hb < n) break;   // the run the bad record cuts short is not a template
    int64_t r1, r2;
    uint64_t dup;
    ord.clear();
    const std::string e = fgb::grp::template_order(
        i, j, [&](uint64_t k) { return fgb::bam::rd16(records + rec_off[k] + 14); }, name, lists, &ord, &r1, &r2, &dup);
    if (!e.empty()) {
      hb = dup;
      *err = e;
      *st = FGB_ERR_INVALID_ARG;
      break;
    }
    prim->push_back(r1);
    prim->push_back(r2);
    first->push_back(j);
    i = j;
  }
  return hb;
}

// The first paired, primary R1 decides whether the input is a consensus BAM (validate_not_consensus_bam,
// shared_metrics.rs:300-350): aD and bD, or cD, refuse it
bool consensus_input(fgb_metrics* m, const uint8_t* records, const uint64_t* rec_off, uint64_t n, uint64_t* at) {
  for (uint64_t i = 0; i < n && !m->checked_consensus; ++i) {
    if (rec_off[i + 1] < rec_off[i] || rec_off[i + 1] - rec_off[i] < 32) return false;
    const uint8_t* r = records + rec_off[i];
    const uint16_t f = fgb::bam::rd16(r + 14);
    if (!(f & 0x1) || !(f & 0x40) || (f & 0x100) || (f & 0x800)) continue;
    m->checked_consensus = true;
    const fgb::bam::View v(r, rec_off[i + 1] - rec_off[i]);
    if (!fgb::grp::record_ok(records, rec_off, i)) return false;
    const uint8_t* aux = r + v.aux_off();
    const size_t an = v.n - v.aux_off();
    const bool duplex = fgb::rfilter::has_tag(aux, an, "aD") && fgb::rfilter::has_tag(aux, an, "bD");
    if (duplex || fgb::rfilter::has_tag(aux, an, "cD")) { *at = i; return true; }
  }
  return false;
}

fgb_status add_impl(fgb_metrics* m, const uint8_t* records, const uint64_t* rec_off, uint64_t n, uint64_t* bad) {
  auto t_host = std::chrono::steady_clock::now();
  const uint64_t g0 = m->records_seen;
  uint64_t ci;
  if (consensus_input(m, records, rec_off, n, &ci))
    return fail_at(m, FGB_ERR_INVALID_ARG, g0 + ci, "fgb_metrics: record " + std::to_string(g0 + ci) +
                   ": the input appears to contain consensus sequences; the metrics need the UMI-grouped records that "
                   "group writes before consensus calling", bad);
  std::vector<uint64_t> first;
  std::vector<int64_t> prim;
  std::string herr;
  fgb_status hst = FGB_OK;
  const uint64_t hb = templates_of(records, rec_off, n, &first, &prim, &herr, &hst);
  const uint64_t n_tpl = first.size() - 1;
  auto fail = [&](cudaError_t e, const char* what) { return link::fail(&m->last_error, "fgb_metrics", e, what); };
  cudaError_t e = cudaSetDevice(m->device);
  if (e != cudaSuccess) return fail(e, "cudaSetDevice");
  uint64_t budget;
  if ((e = link::device_budget(m->opt.device_bytes, &budget)) != cudaSuccess) return fail(e, "cudaMemGetInfo");
  // staged runs of whole templates: the bytes plus ~100 bytes of tables per record
  std::vector<uint64_t> run_tpl{0};
  uint64_t max_t = 0, max_r = 0, max_bytes = 0;
  for (uint64_t t = 0; t < n_tpl;) {
    uint64_t v = t + 1;
    while (v < n_tpl) {
      const uint64_t recs = first[v + 1] - first[t], bytes = rec_off[first[v + 1]] - rec_off[first[t]];
      if (bytes + recs * 100 > budget || recs >= INT32_MAX / 2) break;
      ++v;
    }
    max_t = std::max(max_t, v - t);
    max_r = std::max(max_r, first[v] - first[t]);
    max_bytes = std::max(max_bytes, rec_off[first[v]] - rec_off[first[t]]);
    run_tpl.push_back(v);
    t = v;
  }
  link::Resources r(m->stream, m->opt.n_threads);
  uint8_t* d_rec;
  uint64_t* d_off;
  uint32_t* d_first;
  int32_t* d_prim;
  fgb_metrics_template* d_out;
  if ((e = r.alloc(&d_rec, max_bytes + 16)) || (e = r.alloc(&d_off, max_r + 1)) || (e = r.alloc(&d_first, max_t + 1)) ||
      (e = r.alloc(&d_prim, 2 * max_t)) || (e = r.alloc(&d_out, max_t)))
    return fail(e, "cudaMalloc");
  uint64_t stage = link::kStageBytes;
  if (const char* env = std::getenv("FGB_METRICS_STAGE_BYTES"))
    stage = std::max<uint64_t>(4096, std::min<uint64_t>(link::kStageBytes, std::strtoull(env, nullptr, 10)));
  const char* what;
  if ((e = r.open(std::min<uint64_t>(stage, std::max<uint64_t>(max_bytes + 64, (max_r + 1) * 8)), &what)))
    return fail(e, what);
  m->timing[3] += ms_since(t_host);
  std::vector<uint64_t> loff;
  std::vector<uint32_t> lfirst;
  std::vector<int32_t> lprim;
  std::vector<fgb_metrics_template> out;
  for (size_t x = 0; x + 1 < run_tpl.size(); ++x) {
    auto t_up = std::chrono::steady_clock::now();
    const uint64_t t0 = run_tpl[x], t1 = run_tpl[x + 1], rb = first[t0], nr = first[t1] - rb, nt = t1 - t0;
    const uint64_t base = rec_off[rb];
    loff.resize(nr + 1);
    for (uint64_t k = 0; k <= nr; ++k) loff[k] = rec_off[rb + k] - base;
    lfirst.resize(nt + 1);
    lprim.resize(2 * nt);
    for (uint64_t t = 0; t <= nt; ++t) lfirst[t] = static_cast<uint32_t>(first[t0 + t] - rb);
    for (uint64_t t = 0; t < 2 * nt; ++t)
      lprim[t] = prim[2 * t0 + t] < 0 ? -1 : static_cast<int32_t>(prim[2 * t0 + t] - static_cast<int64_t>(rb));
    if ((e = r.upload(d_rec, records + base, rec_off[rb + nr] - base)) || (e = r.upload(d_off, loff.data(), loff.size() * 8)) ||
        (e = r.upload(d_first, lfirst.data(), lfirst.size() * 4)) || (e = r.upload(d_prim, lprim.data(), lprim.size() * 4)))
      return fail(e, "upload");
    if ((e = mt::template_pass(d_rec, d_off, d_first, d_prim, static_cast<uint32_t>(nt), m->d_iv, d_out, m->stream)))
      return fail(e, "template pass");
    out.resize(nt);
    if ((e = r.download(out.data(), d_out, nt * sizeof(fgb_metrics_template)))) return fail(e, "download");
    m->stats[FGB_MSTAT_RUNS]++;
    m->timing[0] += ms_since(t_up);
    // the host's parts, in template order up to the first error
    t_host = std::chrono::steady_clock::now();
    uint64_t err_t = nt;
    for (uint64_t t = 0; t < nt; ++t) {
      fgb_metrics_template& tp = out[t];
      m->stats[FGB_MSTAT_TEMPLATES]++;
      if (tp.status >= FGB_MT_ERR_MI_MISSING) { err_t = t; break; }
      if (tp.status == FGB_MT_OUTSIDE) m->stats[FGB_MSTAT_OUTSIDE]++;
      if (tp.status != FGB_MT_KEPT) continue;
      m->stats[FGB_MSTAT_KEPT]++;
      const uint8_t* r1 = records + rec_off[rb + tp.r1];
      if (!tp.name_ascii) tp.bucket = static_cast<uint8_t>(mt::bucket_of(name_hash(r1 + 32, r1[8] ? r1[8] - 1u : 0u)));
      mt::FTpl f{tp.ref1, tp.start1, tp.ref2, tp.start2, tp.strand1, tp.strand2, tp.mi_kind, tp.bucket, 0, tp.mi_base};
      if (!tp.mi_canonical) {
        const uint32_t bl = tp.mi_len - (tp.mi_kind ? 2 : 0);
        const auto it = m->dict.emplace(std::string(reinterpret_cast<const char*>(r1 + tp.mi_off), bl), m->dict.size());
        f.base = kDictBit | it.first->second;
      }
      m->pend.push_back(f);
      m->pend_rec.push_back(g0 + first[t0 + t]);
      m->pend_kind.push_back(tp.mi_kind);
      m->pend_rx.append(reinterpret_cast<const char*>(r1 + tp.rx_off), tp.rx_len);
      m->pend_rx_off.push_back(m->pend_rx.size());
    }
    m->timing[3] += ms_since(t_host);
    uint64_t bt;
    const fgb_status st = count_closed(m, closed_count(*m), &bt);
    if (st != FGB_OK) return st;
    if (bt != UINT64_MAX) return umi_failure(m, bt, bad);
    if (err_t < nt) {
      const uint64_t rec = g0 + first[t0 + err_t];
      return fail_at(m, FGB_ERR_INVALID_ARG, rec, "fgb_metrics: record " + std::to_string(rec) + ": read '" +
                     std::string(fgb::grp::read_name(fgb::bam::View(records + rec_off[first[t0 + err_t]], 32 + records[rec_off[first[t0 + err_t]] + 8]))) +
                     "' " + status_text(out[err_t].status), bad);
    }
  }
  if (hb < n) return fail_at(m, hst, g0 + hb, "fgb_metrics: record " + std::to_string(g0 + hb) + " " + herr, bad);
  m->records_seen += n;
  m->stats[FGB_MSTAT_RECORDS] += n;
  return FGB_OK;
}

// ---- the tables (fgumi-metrics duplex.rs:323-472, simplex.rs:157-210, shared.rs:117-135; duplex_metrics.rs:392-503,
// simplex_metrics.rs:302-340) ------------------------------------------------------------------------------------
struct SizeRows {   // family_size_metrics rows 1..max of one fraction
  uint64_t max = 0;
  std::vector<uint64_t> cnt[3];
  uint64_t total[3] = {0, 0, 0};
};
SizeRows size_rows(const fgb_metrics& m, int f, int kinds) {
  SizeRows s;
  for (int k = 0; k < kinds; ++k) {
    if (!m.sizes[k][f].empty()) s.max = std::max(s.max, m.sizes[k][f].rbegin()->first);
    for (const auto& kv : m.sizes[k][f]) s.total[k] += kv.second;
  }
  for (int k = 0; k < kinds; ++k) {
    s.cnt[k].assign(s.max + 1, 0);
    for (const auto& kv : m.sizes[k][f]) s.cnt[k][kv.first] = kv.second;
  }
  return s;
}

void build_tables(fgb_metrics* m) {
  const bool duplex = m->opt.mode == FGB_METRICS_DUPLEX;
  const int kinds = duplex ? 3 : 2;
  const int last = kF - 1;
  {   // family sizes of the 100 % fraction; the >= columns summed from the largest size down
    const SizeRows s = size_rows(*m, last, kinds);
    Table t{duplex ? "family_size\tcs_count\tcs_fraction\tcs_fraction_gt_or_eq_size\tss_count\tss_fraction\t"
                     "ss_fraction_gt_or_eq_size\tds_count\tds_fraction\tds_fraction_gt_or_eq_size"
                   : "family_size\tcs_count\tcs_fraction\tcs_fraction_gt_or_eq_size\tss_count\tss_fraction\t"
                     "ss_fraction_gt_or_eq_size", ""};
    std::vector<double> fr[3], ge[3];
    for (int k = 0; k < kinds; ++k) {
      fr[k].assign(s.max + 2, 0.0);
      ge[k].assign(s.max + 2, 0.0);
      for (uint64_t z = 1; z <= s.max; ++z) fr[k][z] = frac(s.cnt[k][z], s.total[k]);
      for (uint64_t z = s.max; z >= 1; --z) ge[k][z] = fr[k][z] + (z < s.max ? ge[k][z + 1] : 0.0);
    }
    for (uint64_t z = 1; z <= s.max; ++z) {
      if (duplex)
        t.row({u(z), u(s.cnt[0][z]), fmt_f64(fr[0][z]), fmt_f64(ge[0][z]), u(s.cnt[1][z]), fmt_f64(fr[1][z]),
               fmt_f64(ge[1][z]), u(s.cnt[2][z]), fmt_f64(fr[2][z]), fmt_f64(ge[2][z])});
      else
        t.row({u(z), u(s.cnt[0][z]), fmt_f64(fr[0][z]), fmt_f64(ge[0][z]), u(s.cnt[1][z]), fmt_f64(fr[1][z]),
               fmt_f64(ge[1][z])});
    }
    m->tables[FGB_MTABLE_FAMILY_SIZES] = t.text;
    m->has_table[FGB_MTABLE_FAMILY_SIZES] = true;
  }
  if (duplex) {   // (ab, ba) of the 100 % fraction ascending; the 2-D >= count by a Fenwick tree over ba
    const auto& P = m->pairs[last];
    uint64_t total = 0, max_ba = 0;
    for (const auto& kv : P) { total += kv.second; max_ba = std::max(max_ba, kv.first.second); }
    std::vector<uint64_t> fen(max_ba + 2, 0);
    std::map<std::pair<uint64_t, uint64_t>, uint64_t> ge;
    for (auto it = P.rbegin(); it != P.rend();) {   // ab descending: add every pair of this ab, then query
      auto jt = it;
      for (; jt != P.rend() && jt->first.first == it->first.first; ++jt)
        for (uint64_t i = jt->first.second + 1; i <= max_ba + 1; i += i & (~i + 1)) fen[i] += jt->second;
      for (auto kt = it; kt != jt; ++kt) {
        uint64_t below = 0;   // pairs with ba < this ba
        for (uint64_t i = kt->first.second; i > 0; i -= i & (~i + 1)) below += fen[i];
        uint64_t all = 0;
        for (uint64_t i = max_ba + 1; i > 0; i -= i & (~i + 1)) all += fen[i];
        ge[kt->first] = all - below;
      }
      it = jt;
    }
    Table t{"ab_size\tba_size\tcount\tfraction\tfraction_gt_or_eq_size", ""};
    for (const auto& kv : P)
      t.row({u(kv.first.first), u(kv.first.second), u(kv.second), fmt_f64(frac(kv.second, total)),
             fmt_f64(frac(ge[kv.first], total))});
    m->tables[FGB_MTABLE_DUPLEX_FAMILY_SIZES] = t.text;
    m->has_table[FGB_MTABLE_DUPLEX_FAMILY_SIZES] = true;
  }
  {   // yield per fraction
    Table t{duplex ? "fraction\tread_pairs\tcs_families\tss_families\tds_families\tds_duplexes\tds_fraction_duplexes\t"
                     "ds_fraction_duplexes_ideal"
                   : "fraction\tread_pairs\tcs_families\tss_families\tmean_ss_family_size\tss_singletons\t"
                     "ss_singleton_fraction\tss_consensus_families", ""};
    const uint64_t min_ab = m->opt.min_ab_reads, min_ba = m->opt.min_ba_reads;
    std::map<uint64_t, double> prob;   // the ideal-duplex probability of a family size
    for (int f = 0; f < kF; ++f) {
      const SizeRows s = size_rows(*m, f, kinds);
      uint64_t cs = 0, ss = 0;
      for (uint64_t z = 1; z <= s.max; ++z) { cs += s.cnt[0][z]; ss += s.cnt[1][z]; }
      const std::string fs = fmt_f64(mt::fraction_at(f)), rp = u(m->templates[f]);
      if (duplex) {
        uint64_t ds = 0, dup = 0, ssd = 0, n_list = 0;
        for (uint64_t z = 1; z <= s.max; ++z) ds += s.cnt[2][z];
        for (const auto& kv : m->pairs[f]) {
          if (kv.first.first >= min_ab && kv.first.second >= min_ba) dup += kv.second;
          ssd += ((kv.first.first > 0) + (kv.first.second > 0)) * kv.second;
        }
        double ideal = 0.0;
        for (uint64_t z = 1; z <= s.max; ++z) {   // calculate_ideal_duplex_fraction over the expanded size list
          const uint64_t c = s.cnt[2][z];
          n_list += c;
          if (!c || z < min_ab + min_ba) continue;
          auto it = prob.find(z);
          if (it == prob.end()) {
            const uint64_t upper = z - min_ba, lower = min_ab;
            const double p = upper >= lower ? binom_interval_half(lower, upper, z) : 0.0;
            it = prob.emplace(z, p).first;
          }
          for (uint64_t i = 0; i < c; ++i) ideal += it->second;
        }
        ideal = n_list ? ideal / static_cast<double>(n_list) : 0.0;
        t.row({fs, rp, u(cs), u(ssd), u(ds), u(dup), fmt_f64(frac(dup, ds)), fmt_f64(ideal)});
      } else {
        uint64_t reads = 0, cons = 0;
        for (uint64_t z = 1; z <= s.max; ++z) {
          reads += z * s.cnt[1][z];
          if (z >= m->opt.min_reads) cons += s.cnt[1][z];
        }
        const uint64_t single = s.max >= 1 ? s.cnt[1][1] : 0;
        t.row({fs, rp, u(cs), u(ss), fmt_f64(frac(reads, ss)), u(single), fmt_f64(frac(single, ss)), u(cons)});
      }
    }
    m->tables[FGB_MTABLE_YIELD] = t.text;
    m->has_table[FGB_MTABLE_YIELD] = true;
  }
  std::map<std::string, double> single;
  {   // UMI counts by UMI
    uint64_t raw = 0, uniq = 0;
    for (const auto& kv : m->umi) { raw += kv.second.raw; uniq += kv.second.unique; }
    std::map<std::string, UmiCount> sorted(m->umi.begin(), m->umi.end());
    Table t{"umi\traw_observations\traw_observations_with_errors\tunique_observations\tfraction_raw_observations\t"
            "fraction_unique_observations", ""};
    for (const auto& kv : sorted) {
      t.row({field(kv.first), u(kv.second.raw), u(kv.second.err), u(kv.second.unique), fmt_f64(frac(kv.second.raw, raw)),
             fmt_f64(frac(kv.second.unique, uniq))});
      single[kv.first] = frac(kv.second.unique, uniq);
    }
    m->tables[FGB_MTABLE_UMI_COUNTS] = t.text;
    m->has_table[FGB_MTABLE_UMI_COUNTS] = true;
  }
  if (duplex && m->opt.duplex_umi_counts) {   // unique observations descending, ties by UMI (the reference's order of
    uint64_t raw = 0, uniq = 0;               // ties is its HashMap's)
    for (const auto& kv : m->dumi) { raw += kv.second.raw; uniq += kv.second.unique; }
    std::vector<std::pair<std::string, UmiCount>> v(m->dumi.begin(), m->dumi.end());
    std::sort(v.begin(), v.end(), [](const auto& a, const auto& b) {
      return a.second.unique != b.second.unique ? a.second.unique > b.second.unique : a.first < b.first;
    });
    Table t{"umi\traw_observations\traw_observations_with_errors\tunique_observations\tfraction_raw_observations\t"
            "fraction_unique_observations\tfraction_unique_observations_expected", ""};
    for (const auto& kv : v) {
      double expected = 0.0;
      const size_t d = kv.first.find('-');
      if (d != std::string::npos) {
        const auto a = single.find(kv.first.substr(0, d)), b = single.find(kv.first.substr(d + 1));
        expected = (a == single.end() ? 0.0 : a->second) * (b == single.end() ? 0.0 : b->second);
      }
      t.row({field(kv.first), u(kv.second.raw), u(kv.second.err), u(kv.second.unique), fmt_f64(frac(kv.second.raw, raw)),
             fmt_f64(frac(kv.second.unique, uniq)), fmt_f64(expected)});
    }
    m->tables[FGB_MTABLE_DUPLEX_UMI_COUNTS] = t.text;
    m->has_table[FGB_MTABLE_DUPLEX_UMI_COUNTS] = true;
  }
}

template <class F>
fgb_status guarded(fgb_metrics* m, F&& f) {
  try {
    return f();
  } catch (const std::bad_alloc&) {
    m->last_error = "fgb_metrics: out of host memory";
  } catch (const std::exception& x) {
    m->last_error = std::string("fgb_metrics: ") + x.what();
  }
  m->poisoned = true;
  return FGB_ERR_NOMEM;
}

}  // namespace

extern "C" {

fgb_status fgb_host_metrics_templates(const char* header_text, size_t header_len, const char* intervals,
                                      size_t intervals_len, const uint8_t* records, const uint64_t* rec_off,
                                      uint64_t n_records, fgb_metrics_template* out, uint64_t cap,
                                      uint64_t* n_templates, uint64_t* bad_record) {
  if (!n_templates || !rec_off || (n_records && !records) || (header_len && !header_text) ||
      (intervals_len && !intervals))
    return FGB_ERR_INVALID_ARG;
  try {
    std::vector<Interval> ivs;
    if (intervals && !parse_intervals(std::string_view(intervals, intervals_len), &ivs).empty())
      return FGB_ERR_INVALID_ARG;
    IvHost iv;
    build_iv(link::sq_names(std::string_view(header_text ? header_text : "", header_len)), ivs, &iv);
    std::vector<uint64_t> first;
    std::vector<int64_t> prim;
    std::string err;
    fgb_status st = FGB_OK;
    const uint64_t hb = templates_of(records, rec_off, n_records, &first, &prim, &err, &st);
    if (bad_record) *bad_record = hb < n_records ? hb : UINT64_MAX;
    if (hb < n_records) return st;
    const uint64_t nt = first.size() - 1;
    *n_templates = nt;
    if (cap < nt || (nt && !out)) return FGB_ERR_INVALID_ARG;
    const mt::IvTable table = iv.table();
    for (uint64_t t = 0; t < nt; ++t) {
      mt::template_pass([&](int64_t k) { return records + rec_off[k]; },
                        [&](int64_t k) { return rec_off[k + 1] - rec_off[k]; }, first[t + 1] - first[t], prim[2 * t],
                        prim[2 * t + 1], table, out + t);
      if (out[t].status == FGB_MT_KEPT || out[t].status == FGB_MT_OUTSIDE) {
        const uint8_t* r1 = records + rec_off[out[t].r1];
        if (!out[t].name_ascii) out[t].bucket = static_cast<uint8_t>(mt::bucket_of(name_hash(r1 + 32, r1[8] ? r1[8] - 1u : 0u)));
      }
    }
    return FGB_OK;
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
}

fgb_status fgb_host_metrics_name_fraction(const uint8_t* name, size_t len, int32_t* hash, double* fraction,
                                          uint32_t* bucket) {
  if ((len && !name) || !hash || !fraction || !bucket) return FGB_ERR_INVALID_ARG;
  *hash = name_hash(name, len);
  *fraction = mt::hash_fraction(*hash);
  *bucket = mt::bucket_of(*hash);
  return FGB_OK;
}

uint32_t fgb_host_metrics_bucket(int32_t hash) { return mt::bucket_of(hash); }

fgb_status fgb_host_metrics_intervals(const char* text, size_t len, uint64_t* name_off, uint64_t* name_len,
                                      int64_t* start, int64_t* end, uint64_t cap, uint64_t* n) {
  if ((len && !text) || !n) return FGB_ERR_INVALID_ARG;
  std::vector<Interval> ivs;
  if (!parse_intervals(std::string_view(text ? text : "", len), &ivs).empty()) return FGB_ERR_INVALID_ARG;
  *n = ivs.size();
  if (cap < ivs.size()) return FGB_OK;
  // the names' offsets: each name is the first field of a line of `text`; find them again in order
  size_t p = 0;
  for (size_t i = 0; i < ivs.size(); ++i) {
    const size_t at = std::string_view(text, len).find(ivs[i].name, p);
    name_off[i] = at;
    name_len[i] = ivs[i].name.size();
    start[i] = ivs[i].start;
    end[i] = ivs[i].end;
    p = at + ivs[i].name.size();
  }
  return FGB_OK;
}

size_t fgb_host_metrics_format_float(double v, char* buf, size_t cap) {
  const std::string s = fmt_f64(v);
  if (buf && cap) {
    const size_t k = std::min(cap - 1, s.size());
    std::memcpy(buf, s.data(), k);
    buf[k] = 0;
  }
  return s.size();
}

fgb_status fgb_metrics_create(int device, const fgb_metrics_options* opt, const char* header_text, size_t header_len,
                              const char* intervals, size_t intervals_len, fgb_metrics** out) {
  if (!opt || !out || (header_len && !header_text) || (intervals_len && !intervals)) return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  if (opt->mode > FGB_METRICS_DUPLEX) return FGB_ERR_INVALID_ARG;
  if (opt->mode == FGB_METRICS_DUPLEX && opt->min_ab_reads < opt->min_ba_reads) return FGB_ERR_INVALID_ARG;   // :131-137
  try {
    std::unique_ptr<fgb_metrics> m(new fgb_metrics());
    m->opt = *opt;
    m->sq = link::sq_names(std::string_view(header_text ? header_text : "", header_len));
    std::vector<Interval> ivs;
    if (intervals && !parse_intervals(std::string_view(intervals, intervals_len), &ivs).empty())
      return FGB_ERR_INVALID_ARG;
    build_iv(m->sq, ivs, &m->iv);
    if (device != FGB_DEVICE_NONE) {
      int n_dev = 0;
      if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) {
        cudaGetLastError();
        return FGB_ERR_NO_DEVICE;
      }
      m->device = device;
      const size_t nb = m->iv.sq_begin.size() * 4, ns = std::max<size_t>(m->iv.start.size(), 1) * 8;
      cudaError_t e;
      char* d = nullptr;
      if ((e = cudaSetDevice(device)) || (e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking)) ||
          (e = cudaDeviceGetAttribute(&m->sm_count, cudaDevAttrMultiProcessorCount, device)) ||
          (e = cudaMalloc(&m->d_iv_mem, nb + 2 * ns + 16)))
        { cudaGetLastError(); return e == cudaErrorMemoryAllocation ? FGB_ERR_NOMEM : FGB_ERR_CUDA; }
      d = static_cast<char*>(m->d_iv_mem);
      const size_t o_s = (nb + 7) / 8 * 8;
      if ((e = cudaMemcpy(d, m->iv.sq_begin.data(), nb, cudaMemcpyHostToDevice)) ||
          (!m->iv.start.empty() && (e = cudaMemcpy(d + o_s, m->iv.start.data(), m->iv.start.size() * 8, cudaMemcpyHostToDevice))) ||
          (!m->iv.maxend.empty() && (e = cudaMemcpy(d + o_s + ns, m->iv.maxend.data(), m->iv.maxend.size() * 8, cudaMemcpyHostToDevice))))
        { cudaGetLastError(); return FGB_ERR_CUDA; }
      m->d_iv = mt::IvTable{reinterpret_cast<const uint32_t*>(d), reinterpret_cast<const int64_t*>(d + o_s),
                            reinterpret_cast<const int64_t*>(d + o_s + ns), static_cast<uint32_t>(m->sq.size()),
                            m->iv.active};
    }
    *out = m.release();
    return FGB_OK;
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
}

void fgb_metrics_destroy(fgb_metrics* m) { delete m; }

size_t fgb_metrics_last_error(const fgb_metrics* m, char* buf, size_t buf_len) {
  if (!m) return 0;
  if (buf && buf_len) {
    const size_t n = std::min(buf_len - 1, m->last_error.size());
    std::memcpy(buf, m->last_error.data(), n);
    buf[n] = 0;
  }
  return m->last_error.size();
}

fgb_status fgb_metrics_add_records(fgb_metrics* m, const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                   uint64_t* bad_record) {
  if (bad_record) *bad_record = UINT64_MAX;
  if (!m || !rec_off || (n_records && !records)) return FGB_ERR_INVALID_ARG;
  if (m->device < 0) { m->last_error = "fgb_metrics: a planning-only collector has no device"; return FGB_ERR_NO_DEVICE; }
  if (m->poisoned || m->finished) {
    m->last_error = m->finished ? "fgb_metrics: the collector is finished" : "fgb_metrics: an earlier call failed";
    return FGB_ERR_INVALID_ARG;
  }
  if (!n_records) return FGB_OK;
  return guarded(m, [&] { return add_impl(m, records, rec_off, n_records, bad_record); });
}

fgb_status fgb_metrics_finish(fgb_metrics* m, uint64_t* bad_record) {
  if (bad_record) *bad_record = UINT64_MAX;
  if (!m) return FGB_ERR_INVALID_ARG;
  if (m->device < 0) { m->last_error = "fgb_metrics: a planning-only collector has no device"; return FGB_ERR_NO_DEVICE; }
  if (m->poisoned || m->finished) {
    m->last_error = m->finished ? "fgb_metrics: the collector is finished" : "fgb_metrics: an earlier call failed";
    return FGB_ERR_INVALID_ARG;
  }
  return guarded(m, [&]() -> fgb_status {
    cudaError_t e = cudaSetDevice(m->device);
    if (e != cudaSuccess) return link::fail(&m->last_error, "fgb_metrics", e, "cudaSetDevice");
    uint64_t bt;
    const fgb_status st = count_closed(m, m->pend.size(), &bt);
    if (st != FGB_OK) return st;
    if (bt != UINT64_MAX) return umi_failure(m, bt, bad_record);
    auto t0 = std::chrono::steady_clock::now();
    build_tables(m);
    m->timing[3] += ms_since(t0);
    m->finished = true;
    return FGB_OK;
  });
}

fgb_status fgb_metrics_table(const fgb_metrics* m, uint32_t which, const char** text, uint64_t* len) {
  if (!m || !text || !len || which > FGB_MTABLE_DUPLEX_UMI_COUNTS || !m->finished || !m->has_table[which])
    return FGB_ERR_INVALID_ARG;
  *text = m->tables[which].data();
  *len = m->tables[which].size();
  return FGB_OK;
}

fgb_status fgb_metrics_stats(const fgb_metrics* m, uint64_t stats[FGB_METRICS_NSTATS]) {
  if (!m || !stats) return FGB_ERR_INVALID_ARG;
  std::memcpy(stats, m->stats, sizeof(m->stats));
  return FGB_OK;
}

fgb_status fgb_metrics_last_timing(const fgb_metrics* m, double ms[4]) {
  if (!m || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, m->timing, sizeof(m->timing));
  return FGB_OK;
}

}  // extern "C"
