// Host half of UMI assignment: see umi_host.h.  Every rule cites the reference as oracle/umi_oracle.py does.
#include "umi_host.h"

#include <algorithm>
#include <cstring>
#include <deque>
#include <numeric>
#include <unordered_map>

namespace fgb_umi {
namespace {

constexpr uint32_t kNoKey = UINT32_MAX;

inline uint8_t up(uint8_t b) { return (b >= 'a' && b <= 'z') ? static_cast<uint8_t>(b - 32) : b; }

std::string upper(std::string_view s) {   // ASCII only (the reference uses Unicode to_uppercase)
  std::string r(s);
  for (auto& ch : r) ch = static_cast<char>(up(static_cast<uint8_t>(ch)));
  return r;
}

// bitenc.rs:69-90 from_umi_str: ACGT in either case, '-' skipped, anything else or more than 32 bases -> None
bool bitenc(std::string_view s, uint64_t* bits, uint8_t* len) {
  uint64_t b = 0;
  uint32_t n = 0;
  for (char ch : s) {
    int c;
    switch (ch) {
      case 'A': case 'a': c = 0; break;
      case 'C': case 'c': c = 1; break;
      case 'G': case 'g': c = 2; break;
      case 'T': case 't': c = 3; break;
      case '-': continue;
      default: return false;
    }
    if (n >= 32) return false;
    b |= static_cast<uint64_t>(c) << (2 * n);
    ++n;
  }
  *bits = b;
  *len = static_cast<uint8_t>(n);
  return true;
}

// split('-').count() == 2 (assigner.rs:1794, parallel_assigner.rs:632)
bool dash_of(std::string_view s, uint32_t* pos) {
  const size_t p = s.find('-');
  if (p == std::string_view::npos || s.find('-', p + 1) != std::string_view::npos) return false;
  *pos = static_cast<uint32_t>(p);
  return true;
}

std::string reverse_paired(std::string_view s, uint32_t dash) {   // assigner.rs:1695-1703
  std::string r;
  r.reserve(s.size());
  r.append(s.substr(dash + 1)).push_back('-');
  r.append(s.substr(0, dash));
  return r;
}

uint64_t count_mismatches(std::string_view a, std::string_view b) {   // assigner.rs:644-649
  if (a.size() != b.size()) return UINT64_MAX;
  uint64_t n = 0;
  for (size_t i = 0; i < a.size(); ++i) n += a[i] != b[i];
  return n;
}

std::string enc_id(uint64_t bits, uint8_t len) {
  std::string s(9, '\0');
  std::memcpy(&s[0], &bits, 8);
  s[8] = static_cast<char>(len);
  return s;
}

}  // namespace

std::string check_options(const fgb_umi_options& o) {
  if (o.strategy > FGB_UMI_PAIRED) return "unknown strategy";
  if (o.rules > FGB_UMI_RULES_UNMAPPED) return "unknown rules";
  if (o.strategy == FGB_UMI_IDENTITY && o.edits != 0)
    return "edits must be 0 with the identity strategy";   // assigner.rs:605
  if (o.edits > 32) return "edits above 32";
  return "";
}

bool uses_bytes(const fgb_umi_options& o) {
  return o.rules == FGB_UMI_RULES_MAPPED && (o.strategy == FGB_UMI_EDIT || o.strategy == FGB_UMI_PAIRED);
}

bool needs_edges(const fgb_umi_options& o, const Call& c) {
  return o.strategy != FGB_UMI_IDENTITY && c.keys.size() >= 2;
}

std::string prepare(const fgb_umi_options& o, const uint8_t* umis, const uint64_t* off, uint64_t n, Call* c) {
  c->umis.clear(); c->keys.clear(); c->bytes.clear(); c->key_of.assign(n, kNoKey);
  c->umis.reserve(n);
  for (uint64_t i = 0; i < n; ++i)
    c->umis.emplace_back(reinterpret_cast<const char*>(umis) + off[i], off[i + 1] - off[i]);
  if (o.min_umi_length && n) {   // truncate_umis, group.rs:353-364
    size_t m = SIZE_MAX;
    for (auto& u : c->umis) m = std::min(m, u.size());
    if (m < o.min_umi_length)
      return "UMI found that had shorter length than expected (" + std::to_string(m) + " < " +
             std::to_string(o.min_umi_length) + ")";
    for (auto& u : c->umis) u = u.substr(0, o.min_umi_length);
  }
  const bool mapped = o.rules == FGB_UMI_RULES_MAPPED;
  if (o.strategy == FGB_UMI_PAIRED) {
    uint32_t d;
    for (auto& u : c->umis)
      if (!dash_of(u, &d)) return "UMI " + std::string(u) + " is not a paired UMI";
  }
  // Per UMI: the identity of its key (`id`) and the key's string (`disp`, the first occurrence's).
  struct Uniq { std::string disp; uint64_t bits; uint32_t count, first; uint8_t len; };
  std::vector<Uniq> uq;
  std::unordered_map<std::string, uint32_t> index;
  index.reserve(n * 2);
  std::vector<uint32_t> uq_of(n, kNoKey);
  for (uint64_t i = 0; i < n; ++i) {
    std::string_view u = c->umis[i];
    std::string id, disp;
    uint64_t bits = 0;
    uint8_t len = 0;
    bool valid = true;
    switch (o.strategy) {
      case FGB_UMI_IDENTITY: id = disp = upper(u); break;               // assigner.rs:863
      case FGB_UMI_EDIT:
        if (mapped) id = disp = std::string(u);                            // assigner.rs:946-950: raw strings
        else { disp = upper(u); valid = bitenc(disp, &bits, &len); id = enc_id(bits, len); }   // parallel :362-371
        break;
      case FGB_UMI_ADJACENCY:
        if (mapped) { valid = bitenc(u, &bits, &len); id = enc_id(bits, len); disp = std::string(u); }  // :1452-1465
        else { id = disp = upper(u); valid = bitenc(id, &bits, &len); }  // parallel :460-473
        break;
      default: {                                                           // paired
        uint32_t d = 0;
        dash_of(u, &d);
        if (mapped) {   // assigner.rs:1721-1736: the parts are compared
          id = u.substr(0, d) <= u.substr(d + 1) ? std::string(u) : reverse_paired(u, d);
        } else {        // parallel_assigner.rs:609-616: the whole upper-case strings are compared
          std::string uu = upper(u), r = reverse_paired(uu, d);
          id = r < uu ? r : uu;
          valid = bitenc(id, &bits, &len);
        }
        if (mapped) bitenc(id, &bits, &len);
        disp = id;
      }
    }
    if (!valid) continue;
    auto it = index.find(id);
    if (it == index.end()) {
      const uint32_t k = static_cast<uint32_t>(uq.size());
      index.emplace(id, k);
      uq.push_back(Uniq{std::move(disp), bits, 1, static_cast<uint32_t>(i), len});
      uq_of[i] = k;
    } else {
      uq[it->second].count++;
      uq_of[i] = it->second;
    }
  }
  std::vector<uint32_t> order(uq.size());
  std::iota(order.begin(), order.end(), 0u);
  if (o.strategy == FGB_UMI_IDENTITY || (o.strategy == FGB_UMI_EDIT && mapped)) {
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return uq[a].disp < uq[b].disp; });
  } else if (o.strategy != FGB_UMI_EDIT) {   // count descending, then string (assigner.rs:1479, 1799)
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
      return uq[a].count != uq[b].count ? uq[a].count > uq[b].count : uq[a].disp < uq[b].disp;
    });
  }   // unmapped edit: first appearance
  std::vector<uint32_t> rank(uq.size());
  c->keys.resize(uq.size());
  std::unordered_map<std::string, uint32_t> last;
  for (uint32_t r = 0; r < order.size(); ++r) {
    const Uniq& q = uq[order[r]];
    rank[order[r]] = r;
    fgb_umi_key& k = c->keys[r];
    std::memset(&k, 0, sizeof(k));
    k.bits = q.bits; k.len = q.len; k.count = q.count; k.first = q.first;
    k.str_off = c->bytes.size();
    k.str_len = static_cast<uint32_t>(q.disp.size());
    c->bytes.insert(c->bytes.end(), q.disp.begin(), q.disp.end());
    if (o.strategy == FGB_UMI_PAIRED) dash_of(q.disp, &k.dash);
    k.flags = FGB_UMI_KEY_LAST;
    if (!mapped && (o.strategy == FGB_UMI_ADJACENCY || o.strategy == FGB_UMI_PAIRED)) last[enc_id(q.bits, q.len)] = r;   // last index wins
  }
  if (!last.empty())
    for (uint32_t r = 0; r < c->keys.size(); ++r)
      if (last[enc_id(c->keys[r].bits, c->keys[r].len)] != r) c->keys[r].flags = 0;
  for (uint64_t i = 0; i < n; ++i)
    if (uq_of[i] != kNoKey) c->key_of[i] = rank[uq_of[i]];
  if (o.strategy == FGB_UMI_ADJACENCY && mapped && c->keys.size() > 1)   // assigner.rs:1494-1502 asserts
    for (auto& k : c->keys)
      if (k.len != c->keys[0].len)
        return "Multiple UMI lengths: " + std::to_string(k.len) + " vs " + std::to_string(c->keys[0].len);
  return "";
}

namespace {

// BFS from roots in sorted order over the capture lists: a child joins when it is unassigned
// (assigner.rs:1182-1258, parallel_assigner.rs:506-539; the count rule is already in the lists).
uint64_t bfs(const Call& c, const uint64_t* eo, const uint32_t* e, std::vector<int64_t>* comp,
             std::vector<uint32_t>* roots) {
  const size_t n = c.keys.size();
  comp->assign(n, -1);
  roots->clear();
  std::vector<uint32_t> q;
  for (uint32_t r = 0; r < n; ++r) {
    if ((*comp)[r] >= 0) continue;
    const int64_t id = static_cast<int64_t>(roots->size());
    roots->push_back(r);
    (*comp)[r] = id;
    q.assign(1, r);
    for (size_t h = 0; h < q.size(); ++h)
      for (uint64_t x = eo[q[h]]; x < eo[q[h] + 1]; ++x)
        if ((*comp)[e[x]] < 0) { (*comp)[e[x]] = id; q.push_back(e[x]); }
  }
  return roots->size();
}

std::vector<uint32_t> components(const Call& c, const uint64_t* eo, const uint32_t* e) {
  std::vector<uint32_t> p(c.keys.size());
  std::iota(p.begin(), p.end(), 0u);
  auto find = [&](uint32_t x) {
    while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; }
    return x;
  };
  if (eo)
    for (uint32_t i = 0; i < p.size(); ++i)
      for (uint64_t x = eo[i]; x < eo[i + 1]; ++x) {
        const uint32_t a = find(i), b = find(e[x]);
        if (a != b) p[std::max(a, b)] = std::min(a, b);
      }
  for (uint32_t i = 0; i < p.size(); ++i) p[i] = find(i);
  return p;
}

std::string_view key_str(const Call& c, uint32_t k) {
  return std::string_view(reinterpret_cast<const char*>(c.bytes.data()) + c.keys[k].str_off, c.keys[k].str_len);
}

}  // namespace

void resolve(const fgb_umi_options& o, const Call& c, const uint64_t* eo, const uint32_t* e, uint64_t* ids,
             uint8_t* kinds) {
  const uint64_t n = c.umis.size();
  if (!n) return;
  const bool mapped = o.rules == FGB_UMI_RULES_MAPPED;
  const uint64_t nk = c.keys.size();
  auto set = [&](uint64_t i, uint8_t kind, uint64_t id) { kinds[i] = kind; ids[i] = kind == FGB_MOL_NONE ? 0 : id; };
  if (o.strategy == FGB_UMI_IDENTITY) {   // ids in the byte order of the unique keys
    for (uint64_t i = 0; i < n; ++i) set(i, FGB_MOL_SINGLE, c.key_of[i]);
    return;
  }
  if (!mapped && nk == 0) {   // no valid key: input i gets Single(i) (parallel_assigner.rs:374-377, 476-479, 652-654)
    for (uint64_t i = 0; i < n; ++i) set(i, FGB_MOL_SINGLE, i);
    return;
  }
  const uint64_t* eo1 = nk >= 2 ? eo : nullptr;
  std::vector<uint64_t> no_edges(nk + 1, 0);
  if (!eo1) { eo = no_edges.data(); e = nullptr; }
  if (o.strategy == FGB_UMI_EDIT) {
    const std::vector<uint32_t> root = components(c, eo1, e);
    std::vector<int64_t> num(nk, -1);
    uint64_t next = 0;
    if (mapped) {   // components numbered by their smallest string (assigner.rs:990-1004); keys are sorted
      for (uint64_t k = 0; k < nk; ++k)
        if (num[root[k]] < 0) num[root[k]] = static_cast<int64_t>(next++);
      for (uint64_t i = 0; i < n; ++i) set(i, FGB_MOL_SINGLE, num[root[c.key_of[i]]]);
    } else {        // first appearance; every invalid occurrence a fresh id (parallel_assigner.rs:394-417)
      for (uint64_t i = 0; i < n; ++i) {
        if (c.key_of[i] == kNoKey) { set(i, FGB_MOL_SINGLE, next++); continue; }
        const uint32_t r = root[c.key_of[i]];
        if (num[r] < 0) num[r] = static_cast<int64_t>(next++);
        set(i, FGB_MOL_SINGLE, num[r]);
      }
    }
    return;
  }
  if (o.strategy == FGB_UMI_ADJACENCY) {
    if (mapped && nk == 0) { for (uint64_t i = 0; i < n; ++i) set(i, FGB_MOL_NONE, 0); return; }   // :1471-1473
    if (mapped && nk == 1) { for (uint64_t i = 0; i < n; ++i) set(i, FGB_MOL_SINGLE, 0); return; }  // :1488-1491
    std::vector<int64_t> comp;
    std::vector<uint32_t> roots;
    uint64_t next = bfs(c, eo, e, &comp, &roots);
    for (uint64_t i = 0; i < n; ++i) {
      if (c.key_of[i] != kNoKey) set(i, FGB_MOL_SINGLE, comp[c.key_of[i]]);
      else if (mapped) set(i, FGB_MOL_NONE, 0);            // :1522
      else set(i, FGB_MOL_SINGLE, next++);                  // parallel_assigner.rs:554-559
    }
    return;
  }
  // paired
  if (mapped && nk == 1) {   // assigner.rs:1801-1814: A iff umi < reverse(umi)
    for (uint64_t i = 0; i < n; ++i) {
      uint32_t d = 0;
      dash_of(c.umis[i], &d);
      set(i, c.umis[i] < std::string_view(reverse_paired(c.umis[i], d)) ? FGB_MOL_A : FGB_MOL_B, 0);
    }
    return;
  }
  std::vector<int64_t> comp;
  std::vector<uint32_t> roots;
  bfs(c, eo, e, &comp, &roots);
  if (!mapped) {   // parallel_assigner.rs:721-737: A iff the upper-cased UMI is the canonical form
    for (uint64_t i = 0; i < n; ++i) {
      if (c.key_of[i] == kNoKey) { set(i, FGB_MOL_NONE, 0); continue; }
      const bool a = upper(c.umis[i]) == key_str(c, c.key_of[i]);
      set(i, a ? FGB_MOL_A : FGB_MOL_B, comp[c.key_of[i]]);
    }
    return;
  }
  // assigner.rs:1821-1857: per key the kind of the key string and of its reverse; a palindromic X-X key's
  // second insert overwrites the first.
  std::vector<uint8_t> kind_key(nk), kind_rev(nk);
  std::vector<uint8_t> is_root(nk, 0);
  for (uint32_t r : roots) { is_root[r] = 1; kind_key[r] = FGB_MOL_A; kind_rev[r] = FGB_MOL_B; }
  for (uint32_t k = 0; k < nk; ++k) {
    if (is_root[k]) continue;
    std::string_view rs = key_str(c, roots[comp[k]]), cs = key_str(c, k);
    const std::string crev = reverse_paired(cs, c.keys[k].dash);
    const bool a = count_mismatches(rs, cs) < count_mismatches(rs, crev);
    kind_key[k] = a ? FGB_MOL_A : FGB_MOL_B;
    kind_rev[k] = a ? FGB_MOL_B : FGB_MOL_A;
  }
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t k = c.key_of[i];
    std::string_view ks = key_str(c, k);
    const std::string krev = reverse_paired(ks, c.keys[k].dash);
    const uint8_t kind = (c.umis[i] == std::string_view(krev)) ? kind_rev[k] : kind_key[k];   // rev inserted last
    set(i, kind, comp[k]);
  }
}

}  // namespace fgb_umi

extern "C" {

fgb_status fgb_host_umi_for_read(const fgb_umi_options* opt, const uint8_t* umi, size_t len, int is_r1_earlier,
                                 uint8_t* out, size_t cap, size_t* out_len) {
  if (!opt || (!umi && len) || !out_len || !fgb_umi::check_options(*opt).empty()) return FGB_ERR_INVALID_ARG;
  std::string_view u(reinterpret_cast<const char*>(umi), len);
  std::string r;
  if (opt->strategy != FGB_UMI_PAIRED) {
    r = fgb_umi::upper(u);                                 // group.rs:301-308
  } else {
    uint32_t d;
    if (!fgb_umi::dash_of(u, &d)) return FGB_ERR_INVALID_ARG;   // :311-317
    if (opt->rules == FGB_UMI_RULES_UNMAPPED) {
      r = fgb_umi::upper(u);                               // :320-322
    } else {                                               // :330-346, prefixes of edits + 1 characters
      const std::string lo(opt->edits + 1, 'a'), hi(opt->edits + 1, 'b');
      const std::string& p0 = is_r1_earlier ? lo : hi;
      const std::string& p1 = is_r1_earlier ? hi : lo;
      r = p0 + ":" + std::string(u.substr(0, d)) + "-" + p1 + ":" + std::string(u.substr(d + 1));
    }
  }
  *out_len = r.size();
  if (r.size() > cap || (!out && r.size())) return FGB_ERR_INVALID_ARG;
  if (!r.empty()) std::memcpy(out, r.data(), r.size());
  return FGB_OK;
}

fgb_status fgb_host_umi_prepare(const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                                uint64_t n_umis, fgb_umi_key* keys, uint64_t* n_keys, uint8_t* key_bytes,
                                uint32_t* key_of) {
  if (!opt || !umi_off || !n_keys || (n_umis && (!umis || !keys || !key_of)) ||
      !fgb_umi::check_options(*opt).empty())
    return FGB_ERR_INVALID_ARG;
  for (uint64_t i = 0; i < n_umis; ++i) if (umi_off[i + 1] < umi_off[i]) return FGB_ERR_INVALID_ARG;
  fgb_umi::Call c;
  try {
    if (!fgb_umi::prepare(*opt, umis, umi_off, n_umis, &c).empty()) return FGB_ERR_INVALID_ARG;
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
  *n_keys = c.keys.size();
  if (!c.keys.empty()) std::memcpy(keys, c.keys.data(), c.keys.size() * sizeof(fgb_umi_key));
  if (!c.bytes.empty()) std::memcpy(key_bytes, c.bytes.data(), c.bytes.size());
  if (n_umis) std::memcpy(key_of, c.key_of.data(), n_umis * sizeof(uint32_t));
  return FGB_OK;
}

fgb_status fgb_host_umi_resolve(const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                                uint64_t n_umis, const fgb_umi_key* keys, uint64_t n_keys, const uint8_t* key_bytes,
                                const uint32_t* key_of, const uint64_t* edge_off, const uint32_t* edges,
                                uint64_t* ids, uint8_t* kinds) {
  if (!opt || !umi_off || (n_umis && (!umis || !key_of || !ids || !kinds)) || (n_keys && !keys) ||
      !fgb_umi::check_options(*opt).empty())
    return FGB_ERR_INVALID_ARG;
  fgb_umi::Call c;
  try {
    // The views (truncation included) come from prepare; the table itself is the caller's.
    if (!fgb_umi::prepare(*opt, umis, umi_off, n_umis, &c).empty()) return FGB_ERR_INVALID_ARG;
    c.keys.assign(keys, keys + n_keys);
    uint64_t nb = 0;
    for (uint64_t k = 0; k < n_keys; ++k) nb = std::max<uint64_t>(nb, keys[k].str_off + keys[k].str_len);
    c.bytes.assign(key_bytes, key_bytes + nb);
    c.key_of.assign(key_of, key_of + n_umis);
    for (uint64_t i = 0; i < n_umis; ++i) if (key_of[i] != UINT32_MAX && key_of[i] >= n_keys) return FGB_ERR_INVALID_ARG;
    if (n_keys >= 2 && fgb_umi::needs_edges(*opt, c)) {
      if (!edge_off || edge_off[0] != 0) return FGB_ERR_INVALID_ARG;
      for (uint64_t k = 0; k < n_keys; ++k) {
        if (edge_off[k + 1] < edge_off[k]) return FGB_ERR_INVALID_ARG;
        for (uint64_t x = edge_off[k]; x < edge_off[k + 1]; ++x) if (edges[x] >= n_keys) return FGB_ERR_INVALID_ARG;
      }
    }
    fgb_umi::resolve(*opt, c, edge_off, edges, ids, kinds);
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
  return FGB_OK;
}

}  // extern "C"
