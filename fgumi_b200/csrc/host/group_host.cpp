// `fgumi group` around the UMI assignment: position grouping of the input stream (fgb_host_group_by_position) and
// the record-level grouper (fgb_grouper_*): templates, filter, orientation split and UMIs before fgb_umi_assign,
// MI tags, order, histograms and the MI counter after it.  Restated in oracle/group_oracle.py, which cites the
// reference (fgumi 0.2.0) line by line; the citations here are the same.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <map>
#include <memory>
#include <new>
#include <numeric>
#include <string>
#include <string_view>
#include <tuple>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "bam.h"
#include "group_rules.h"
#include "record_link.h"
#include "umi_host.h"

namespace {

using fgb::bam::View;
namespace bam = fgb::bam;
using namespace fgb::grp;
using fgb::link::guarded;

// ---- position grouping (unified_pipeline/bam.rs:415-499, base.rs:1375-1436, grouper.rs:406-588) ----------------
struct PosKey {
  int32_t ref1, pos1, ref2, pos2;
  uint8_t strand1, strand2;
  uint16_t library;
  bool has_cell;
  std::string cell;   // the reference compares a hash of the bytes; equal bytes <=> equal hash barring collisions
  bool operator==(const PosKey& o) const {
    return ref1 == o.ref1 && pos1 == o.pos1 && strand1 == o.strand1 && ref2 == o.ref2 && pos2 == o.pos2 &&
           strand2 == o.strand2 && library == o.library && has_cell == o.has_cell && cell == o.cell;
  }
};

// LibraryIndex::from_header (read_info.rs:104-131): libraries numbered from 1 in order of first appearance over the
// @RG lines, an RG without LB is library "unknown" = 0, as is an RG the header does not declare.
std::map<std::string, uint16_t> library_index(std::string_view text) {
  std::map<std::string, uint16_t> lib_of_name{{"unknown", 0}}, lib_of_rg;
  bam::for_each_read_group(text, [&](std::string_view id, std::string_view lb, bool has_lb) {
    const std::string name = has_lb ? std::string(lb) : "unknown";
    auto it = lib_of_name.find(name);
    if (it == lib_of_name.end()) it = lib_of_name.emplace(name, static_cast<uint16_t>(lib_of_name.size())).first;
    lib_of_rg[std::string(id)] = it->second;
  });
  return lib_of_rg;
}

}  // namespace

// ---- the grouper -------------------------------------------------------------------------------------------------
namespace {

struct Tpl {                    // one template's primary reads in its group's byte copy (kNone: absent)
  uint64_t r1 = kNone, r1_len = 0, r2 = kNone, r2_len = 0;
  uint64_t name = 0, name_len = 0;
};

struct GroupPrep {              // one position group after the host rules in front of the assignment
  std::vector<uint8_t> bytes;
  std::vector<Tpl> tpls;        // templates that passed the filter, in input order
  Calls c;                      // the calls and their UMIs
  uint64_t filter[6] = {0, 0, 0, 0, 0, 0};
  bool dropped = false;         // the reference's assignment returns an error: nothing but the filter counts
};

enum { F_TOTAL, F_ACCEPTED, F_NON_PF, F_POOR, F_NS, F_SHORT };

}  // namespace

struct fgb_grouper {
  fgb_group_options opt{};
  fgb_umi_options umi{};        // what goes to fgb_umi_assign (no_umi: identity, 0 edits)
  fgb_handle* h = nullptr;
  std::vector<GroupPrep> queue;
  uint64_t stats[FGB_GROUP_NSTATS] = {};
  std::map<uint64_t, uint64_t> family_sizes, group_sizes;
  std::string last_error;
  UmiBatch batch;               // the queue's UMI batch (fgb_grouper_pending)
  std::vector<uint8_t> out;
  double timing[5] = {0, 0, 0, 0, 0};   // fgb_grouper_last_timing
};

namespace {

// filter_template_raw (group.rs:113-262): counts are per primary READ of the template
bool filter_template(const fgb_grouper& g, const View* r1, const View* r2, uint64_t* fc) {
  const uint64_t n = (r1 != nullptr) + (r2 != nullptr);
  fc[F_TOTAL] += n;
  if (!r1 && !r2) { fc[F_POOR] += n; return false; }
  const bool both_unmapped = (!r1 || (r1->flags() & bam::kUnmapped)) && (!r2 || (r2->flags() & bam::kUnmapped));
  if (both_unmapped && g.opt.umi.rules != FGB_UMI_RULES_UNMAPPED) { fc[F_POOR] += n; return false; }
  const View* reads[2] = {r1, r2};
  for (const View* r : reads) {   // phase 1: flags and MAPQ
    if (!r) continue;
    const uint16_t f = r->flags();
    if (!g.opt.include_non_pf && (f & 0x200)) { fc[F_NON_PF] += n; return false; }
    if (!(f & bam::kUnmapped) && r->b[9] < g.opt.min_map_q) { fc[F_POOR] += n; return false; }
  }
  for (const View* r : reads) {   // phase 2: one aux walk for MQ and the UMI (:157-221)
    if (!r) continue;
    const bool check_mq = !(r->flags() & bam::kMateUnmapped), check_umi = !g.opt.no_umi;
    const MqUmi s = scan_mq_umi(*r, check_mq, check_umi, g.opt.umi_tag);
    if (check_mq && s.have_mq && static_cast<uint8_t>(s.mq) < g.opt.min_map_q) { fc[F_POOR] += n; return false; }   // `as u8`
    if (g.opt.no_umi) continue;
    if (!s.have_umi) { fc[F_POOR] += n; return false; }
    const int64_t bases = umi_bases(s.umi, s.umi_len);
    if (bases < 0) { fc[F_NS] += n; return false; }
    if (g.opt.umi.min_umi_length && static_cast<uint64_t>(bases) < g.opt.umi.min_umi_length) { fc[F_SHORT] += n; return false; }
  }
  fc[F_ACCEPTED] += n;
  return true;
}

// One position group: templates, filter, split, UMIs.  "" or the message of an error that fails the whole call.
std::string prepare_group(const fgb_grouper& g, const uint8_t* records, const uint64_t* rec_off, uint64_t b,
                          uint64_t e, GroupPrep* gp) {
  // build_templates_from_records (grouper.rs:596-651) + Template::from_records (template.rs:159-273)
  std::vector<View> views;
  views.reserve(e - b);
  for (uint64_t i = b; i < e; ++i) views.emplace_back(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
  const uint64_t n = e - b;
  std::vector<uint64_t> lists[4], order;
  for (uint64_t i = 0; i < n;) {
    uint64_t j = i + 1;
    const std::string_view name = read_name(views[i]);
    while (j < n && read_name(views[j]) == name) ++j;
    int64_t r1, r2;
    uint64_t dup;
    order.clear();
    const std::string err = template_order(i, j, [&](uint64_t k) { return views[k].flags(); }, name, lists, &order,
                                           &r1, &r2, &dup);
    if (!err.empty()) return err;
    const View* v1 = r1 >= 0 ? &views[r1] : nullptr;
    const View* v2 = r2 >= 0 ? &views[r2] : nullptr;
    if (filter_template(g, v1, v2, gp->filter)) {
      Tpl t;
      auto copy = [&](const View* v, uint64_t* off, uint64_t* len) {
        *off = gp->bytes.size();
        *len = v->n;
        gp->bytes.insert(gp->bytes.end(), v->b, v->b + v->n);
      };
      if (v1) copy(v1, &t.r1, &t.r1_len);
      if (v2) copy(v2, &t.r2, &t.r2_len);
      const uint64_t at = t.r1 != kNone ? t.r1 : t.r2;
      t.name = at + 32;
      t.name_len = name.size();
      gp->tpls.push_back(t);
    }
    i = j;
  }
  if (gp->tpls.empty()) return "";
  // the orientation split and each template's UMI; where the reference's assignment fails the group is dropped
  // (group.rs:1512-1522)
  auto view_of = [&](uint64_t off, uint64_t len) { return View(gp->bytes.data() + off, len); };
  std::vector<View> v1, v2;   // the copies' views (Tpl offsets), nullptr through the accessors when absent
  for (const Tpl& x : gp->tpls) {
    v1.push_back(view_of(x.r1 != kNone ? x.r1 : 0, x.r1_len));
    v2.push_back(view_of(x.r2 != kNone ? x.r2 : 0, x.r2_len));
  }
  if (!split_and_umis(g.umi, g.opt.no_umi, g.opt.umi_tag, gp->tpls.size(),
                      [&](size_t t) { return gp->tpls[t].r1 != kNone ? &v1[t] : nullptr; },
                      [&](size_t t) { return gp->tpls[t].r2 != kNone ? &v2[t] : nullptr; }, &gp->c).empty())
    gp->dropped = true;
  return "";
}

struct GroupOut {
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> families;   // template count of each molecule, in output order
  uint64_t n_records = 0;
};

// process_and_write_position_group after the assignment (group.rs:1524-1592, 1650-1682) for queued group `gp`;
// ids / kinds indexed like its batch entries (gp.c.order).
void emit_group(const fgb_grouper& g, const GroupPrep& gp, const uint64_t* ids, const uint8_t* kinds, uint64_t base_mi,
                GroupOut* go) {
  const size_t nt = gp.tpls.size();
  std::vector<uint64_t> tid(nt), vidx(nt);   // vidx: MoleculeId::to_vec_index + 1, 0 = None (sorts first)
  std::vector<uint8_t> tkind(nt);
  for (size_t u = 0; u < nt; ++u) {
    const uint32_t t = gp.c.order[u];
    tkind[t] = kinds[u];
    tid[t] = ids[u];
    vidx[t] = vec_index(kinds[u], ids[u]);
  }
  auto name = [&](size_t t) {
    return std::string_view(reinterpret_cast<const char*>(gp.bytes.data() + gp.tpls[t].name), gp.tpls[t].name_len);
  };
  std::vector<uint32_t> sorted(nt);
  std::iota(sorted.begin(), sorted.end(), 0u);
  std::stable_sort(sorted.begin(), sorted.end(), [&](uint32_t a, uint32_t b) {
    return vidx[a] != vidx[b] ? vidx[a] < vidx[b] : name(a) < name(b);
  });
  for (size_t s = 0; s < nt;) {   // family sizes (:1531-1560)
    size_t e = s + 1;
    while (e < nt && vidx[sorted[e]] == vidx[sorted[s]]) ++e;
    if (vidx[sorted[s]]) go->families.push_back(e - s);
    s = e;
  }
  std::string mi;
  for (uint32_t t : sorted) {
    const Tpl& x = gp.tpls[t];
    const bool has = tkind[t] != FGB_MOL_NONE;
    if (has) mi_string(tkind[t], tid[t], base_mi, &mi);
    for (auto [off, len] : {std::pair<uint64_t, uint64_t>{x.r1, x.r1_len}, {x.r2, x.r2_len}}) {
      if (off == kNone) continue;
      if (has) emit_with_tag(gp.bytes.data() + off, len, g.opt.assign_tag, mi, &go->bytes);
      else emit_plain(gp.bytes.data() + off, len, &go->bytes);
      go->n_records++;
    }
  }
}

fgb_status finish_flush(fgb_grouper* g, const uint64_t* ids, const uint8_t* kinds, const uint64_t* mi_count,
                        const uint8_t** out, uint64_t* out_len, uint64_t* n_records) {
  const uint64_t ng = g->queue.size();
  std::vector<uint64_t> base;
  uint64_t next = g->stats[FGB_GSTAT_NEXT_MI];
  if (!mi_bases(mi_count, ng, &next, &base)) {
    g->last_error = "fgb_grouper_flush: MI counter overflow";
    return FGB_ERR_INVALID_ARG;
  }
  std::vector<GroupOut> outs(ng);
  fgb_umi::parallel_for(ng, g->opt.umi.n_threads, [&](uint64_t b) {
    const uint64_t u0 = g->batch.call_off[g->batch.group_off[b]];
    emit_group(*g, g->queue[b], ids + u0, kinds + u0, base[b], &outs[b]);
  });
  const uint64_t recs = concat_outputs(outs, g->opt.umi.n_threads, &g->out);
  for (uint64_t b = 0; b < ng; ++b) {
    for (uint64_t f : outs[b].families) g->family_sizes[f]++;
    if (!outs[b].families.empty()) g->group_sizes[outs[b].families.size()]++;
  }
  g->stats[FGB_GSTAT_NEXT_MI] = next;
  g->stats[FGB_GSTAT_RECORDS_OUT] += recs;
  g->queue.clear();
  g->batch.ready = false;
  *out = g->out.data();
  *out_len = g->out.size();
  *n_records = recs;
  return FGB_OK;
}

}  // namespace

fgb_status fgb::grp::group_by_position(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                       const char* header_text, size_t header_len, const char* cell_tag,
                                       bool include_secondary_supplementary, uint8_t* keep, uint64_t* group_begin,
                                       uint64_t* n_groups, uint64_t* bad_record) {
  if (!keep || !group_begin || !n_groups || (n_records && (!records || !rec_off)) || (header_len && !header_text))
    return FGB_ERR_INVALID_ARG;
  if (bad_record) *bad_record = kNone;
  try {
    const auto libs = library_index(std::string_view(header_text ? header_text : "", header_len));
    const char want[3][2] = {{'R', 'G'}, {'M', 'C'}, {cell_tag ? cell_tag[0] : '\0', cell_tag ? cell_tag[1] : '\0'}};
    PosKey cur{};
    bool have = false;
    uint64_t kept = 0, groups = 0, last = 0;
    auto join = [&](uint64_t i, PosKey&& k) {
      keep[i] = 1;
      bool same = have && k == cur;
      if (have && !same) {   // a new position continuing the previous record's QNAME stays (unmapped mates)
        const View lv(records + rec_off[last], rec_off[last + 1] - rec_off[last]);
        const View v(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
        same = read_name(lv) == read_name(v);
      }
      if (!same) { group_begin[groups++] = kept; cur = std::move(k); have = true; }
      last = i;
      ++kept;
    };
    for (uint64_t i = 0; i < n_records; ++i) {
      if (!record_ok(records, rec_off, i)) { if (bad_record) *bad_record = i; return FGB_ERR_LAYOUT; }
      const View v(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
      const uint16_t f = v.flags();
      keep[i] = 0;
      PosKey k{};
      if (f & (bam::kSecondary | bam::kSupplementary)) {   // grouper.rs:489-493
        if (!include_secondary_supplementary) continue;
        // GroupKey::default() with only the name hash (bam.rs:431-435); MC is not validated (:452-475)
        k.ref1 = INT32_MAX; k.pos1 = INT32_MAX; k.strand1 = UINT8_MAX;
        k.ref2 = INT32_MAX; k.pos2 = INT32_MAX; k.strand2 = UINT8_MAX;
        k.library = 0;
        k.has_cell = false;
        join(i, std::move(k));
        continue;
      }
      const uint8_t* val[3];
      size_t len[3];
      bam::find_string_tags(v, want, cell_tag ? 3 : 2, val, len);
      const bool mc = val[1] && bam::valid_utf8(val[1], len[1]);
      const bool paired = f & bam::kPaired, mate_unmapped = f & bam::kMateUnmapped;
      if (paired && !(f & bam::kUnmapped) && !mate_unmapped && !mc) {   // validate_mc_tag (:452-475)
        if (bad_record) *bad_record = i;
        return FGB_ERR_INVALID_ARG;
      }
      k.library = 0;
      if (val[0]) {
        auto it = libs.find(std::string(reinterpret_cast<const char*>(val[0]), len[0]));
        if (it != libs.end()) k.library = it->second;
      }
      k.has_cell = cell_tag && val[2];
      if (k.has_cell) k.cell.assign(reinterpret_cast<const char*>(val[2]), len[2]);
      const int32_t own_ref = v.ref_id(), own_pos = unclipped_5prime(v);
      const uint8_t strand = (f & bam::kReverse) ? 1 : 0;
      k.ref1 = own_ref; k.pos1 = own_pos; k.strand1 = strand;
      k.ref2 = INT32_MAX; k.pos2 = INT32_MAX; k.strand2 = UINT8_MAX;
      if (paired && !mate_unmapped && mc) {   // GroupKey::paired, lower (ref, pos, strand) first
        const char* c = reinterpret_cast<const char*>(val[1]);
        const bool mrev = f & bam::kMateReverse;
        const int32_t mpos1 = v.mate_pos() + 1;
        int32_t mp;
        if (mrev) {
          int32_t rl, tr;
          bam::mc_ref_len_and_trailing(c, len[1], &rl, &tr);
          mp = mpos1 + rl + tr - 1;
        } else {
          mp = mpos1 - bam::mc_leading_clips(c, len[1]);
        }
        const uint8_t ms = mrev ? 1 : 0;
        const int32_t mref = v.mate_ref_id();
        if (std::make_tuple(own_ref, own_pos, strand) <= std::make_tuple(mref, mp, ms)) {
          k.ref2 = mref; k.pos2 = mp; k.strand2 = ms;
        } else {
          k.ref1 = mref; k.pos1 = mp; k.strand1 = ms;
          k.ref2 = own_ref; k.pos2 = own_pos; k.strand2 = strand;
        }
      }
      join(i, std::move(k));
    }
    group_begin[groups] = kept;
    *n_groups = groups;
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
  return FGB_OK;
}

extern "C" {

fgb_status fgb_host_group_by_position(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                      const char* header_text, size_t header_len, const char* cell_tag,
                                      uint8_t* keep, uint64_t* group_begin, uint64_t* n_groups, uint64_t* bad_record) {
  return fgb::grp::group_by_position(records, rec_off, n_records, header_text, header_len, cell_tag, false, keep,
                                     group_begin, n_groups, bad_record);
}

fgb_status fgb_host_dedup_group_by_position(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                            const char* header_text, size_t header_len, const char* cell_tag,
                                            uint8_t* keep, uint64_t* group_begin, uint64_t* n_groups,
                                            uint64_t* bad_record) {
  return fgb::grp::group_by_position(records, rec_off, n_records, header_text, header_len, cell_tag, true, keep,
                                     group_begin, n_groups, bad_record);
}

fgb_status fgb_grouper_create(int device, const fgb_group_options* opt, fgb_grouper** out) {
  if (!opt || !out) return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  fgb_umi_options u = opt->umi;
  if (opt->no_umi) { u.strategy = FGB_UMI_IDENTITY; u.edits = 0; u.min_umi_length = 0; }   // group.rs:732-757
  if (!fgb_umi::check_options(u).empty()) return FGB_ERR_INVALID_ARG;
  if (opt->umi.strategy == FGB_UMI_PAIRED && (opt->umi.min_umi_length || opt->no_umi)) return FGB_ERR_INVALID_ARG;   // :723-730
  std::unique_ptr<fgb_grouper> g(new (std::nothrow) fgb_grouper());
  if (!g) return FGB_ERR_NOMEM;
  g->opt = *opt;
  g->umi = u;
  g->stats[FGB_GSTAT_NEXT_MI] = opt->first_mi;
  const fgb_status st = open_handle(device, &g->h);
  if (st != FGB_OK) return st;
  *out = g.release();
  return FGB_OK;
}

void fgb_grouper_destroy(fgb_grouper* g) {
  if (!g) return;
  if (g->h) fgb_destroy(g->h);
  delete g;
}

size_t fgb_grouper_last_error(const fgb_grouper* g, char* buf, size_t buf_len) {
  return g ? copy_error(g->last_error, buf, buf_len) : 0;
}

fgb_status fgb_grouper_add_groups(fgb_grouper* g, const uint8_t* records, const uint64_t* rec_off,
                                  const uint64_t* group_rec, uint64_t n_groups) {
  if (!g || !group_rec || (n_groups && (!records || !rec_off))) return FGB_ERR_INVALID_ARG;
  static const char kWho[] = "fgb_grouper_add_groups";
  return guarded(&g->last_error, kWho, [&]() -> fgb_status {
    std::vector<GroupPrep> prep;
    const fgb_status st = prepare_groups(
        kWho, records, rec_off, group_rec, n_groups, g->opt.umi.n_threads,
        [&](uint64_t b, uint64_t e, GroupPrep* gp) { return prepare_group(*g, records, rec_off, b, e, gp); }, &prep,
        &g->last_error);
    if (st != FGB_OK) return st;
    g->queue.reserve(g->queue.size() + n_groups);
    for (auto& gp : prep) {
      for (int k = 0; k < 6; ++k) g->stats[FGB_GSTAT_TOTAL + k] += gp.filter[k];
      g->stats[FGB_GSTAT_POSITION_GROUPS]++;
      if (gp.dropped) g->stats[FGB_GSTAT_GROUPS_DROPPED]++;
      if (gp.dropped || gp.tpls.empty()) continue;   // nothing of it reaches the output
      g->queue.push_back(std::move(gp));
    }
    g->batch.ready = false;
    return FGB_OK;
  });
}

fgb_status fgb_grouper_pending(fgb_grouper* g, const uint8_t** umis, const uint64_t** umi_off, uint64_t* n_umis,
                               const uint64_t** call_off, uint64_t* n_calls, const uint64_t** group_off,
                               uint64_t* n_groups) {
  if (!g || !umis || !umi_off || !n_umis || !call_off || !n_calls || !group_off || !n_groups) return FGB_ERR_INVALID_ARG;
  return guarded(&g->last_error, "fgb_grouper_pending", [&]() -> fgb_status {
    g->batch.build(g->queue);
    g->batch.pending(umis, umi_off, n_umis, call_off, n_calls, group_off, n_groups);
    return FGB_OK;
  });
}

fgb_status fgb_grouper_flush(fgb_grouper* g, const uint8_t** out, uint64_t* out_len, uint64_t* n_records) {
  if (!g || !out || !out_len || !n_records) return FGB_ERR_INVALID_ARG;
  if (!g->h) { g->last_error = "fgb_grouper_flush: a planning-only grouper has no device"; return FGB_ERR_NO_DEVICE; }
  return guarded(&g->last_error, "fgb_grouper_flush", [&]() -> fgb_status {
    g->batch.build(g->queue);
    const uint64_t n = g->batch.n_umis(), ng = g->batch.n_groups();
    std::vector<uint64_t> ids(n + 1), counts(ng + 1);
    std::vector<uint8_t> kinds(n + 1);
    const fgb_status st = g->batch.assign(g->h, g->umi, "fgb_grouper_flush", ids.data(), kinds.data(), counts.data(),
                                          &g->last_error);
    if (st != FGB_OK) return st;
    fgb_umi_last_timing(g->h, g->timing);
    const auto t0 = std::chrono::steady_clock::now();
    const fgb_status fs = finish_flush(g, ids.data(), kinds.data(), counts.data(), out, out_len, n_records);
    g->timing[4] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return fs;
  });
}

fgb_status fgb_grouper_last_timing(const fgb_grouper* g, double ms[5]) {
  if (!g || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, g->timing, sizeof(g->timing));
  return FGB_OK;
}

fgb_status fgb_grouper_flush_with_ids(fgb_grouper* g, const uint64_t* ids, const uint8_t* kinds,
                                      const uint64_t* group_mi_count, const uint8_t** out, uint64_t* out_len,
                                      uint64_t* n_records) {
  if (!g || !out || !out_len || !n_records) return FGB_ERR_INVALID_ARG;
  return guarded(&g->last_error, "fgb_grouper_flush_with_ids", [&]() -> fgb_status {
    g->batch.build(g->queue);
    const uint64_t n = g->batch.n_umis(), ng = g->batch.n_groups();
    if ((n && (!ids || !kinds)) || (ng && !group_mi_count)) return FGB_ERR_INVALID_ARG;
    for (uint64_t u = 0; u < n; ++u)
      if (kinds[u] > FGB_MOL_B) { g->last_error = "fgb_grouper_flush_with_ids: unknown kind"; return FGB_ERR_INVALID_ARG; }
    return finish_flush(g, ids, kinds, group_mi_count, out, out_len, n_records);
  });
}

fgb_status fgb_grouper_stats(const fgb_grouper* g, uint64_t stats[FGB_GROUP_NSTATS]) {
  if (!g || !stats) return FGB_ERR_INVALID_ARG;
  std::memcpy(stats, g->stats, sizeof(g->stats));
  return FGB_OK;
}

fgb_status fgb_grouper_histogram(const fgb_grouper* g, int which, uint64_t* sizes, uint64_t* counts, uint64_t cap,
                                 uint64_t* n) {
  if (!g || !n || (which != FGB_GROUP_HIST_FAMILY && which != FGB_GROUP_HIST_POSITION)) return FGB_ERR_INVALID_ARG;
  return copy_histogram(which == FGB_GROUP_HIST_FAMILY ? g->family_sizes : g->group_sizes, sizes, counts, cap, n);
}

}  // extern "C"
