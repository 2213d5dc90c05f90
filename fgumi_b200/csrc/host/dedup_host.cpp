// `fgumi dedup` around the UMI assignment and the template scores: the record-level deduper (fgb_deduper_*):
// templates with their secondary and supplementary records, dedup's filter, the orientation split and UMIs before
// fgb_umi_assign; the representative of each molecule, duplicate flags, MI tags and the MI counter after it.  The
// template scores come from the device (dedup_kernels.cuh through dedup_device.h) while the assignment runs.  Restated
// in tests/dedup_oracle.py; citations are to fgumi 0.2.0, dedup.rs = src/lib/commands/dedup.rs.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <map>
#include <memory>
#include <new>
#include <numeric>
#include <string>
#include <string_view>
#include <thread>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "bam.h"
#include "dedup_device.h"
#include "group_rules.h"
#include "record_link.h"
#include "umi_host.h"

namespace {

using fgb::bam::View;
namespace bam = fgb::bam;
using namespace fgb::grp;
using fgb::link::guarded;
using fgb::link::ms_since;

constexpr uint16_t kDuplicate = 0x400;

struct DRec { uint64_t off, len; };   // one record in its group's byte copy

struct DTpl {                         // one template that passed the filter
  uint64_t rec_begin = 0, rec_end = 0;   // its records in Template::from_records order (DGroup::recs)
  int64_t r1 = -1, r2 = -1;              // its primary reads (DGroup::recs index, -1: absent)
  uint64_t name = 0, name_len = 0;
};

struct DGroup {                       // one position group after the host rules in front of the assignment
  std::vector<uint8_t> bytes;
  std::vector<DRec> recs;
  std::vector<DTpl> tpls;             // in input order
  Calls c;
  uint64_t filter[6] = {0, 0, 0, 0, 0, 0};
};

enum { F_TOTAL, F_ACCEPTED, F_NON_PF, F_POOR, F_NS, F_SHORT };

}  // namespace

struct fgb_deduper {
  fgb_dedup_options opt{};
  fgb_umi_options umi{};              // what goes to fgb_umi_assign (identity and no_umi: 0 edits)
  fgb_handle* h = nullptr;
  std::vector<DGroup> queue;
  uint64_t stats[FGB_DEDUP_NSTATS] = {};
  std::map<uint64_t, uint64_t> family_sizes;
  std::string last_error;
  UmiBatch batch;                     // the queue's UMI batch (fgb_deduper_pending)
  std::vector<uint8_t> out;
  double timing[7] = {0, 0, 0, 0, 0, 0, 0};   // fgb_deduper_last_timing
};

namespace {

// filter_template (dedup.rs:257-402): counts are per TEMPLATE; a both-unmapped template is always rejected; the
// mate's MQ is compared signed (:363-372)
bool filter_template(const fgb_deduper& d, const View* r1, const View* r2, uint64_t* fc) {
  fc[F_TOTAL]++;
  if (!r1 && !r2) { fc[F_POOR]++; return false; }
  const bool both_unmapped = (!r1 || (r1->flags() & bam::kUnmapped)) && (!r2 || (r2->flags() & bam::kUnmapped));
  if (both_unmapped) { fc[F_POOR]++; return false; }
  const View* reads[2] = {r1, r2};
  for (const View* r : reads) {   // phase 1: flags and MAPQ (:281-297)
    if (!r) continue;
    const uint16_t f = r->flags();
    if (!d.opt.include_non_pf && (f & 0x200)) { fc[F_NON_PF]++; return false; }
    if (!(f & bam::kUnmapped) && r->b[9] < d.opt.min_map_q) { fc[F_POOR]++; return false; }
  }
  for (const View* r : reads) {   // phase 2: one aux walk for MQ and the UMI (:299-398)
    if (!r) continue;
    const bool check_mq = !(r->flags() & bam::kMateUnmapped);
    const MqUmi s = scan_mq_umi(*r, check_mq, !d.opt.no_umi, d.opt.umi_tag);
    if (check_mq && s.have_mq && s.mq < static_cast<int64_t>(d.opt.min_map_q)) { fc[F_POOR]++; return false; }
    if (d.opt.no_umi) continue;
    if (!s.have_umi) { fc[F_POOR]++; return false; }
    const int64_t bases = umi_bases(s.umi, s.umi_len);
    if (bases < 0) { fc[F_NS]++; return false; }
    if (d.opt.umi.min_umi_length && static_cast<uint64_t>(bases) < d.opt.umi.min_umi_length) { fc[F_SHORT]++; return false; }
  }
  fc[F_ACCEPTED]++;
  return true;
}

// One position group (process_position_group, dedup.rs:673-719): templates, filter, cleared duplicate flags, split,
// UMIs.  "" or the message of an error that fails the whole call.
std::string prepare_group(const fgb_deduper& d, const uint8_t* records, const uint64_t* rec_off, uint64_t b, uint64_t e,
                          DGroup* gp) {
  // build_templates_from_records (grouper.rs:596-651) + Template::from_records (template.rs:159-330)
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
    if (filter_template(d, v1, v2, gp->filter)) {
      DTpl t;
      t.rec_begin = gp->recs.size();
      auto copy = [&](uint64_t k) {   // the copy with 0x400 cleared (:706-716)
        const View& v = views[k];
        const uint64_t at = gp->bytes.size();
        gp->bytes.insert(gp->bytes.end(), v.b, v.b + v.n);
        const uint16_t f = static_cast<uint16_t>(v.flags() & ~kDuplicate);
        std::memcpy(gp->bytes.data() + at + 14, &f, 2);
        gp->recs.push_back(DRec{at, v.n});
      };
      for (uint64_t k : order) {
        if (static_cast<int64_t>(k) == r1) t.r1 = static_cast<int64_t>(gp->recs.size());
        if (static_cast<int64_t>(k) == r2) t.r2 = static_cast<int64_t>(gp->recs.size());
        copy(k);
      }
      t.rec_end = gp->recs.size();
      t.name = gp->recs[t.rec_begin].off + 32;
      t.name_len = name.size();
      gp->tpls.push_back(t);
    }
    i = j;
  }
  if (gp->tpls.empty()) return "";
  std::vector<View> pv;   // views of every copied record
  pv.reserve(gp->recs.size());
  for (const DRec& r : gp->recs) pv.emplace_back(gp->bytes.data() + r.off, r.len);
  return split_and_umis(d.umi, d.opt.no_umi, d.opt.umi_tag, gp->tpls.size(),
                        [&](size_t t) { return gp->tpls[t].r1 >= 0 ? &pv[gp->tpls[t].r1] : nullptr; },
                        [&](size_t t) { return gp->tpls[t].r2 >= 0 ? &pv[gp->tpls[t].r2] : nullptr; }, &gp->c);
}

// find_tag_type (fgumi-raw-bam): whether the record has an aux entry `tag` of any type
bool has_tag(const View& v, const char tag[2]) {
  const size_t aux = v.aux_off();
  for (size_t p = aux; aux <= v.n && p + 3 <= v.n;) {
    if (v.b[p] == static_cast<uint8_t>(tag[0]) && v.b[p + 1] == static_cast<uint8_t>(tag[1])) return true;
    const size_t size = tag_value_size(v.b[p + 2], v.b + p + 3, v.n - (p + 3));
    if (!size) return false;
    p += 3 + size;
  }
  return false;
}

struct DedupOut {
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> families;   // template count of each assigned molecule
  uint64_t n_records = 0;
  uint64_t m[9] = {};               // FGB_DSTAT_TOTAL_TEMPLATES .. FGB_DSTAT_MISSING_TC_TAG (unique_reads unset)
};

// process_position_group after the assignment (dedup.rs:721-806) and the output (:1080-1110) for queued group `gp`;
// ids / kinds / scores indexed like its batch entries (gp.c.order).
void emit_group(const fgb_deduper& d, const DGroup& gp, const uint64_t* ids, const uint8_t* kinds, const uint32_t* scores,
                uint64_t base_mi, DedupOut* go) {
  const size_t nt = gp.tpls.size();
  std::vector<uint64_t> tid(nt), vidx(nt);
  std::vector<uint8_t> tkind(nt), dup(nt, 0);
  std::vector<uint32_t> tscore(nt);
  for (size_t u = 0; u < nt; ++u) {
    const uint32_t t = gp.c.order[u];
    tkind[t] = kinds[u];
    tid[t] = ids[u];
    tscore[t] = scores[u];
    vidx[t] = vec_index(kinds[u], ids[u]);
  }
  auto name = [&](size_t t) {
    return std::string_view(reinterpret_cast<const char*>(gp.bytes.data() + gp.tpls[t].name), gp.tpls[t].name_len);
  };
  std::vector<uint32_t> sorted(nt);   // (:721-726)
  std::iota(sorted.begin(), sorted.end(), 0u);
  std::stable_sort(sorted.begin(), sorted.end(), [&](uint32_t a, uint32_t b) {
    return vidx[a] != vidx[b] ? vidx[a] < vidx[b] : name(a) < name(b);
  });
  // families (:728-762): the representative is the first template of the family in sorted order with the highest
  // score -- what mark_duplicates_in_family's size-2, size-3 (ties to the earlier) and general paths (a stable sort by
  // score descending) all pick
  for (size_t s = 0; s < nt;) {
    size_t e = s + 1;
    while (e < nt && vidx[sorted[e]] == vidx[sorted[s]]) ++e;
    if (vidx[sorted[s]]) {
      go->families.push_back(e - s);
      size_t best = s;
      for (size_t x = s + 1; x < e; ++x) if (tscore[sorted[x]] > tscore[sorted[best]]) best = x;
      for (size_t x = s; x < e; ++x) if (x != best) dup[sorted[x]] = 1;
      go->m[FGB_DSTAT_UNIQUE_TEMPLATES]++;
      go->m[FGB_DSTAT_DUPLICATE_TEMPLATES] += e - s - 1;
    }
    s = e;
  }
  static const char kTc[2] = {'t', 'c'};
  go->bytes.reserve(gp.bytes.size() + 32 * gp.recs.size());   // the records, their block_size words and MI tags
  std::string mi;
  for (uint32_t t : sorted) {
    const DTpl& x = gp.tpls[t];
    const bool has = tkind[t] != FGB_MOL_NONE;
    if (has) mi_string(tkind[t], tid[t], base_mi, &mi);
    go->m[FGB_DSTAT_TOTAL_TEMPLATES]++;
    for (uint64_t r = x.rec_begin; r < x.rec_end; ++r) {
      const uint8_t* rec = gp.bytes.data() + gp.recs[r].off;
      const uint64_t len = gp.recs[r].len;
      const View v(rec, len);
      const uint16_t f = v.flags();   // counts (:764-787)
      go->m[FGB_DSTAT_TOTAL_READS]++;
      if (dup[t]) go->m[FGB_DSTAT_DUPLICATE_READS]++;
      if (f & bam::kSecondary) go->m[FGB_DSTAT_SECONDARY_READS]++;
      if (f & bam::kSupplementary) go->m[FGB_DSTAT_SUPPLEMENTARY_READS]++;
      if ((f & (bam::kSecondary | bam::kSupplementary)) && !has_tag(v, kTc)) go->m[FGB_DSTAT_MISSING_TC_TAG]++;
      if (dup[t] && d.opt.remove_duplicates) continue;   // (:1087-1092)
      const size_t at = go->bytes.size();
      if (has) emit_with_tag(rec, len, d.opt.assign_tag, mi, &go->bytes);
      else emit_plain(rec, len, &go->bytes);
      if (dup[t]) {   // mark_template_as_duplicate (:660-666)
        const uint16_t fd = static_cast<uint16_t>(f | kDuplicate);
        std::memcpy(go->bytes.data() + at + 4 + 14, &fd, 2);
      }
      go->n_records++;
    }
  }
}

fgb_status finish_flush(fgb_deduper* d, const uint64_t* ids, const uint8_t* kinds, const uint64_t* mi_count,
                        const uint32_t* scores, const uint8_t** out, uint64_t* out_len, uint64_t* n_records) {
  const uint64_t ng = d->queue.size();
  std::vector<uint64_t> base;
  uint64_t next = d->stats[FGB_DSTAT_NEXT_MI];
  if (!mi_bases(mi_count, ng, &next, &base)) {
    d->last_error = "fgb_deduper_flush: MI counter overflow";
    return FGB_ERR_INVALID_ARG;
  }
  std::vector<DedupOut> outs(ng);
  fgb_umi::parallel_for(ng, d->opt.umi.n_threads, [&](uint64_t b) {
    const uint64_t u0 = d->batch.call_off[d->batch.group_off[b]];
    emit_group(*d, d->queue[b], ids + u0, kinds + u0, scores + u0, base[b], &outs[b]);
  });
  const uint64_t recs = concat_outputs(outs, d->opt.umi.n_threads, &d->out);
  for (uint64_t b = 0; b < ng; ++b) {
    for (uint64_t f : outs[b].families) d->family_sizes[f]++;
    for (int k = 0; k <= FGB_DSTAT_MISSING_TC_TAG; ++k) d->stats[k] += outs[b].m[k];
  }
  d->stats[FGB_DSTAT_UNIQUE_READS] = d->stats[FGB_DSTAT_TOTAL_READS] - d->stats[FGB_DSTAT_DUPLICATE_READS];
  d->stats[FGB_DSTAT_NEXT_MI] = next;
  d->stats[FGB_DSTAT_RECORDS_OUT] += recs;
  d->queue.clear();
  d->batch.ready = false;
  *out = d->out.data();
  *out_len = d->out.size();
  *n_records = recs;
  return FGB_OK;
}

}  // namespace

extern "C" {

fgb_status fgb_deduper_create(int device, const fgb_dedup_options* opt, fgb_deduper** out) {
  if (!opt || !out) return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  if (opt->umi.rules != FGB_UMI_RULES_MAPPED) return FGB_ERR_INVALID_ARG;   // dedup has no --allow-unmapped
  if (opt->umi.strategy == FGB_UMI_PAIRED && (opt->umi.min_umi_length || opt->no_umi)) return FGB_ERR_INVALID_ARG;   // :913-921
  fgb_umi_options u = opt->umi;
  if (opt->no_umi) { u.strategy = FGB_UMI_IDENTITY; u.min_umi_length = 0; }   // :923-931
  if (u.strategy == FGB_UMI_IDENTITY) u.edits = 0;                             // :940-947
  if (!fgb_umi::check_options(u).empty()) return FGB_ERR_INVALID_ARG;
  std::unique_ptr<fgb_deduper> d(new (std::nothrow) fgb_deduper());
  if (!d) return FGB_ERR_NOMEM;
  d->opt = *opt;
  d->umi = u;
  d->stats[FGB_DSTAT_NEXT_MI] = opt->first_mi;
  const fgb_status st = open_handle(device, &d->h);
  if (st != FGB_OK) return st;
  *out = d.release();
  return FGB_OK;
}

void fgb_deduper_destroy(fgb_deduper* d) {
  if (!d) return;
  if (d->h) fgb_destroy(d->h);
  delete d;
}

size_t fgb_deduper_last_error(const fgb_deduper* d, char* buf, size_t buf_len) {
  return d ? copy_error(d->last_error, buf, buf_len) : 0;
}

fgb_status fgb_deduper_add_groups(fgb_deduper* d, const uint8_t* records, const uint64_t* rec_off,
                                  const uint64_t* group_rec, uint64_t n_groups) {
  if (!d || !group_rec || (n_groups && (!records || !rec_off))) return FGB_ERR_INVALID_ARG;
  static const char kWho[] = "fgb_deduper_add_groups";
  return guarded(&d->last_error, kWho, [&]() -> fgb_status {
    std::vector<DGroup> prep;   // an assignment error fails the command (dedup.rs:717-719)
    const fgb_status st = prepare_groups(
        kWho, records, rec_off, group_rec, n_groups, d->opt.umi.n_threads,
        [&](uint64_t b, uint64_t e, DGroup* gp) { return prepare_group(*d, records, rec_off, b, e, gp); }, &prep,
        &d->last_error);
    if (st != FGB_OK) return st;
    d->queue.reserve(d->queue.size() + n_groups);
    for (auto& gp : prep) {
      for (int k = 0; k < 6; ++k) d->stats[FGB_DSTAT_FILTER_TOTAL + k] += gp.filter[k];
      d->stats[FGB_DSTAT_POSITION_GROUPS]++;
      if (gp.tpls.empty()) continue;   // nothing of it reaches the output (:696-704)
      d->queue.push_back(std::move(gp));
    }
    d->batch.ready = false;
    return FGB_OK;
  });
}

fgb_status fgb_deduper_pending(fgb_deduper* d, const uint8_t** umis, const uint64_t** umi_off, uint64_t* n_umis,
                               const uint64_t** call_off, uint64_t* n_calls, const uint64_t** group_off,
                               uint64_t* n_groups) {
  if (!d || !umis || !umi_off || !n_umis || !call_off || !n_calls || !group_off || !n_groups) return FGB_ERR_INVALID_ARG;
  return guarded(&d->last_error, "fgb_deduper_pending", [&]() -> fgb_status {
    d->batch.build(d->queue);
    d->batch.pending(umis, umi_off, n_umis, call_off, n_calls, group_off, n_groups);
    return FGB_OK;
  });
}

fgb_status fgb_deduper_flush(fgb_deduper* d, const uint8_t** out, uint64_t* out_len, uint64_t* n_records) {
  if (!d || !out || !out_len || !n_records) return FGB_ERR_INVALID_ARG;
  if (!d->h) { d->last_error = "fgb_deduper_flush: a planning-only deduper has no device"; return FGB_ERR_NO_DEVICE; }
  return guarded(&d->last_error, "fgb_deduper_flush", [&]() -> fgb_status {
    d->batch.build(d->queue);
    const uint64_t n = d->batch.n_umis(), ng = d->batch.n_groups();
    // the primary records of every batch entry, R1 then R2 (score_template, dedup.rs:230-249)
    std::vector<const uint8_t*> rp;
    std::vector<uint64_t> rl, first(n + 1);
    rp.reserve(2 * n);
    rl.reserve(2 * n);
    uint64_t u = 0;
    for (const DGroup& gp : d->queue)
      for (uint32_t t : gp.c.order) {
        first[u++] = rp.size();
        for (int64_t r : {gp.tpls[t].r1, gp.tpls[t].r2}) {
          if (r < 0) continue;
          rp.push_back(gp.bytes.data() + gp.recs[r].off);
          rl.push_back(gp.recs[r].len);
        }
      }
    first[n] = rp.size();
    std::vector<uint32_t> rscore(rp.size() + 1);
    std::vector<uint64_t> ids(n + 1), counts(ng + 1);
    std::vector<uint8_t> kinds(n + 1);
    // the score phase runs on its own thread and stream while the assignment runs here
    fgb_status score_st = FGB_OK;
    float kernel_ms = 0.f;
    double score_ms = 0.0;
    std::string score_err;
    std::thread scorer([&] {
      const auto t0 = std::chrono::steady_clock::now();
      score_st = guarded(&score_err, "template scores", [&] {
        return fgb::dedupdev::quality_scores(d->h, rp.size(), rp.data(), rl.data(), d->opt.umi.n_threads,
                                             rscore.data(), &kernel_ms, &score_err);
      });
      score_ms = ms_since(t0);
    });
    const fgb_status st = d->batch.assign(d->h, d->umi, "fgb_deduper_flush", ids.data(), kinds.data(), counts.data(),
                                          &d->last_error);
    scorer.join();
    if (st != FGB_OK) return st;
    if (score_st != FGB_OK) { d->last_error = "fgb_deduper_flush: " + score_err; return score_st; }
    fgb_umi_last_timing(d->h, d->timing);
    d->timing[4] = score_ms;
    d->timing[5] = kernel_ms;
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<uint32_t> scores(n + 1);   // a template's score: its R1 score plus its R2 score
    for (uint64_t x = 0; x < n; ++x)
      for (uint64_t k = first[x]; k < first[x + 1]; ++k) scores[x] += rscore[k];
    const fgb_status fs = finish_flush(d, ids.data(), kinds.data(), counts.data(), scores.data(), out, out_len, n_records);
    d->timing[6] = ms_since(t0);
    return fs;
  });
}

fgb_status fgb_deduper_flush_with_ids(fgb_deduper* d, const uint64_t* ids, const uint8_t* kinds,
                                      const uint64_t* group_mi_count, const uint32_t* scores, const uint8_t** out,
                                      uint64_t* out_len, uint64_t* n_records) {
  if (!d || !out || !out_len || !n_records) return FGB_ERR_INVALID_ARG;
  return guarded(&d->last_error, "fgb_deduper_flush_with_ids", [&]() -> fgb_status {
    d->batch.build(d->queue);
    const uint64_t n = d->batch.n_umis(), ng = d->batch.n_groups();
    if ((n && (!ids || !kinds || !scores)) || (ng && !group_mi_count)) return FGB_ERR_INVALID_ARG;
    for (uint64_t u = 0; u < n; ++u)
      if (kinds[u] > FGB_MOL_B) { d->last_error = "fgb_deduper_flush_with_ids: unknown kind"; return FGB_ERR_INVALID_ARG; }
    return finish_flush(d, ids, kinds, group_mi_count, scores, out, out_len, n_records);
  });
}

fgb_status fgb_deduper_stats(const fgb_deduper* d, uint64_t stats[FGB_DEDUP_NSTATS]) {
  if (!d || !stats) return FGB_ERR_INVALID_ARG;
  std::memcpy(stats, d->stats, sizeof(d->stats));
  return FGB_OK;
}

fgb_status fgb_deduper_histogram(const fgb_deduper* d, uint64_t* sizes, uint64_t* counts, uint64_t cap, uint64_t* n) {
  if (!d || !n) return FGB_ERR_INVALID_ARG;
  return copy_histogram(d->family_sizes, sizes, counts, cap, n);
}

fgb_status fgb_deduper_last_timing(const fgb_deduper* d, double ms[7]) {
  if (!d || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, d->timing, sizeof(d->timing));
  return FGB_OK;
}

}  // extern "C"
