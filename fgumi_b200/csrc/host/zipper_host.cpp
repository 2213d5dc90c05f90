// `fgumi zipper` from raw BAM records (src/lib/commands/zipper.rs:826-941): the driver of the device zipper
// (fgb_zipper_records) and its host twin for tests (fgb_host_zipper_records).  The host checks the records it reaches,
// walks the join of the two streams' QNAME runs (Template::from_records order for both) and builds one ZRec per output
// record; runs of whole templates that fit a device budget cross the link through record_link.h's staging and are
// sized and written by the kernels of ../zipper_kernels.cuh, with the per-record rules of zipper_rules.h.  Restated in
// tests/zipper_oracle.py.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <string>
#include <string_view>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "group_rules.h"
#include "record_link.h"
#include "umi_host.h"
#include "zipper_device.h"
#include "zipper_rules.h"

namespace {

namespace link = fgb::link;
namespace zip = fgb::zip;
using link::ms_since;
constexpr uint64_t kNone = UINT64_MAX;

struct Stream {
  const uint8_t* rec;
  const uint64_t* off;
  uint64_t n;
  uint64_t bad_base;   // the stream's first record as bad_record counts it
  bool mapped;
};

struct Fail {
  fgb_status st = FGB_OK;
  uint64_t bad = kNone;
  std::string why;
};

// "" or why record i fails the call; *layout: FGB_ERR_LAYOUT rather than FGB_ERR_INVALID_ARG
std::string check_record(const Stream& s, uint64_t i, bool* layout) {
  *layout = true;
  if (s.off[i + 1] < s.off[i] || s.off[i + 1] - s.off[i] < 32) return "is shorter than 32 bytes";
  const uint8_t* r = s.rec + s.off[i];
  const uint64_t len = s.off[i + 1] - s.off[i];
  const uint64_t nc = zip::ld16(r + 12), L = zip::ld32(r + 16);
  const uint64_t ao = 32ull + r[8] + 4 * nc + (L + 1) / 2 + L;
  if (ao > len || len > UINT32_MAX) return "is truncated: its name, CIGAR, sequence or qualities run past its end";
  std::vector<uint16_t> names;
  for (uint64_t p = ao; p < len;) {
    uint8_t sub;
    uint32_t cnt;
    const size_t sz = p + 3 <= len ? fgb::rfilter::value_size(r + ao, len - ao, p - ao, &sub, &cnt) : 0;
    if (!sz || p + 3 + sz > len) return "has an aux area that does not parse to its end";
    names.push_back(static_cast<uint16_t>(r[p] | (r[p + 1] << 8)));
    p += 3 + sz;
  }
  *layout = false;
  for (size_t a = 0; a < names.size(); ++a)
    for (size_t b = a + 1; b < names.size(); ++b)
      if (names[a] == names[b])
        return std::string("carries the tag ") + static_cast<char>(names[a] & 0xFF) + static_cast<char>(names[a] >> 8) +
               " twice";
  if (s.mapped)
    for (uint64_t k = 0; k < nc; ++k)
      if ((zip::ld32(r + 32 + r[8] + 4 * k) & 0xF) > 8) return "has a CIGAR op code past 8";
  return "";
}

std::string_view name_of(const Stream& s, uint64_t i) {
  const uint8_t* r = s.rec + s.off[i];
  return std::string_view(reinterpret_cast<const char*>(r + 32), r[8] ? r[8] - 1 : 0);
}

// The QNAME run at i, each record checked as it is reached: [i, *e), its template order and primaries
struct Tpl {
  uint64_t b = 0, e = 0;
  int64_t r1 = -1, r2 = -1;
  std::vector<uint64_t> order;
};
bool take_template(const Stream& s, uint64_t i, Tpl* t, std::vector<uint64_t> lists[4], Fail* f) {
  bool layout;
  std::string why = check_record(s, i, &layout);
  uint64_t j = i + 1;
  if (why.empty()) {
    const std::string_view nm = name_of(s, i);
    for (; j < s.n; ++j) {
      if ((why = check_record(s, j, &layout)).empty() && name_of(s, j) != nm) break;
      if (!why.empty()) { i = j; break; }
    }
  }
  if (!why.empty()) {
    f->st = layout ? FGB_ERR_LAYOUT : FGB_ERR_INVALID_ARG;
    f->bad = s.bad_base + i;
    f->why = why;
    return false;
  }
  t->b = i;
  t->e = j;
  t->order.clear();
  uint64_t dup = 0;
  why = fgb::grp::template_order(i, j, [&](uint64_t k) { return zip::ld16(s.rec + s.off[k] + 14); }, name_of(s, i),
                                 lists, &t->order, &t->r1, &t->r2, &dup);
  if (!why.empty()) {
    f->st = FGB_ERR_INVALID_ARG;
    f->bad = s.bad_base + dup;
    f->why = why;
    return false;
  }
  return true;
}

// The join (process_raw, zipper.rs:849-930): the output records, and per template where it ends in the output and
// in both streams
struct Join {
  std::vector<zip::ZRec> zr;        // global record indices
  std::vector<uint64_t> z_end, u_end, m_end;
  uint64_t consumed = 0, merged = 0, passed = 0, excluded = 0;
};

bool join(const fgb_zipper_options& o, const Stream& us, const Stream& ms, bool last_call, Join* J, Fail* f) {
  std::vector<uint64_t> lists[4];
  Tpl ut, mt;
  bool peeked = false;
  uint64_t m = 0;
  for (uint64_t u = 0; u < us.n; u = ut.e) {
    if (!take_template(us, u, &ut, lists, f)) return false;
    if (!peeked && m < ms.n) {
      if (!take_template(ms, m, &mt, lists, f)) return false;
      peeked = true;
    }
    if (peeked && name_of(ms, mt.b) == name_of(us, ut.b)) {
      const uint32_t mr1 = mt.r1 < 0 ? zip::kNone : static_cast<uint32_t>(mt.r1);
      const uint32_t mr2 = mt.r2 < 0 ? zip::kNone : static_cast<uint32_t>(mt.r2);
      for (uint64_t k : mt.order) {
        const uint16_t fl = zip::ld16(ms.rec + ms.off[k] + 14);
        const bool is_r1 = !(fl & 1) || (fl & 0x40);
        zip::ZRec z{};
        z.src = static_cast<uint32_t>(k);
        z.mate = z.partner = zip::kNone;
        z.kind = zip::kMerged;
        z.r1 = mr1;
        z.r2 = mr2;
        const int64_t u_seg = is_r1 ? ut.r1 : ut.r2;
        z.umap = u_seg < 0 ? zip::kNone : static_cast<uint32_t>(u_seg);
        const bool primary = !(fl & 0x900);
        if (primary && mt.r1 >= 0 && mt.r2 >= 0) {
          z.role = zip::kRolePrim;
          z.mate = is_r1 ? mr2 : mr1;
          z.partner = static_cast<uint32_t>(k);
          z.mate_is_r1 = !is_r1;
        } else if (!(fl & 0x100) && (fl & 0x800) && (is_r1 ? mt.r2 : mt.r1) >= 0) {
          z.role = zip::kRoleSupp;
          z.mate = is_r1 ? mr2 : mr1;
          z.partner = is_r1 ? mr1 : mr2;
          z.mate_is_r1 = !is_r1;
        }
        J->zr.push_back(z);
      }
      m = mt.e;
      peeked = false;
      ++J->merged;
    } else if (o.exclude_missing_reads) {
      ++J->excluded;
    } else {
      for (uint64_t k : ut.order) {
        zip::ZRec z{};
        z.src = static_cast<uint32_t>(k);
        z.mate = z.partner = z.umap = z.r1 = z.r2 = zip::kNone;
        z.kind = zip::kPass;
        J->zr.push_back(z);
      }
      ++J->passed;
    }
    J->z_end.push_back(J->zr.size());
    J->u_end.push_back(ut.e);
    J->m_end.push_back(m);
  }
  if (last_call && m < ms.n) {
    if (!peeked && !take_template(ms, m, &mt, lists, f)) return false;
    f->st = FGB_ERR_INVALID_ARG;
    f->bad = ms.bad_base + mt.b;
    f->why = "is in a mapped template left over after every unmapped template: '" + std::string(name_of(ms, mt.b)) +
             "'; the unmapped and mapped reads must have the same read names in the same order, each name's records "
             "consecutive";
    return false;
  }
  J->consumed = m;
  return true;
}

// The tag lists as one array of names (remove, reverse, revcomp); false for a name with a NUL byte
bool tag_lists(const fgb_zipper_options& o, std::vector<uint8_t>* names) {
  const uint64_t n[3] = {o.n_remove, o.n_reverse, o.n_revcomp};
  const char (*l[3])[2] = {o.tags_to_remove, o.tags_to_reverse, o.tags_to_revcomp};
  for (int k = 0; k < 3; ++k) {
    if (n[k] && !l[k]) return false;
    for (uint64_t i = 0; i < n[k]; ++i) {
      if (!l[k][i][0] || !l[k][i][1]) return false;
      names->push_back(static_cast<uint8_t>(l[k][i][0]));
      names->push_back(static_cast<uint8_t>(l[k][i][1]));
    }
  }
  return true;
}

zip::Sets sets_at(const fgb_zipper_options& o, const uint8_t* names) {
  return zip::Sets{names, names + 2 * o.n_remove, names + 2 * (o.n_remove + o.n_reverse), static_cast<uint32_t>(o.n_remove),
                   static_cast<uint32_t>(o.n_reverse), static_cast<uint32_t>(o.n_revcomp)};
}

fgb_status zipper_impl(const link::HandleInfo& hi, const fgb_zipper_options& o, const Stream& us, const Stream& ms,
                       bool last_call, uint64_t* consumed, uint64_t* stats, Fail* fl) {
  auto fail = [&](cudaError_t e, const char* what) { return link::fail(hi.last_error, "fgb_zipper_records", e, what); };
  double* tm = hi.timing;
  auto t_host = std::chrono::steady_clock::now();
  std::vector<uint8_t> names;
  tag_lists(o, &names);
  Join J;
  if (!join(o, us, ms, last_call, &J, fl)) return fl->st;
  const uint64_t n_tpl = J.z_end.size();
  link::Resources r(hi.stream, o.n_threads);
  cudaError_t e = cudaSetDevice(hi.device);
  if (e != cudaSuccess) return fail(e, "cudaSetDevice");
  uint64_t budget;
  if ((e = link::device_budget(o.device_bytes, &budget)) != cudaSuccess) return fail(e, "cudaMemGetInfo");
  // runs of whole templates: both streams' bytes, the output and ~160 bytes of tables per record
  std::vector<uint64_t> run_tpl{0};
  uint64_t max_z = 0, max_u = 0, max_m = 0, max_ub = 0, max_mb = 0;
  auto at = [](const std::vector<uint64_t>& v, uint64_t t) { return t ? v[t - 1] : 0; };
  for (uint64_t t = 0; t < n_tpl;) {
    uint64_t v = t + 1;
    while (v < n_tpl) {
      const uint64_t recs = J.z_end[v] - at(J.z_end, t) + J.u_end[v] - at(J.u_end, t) + J.m_end[v] - at(J.m_end, t);
      const uint64_t bytes = us.off[J.u_end[v]] - us.off[at(J.u_end, t)] + ms.off[J.m_end[v]] - ms.off[at(J.m_end, t)];
      if (3 * bytes + recs * 160 > budget || J.z_end[v] - at(J.z_end, t) >= INT32_MAX / 2) break;
      ++v;
    }
    max_z = std::max(max_z, J.z_end[v - 1] - at(J.z_end, t));
    max_u = std::max(max_u, J.u_end[v - 1] - at(J.u_end, t));
    max_m = std::max(max_m, J.m_end[v - 1] - at(J.m_end, t));
    max_ub = std::max(max_ub, us.off[J.u_end[v - 1]] - us.off[at(J.u_end, t)]);
    max_mb = std::max(max_mb, ms.off[J.m_end[v - 1]] - ms.off[at(J.m_end, t)]);
    run_tpl.push_back(v);
    t = v;
  }
  uint8_t *d_um, *d_mp, *d_names, *d_temp, *d_out = nullptr;
  uint64_t *d_uoff, *d_moff, *d_size, *d_off, cap_out = 0;
  zip::ZRec* d_zr;
  size_t t_scan = 0;
  if ((e = fgb::zipdev::offsets(nullptr, &t_scan, nullptr, nullptr, static_cast<uint32_t>(max_z), hi.stream)))
    return fail(e, "CUB temp storage");
  if ((e = r.alloc(&d_um, max_ub + 16)) || (e = r.alloc(&d_mp, max_mb + 16)) || (e = r.alloc(&d_uoff, max_u + 1)) ||
      (e = r.alloc(&d_moff, max_m + 1)) || (e = r.alloc(&d_zr, max_z)) || (e = r.alloc(&d_size, max_z + 1)) ||
      (e = r.alloc(&d_off, max_z + 1)) || (e = r.alloc(&d_names, names.size() + 2)) || (e = r.alloc(&d_temp, t_scan + 16)))
    return fail(e, "cudaMalloc");
  // FGB_ZIPPER_STAGE_BYTES (at least 4096) lowers the staging buffers' size, so that small inputs cross several chunks
  uint64_t stage_cap = link::kStageBytes;
  if (const char* env = std::getenv("FGB_ZIPPER_STAGE_BYTES"))
    stage_cap = std::max<uint64_t>(4096, std::min<uint64_t>(link::kStageBytes, std::strtoull(env, nullptr, 10)));
  const char* what;
  if ((e = r.open(std::min<uint64_t>(stage_cap, std::max<uint64_t>(std::max(max_ub, max_mb) + 64, (max_z + 1) * 28)),
                  &what)))
    return fail(e, what);
  if (!names.empty() && (e = cudaMemcpy(d_names, names.data(), names.size(), cudaMemcpyHostToDevice)))
    return fail(e, "cudaMemcpy");
  const zip::Sets sets = sets_at(o, d_names);
  tm[5] += ms_since(t_host);
  std::vector<uint8_t>& out = *hi.kept;
  std::vector<uint64_t> lu, lm;
  std::vector<zip::ZRec> lz;
  for (uint64_t x = 0; x + 1 < run_tpl.size(); ++x) {
    t_host = std::chrono::steady_clock::now();
    const uint64_t t0 = run_tpl[x], t1 = run_tpl[x + 1];
    const uint64_t z0 = at(J.z_end, t0), z1 = J.z_end[t1 - 1], u0 = at(J.u_end, t0), u1 = J.u_end[t1 - 1],
                   m0 = at(J.m_end, t0), m1 = J.m_end[t1 - 1];
    const uint32_t nz = static_cast<uint32_t>(z1 - z0);
    lu.resize(u1 - u0 + 1);
    lm.resize(m1 - m0 + 1);
    for (uint64_t i = u0; i <= u1; ++i) lu[i - u0] = us.off[i] - us.off[u0];
    for (uint64_t i = m0; i <= m1; ++i) lm[i - m0] = ms.off[i] - ms.off[m0];
    lz.assign(J.zr.begin() + z0, J.zr.begin() + z1);
    for (zip::ZRec& z : lz) {   // run-local indices
      const uint64_t sb = z.kind == zip::kPass ? u0 : m0;
      z.src -= static_cast<uint32_t>(sb);
      for (uint32_t* q : {&z.mate, &z.partner, &z.r1, &z.r2})
        if (*q != zip::kNone) *q -= static_cast<uint32_t>(m0);
      if (z.umap != zip::kNone) z.umap -= static_cast<uint32_t>(u0);
    }
    tm[5] += ms_since(t_host);
    auto t_up = std::chrono::steady_clock::now();
    if ((e = r.upload(d_um, us.rec + us.off[u0], lu.back())) || (e = r.upload(d_uoff, lu.data(), lu.size() * 8)) ||
        (e = r.upload(d_mp, ms.rec + ms.off[m0], lm.back())) || (e = r.upload(d_moff, lm.data(), lm.size() * 8)) ||
        (e = r.upload(d_zr, lz.data(), lz.size() * sizeof(zip::ZRec))) || (e = cudaStreamSynchronize(hi.stream)))
      return fail(e, "upload");
    tm[0] += ms_since(t_up);
    uint64_t total = 0;
    size_t tb = t_scan + 16;
    if ((e = cudaEventRecord(r.ev[0], hi.stream)) ||
        (e = fgb::zipdev::sizes(d_um, d_uoff, d_mp, d_moff, d_zr, nz, sets, o.skip_pa_tags != 0, d_size, hi.sm_count,
                                hi.stream)) ||
        (e = cudaEventRecord(r.ev[1], hi.stream)) ||
        (e = fgb::zipdev::offsets(d_temp, &tb, d_size, d_off, nz, hi.stream)) ||
        (e = cudaEventRecord(r.ev[2], hi.stream)) ||
        (e = cudaMemcpyAsync(&total, d_off + nz, 8, cudaMemcpyDeviceToHost, hi.stream)) ||
        (e = cudaStreamSynchronize(hi.stream)))
      return fail(e, "size pass");
    t_host = std::chrono::steady_clock::now();
    if ((e = r.grow(&d_out, &cap_out, total + 16))) return fail(e, "cudaMalloc");
    tm[5] += ms_since(t_host);
    if ((e = cudaEventRecord(r.ev[3], hi.stream)) ||
        (e = fgb::zipdev::write(d_um, d_uoff, d_mp, d_moff, d_zr, nz, sets, o.skip_pa_tags != 0, d_off, d_out,
                                hi.sm_count, hi.stream)) ||
        (e = cudaEventRecord(r.ev[4], hi.stream)) || (e = cudaStreamSynchronize(hi.stream)))
      return fail(e, "write pass");
    float a = 0, b = 0, c = 0;
    cudaEventElapsedTime(&a, r.ev[0], r.ev[1]);
    cudaEventElapsedTime(&b, r.ev[1], r.ev[2]);
    cudaEventElapsedTime(&c, r.ev[3], r.ev[4]);
    tm[1] += a; tm[2] += b; tm[3] += c;
    auto t_dn = std::chrono::steady_clock::now();
    const uint64_t o0 = out.size();
    out.resize(o0 + total);
    if ((e = r.download(out.data() + o0, d_out, total))) return fail(e, "download");
    tm[4] += ms_since(t_dn);
  }
  *consumed = J.consumed;
  stats[FGB_ZSTAT_MERGED] = J.merged;
  stats[FGB_ZSTAT_UNMAPPED_ONLY] = J.passed;
  stats[FGB_ZSTAT_EXCLUDED] = J.excluded;
  stats[FGB_ZSTAT_RECORDS_OUT] = J.zr.size();
  return FGB_OK;
}

bool args_ok(const fgb_zipper_options* opt, const uint8_t* unmapped, const uint64_t* u_off, uint64_t n_unmapped,
             const uint8_t* mapped, const uint64_t* m_off, uint64_t n_mapped, const void* out, const void* out_len,
             const void* consumed, const void* stats) {
  return opt && u_off && m_off && out && out_len && consumed && stats && (!n_unmapped || unmapped) &&
         (!n_mapped || mapped) && !opt->restore_unconverted_bases && n_unmapped < UINT32_MAX && n_mapped < UINT32_MAX;
}

}  // namespace

extern "C" {

fgb_status fgb_zipper_records(fgb_handle* h, const fgb_zipper_options* opt, const uint8_t* unmapped,
                              const uint64_t* u_off, uint64_t n_unmapped, const uint8_t* mapped, const uint64_t* m_off,
                              uint64_t n_mapped, int last_call, const uint8_t** out, uint64_t* out_len,
                              uint64_t* mapped_consumed, uint64_t stats[FGB_ZIPPER_NSTATS], uint64_t* bad_record) {
  if (bad_record) *bad_record = kNone;
  if (!h || !args_ok(opt, unmapped, u_off, n_unmapped, mapped, m_off, n_mapped, out, out_len, mapped_consumed, stats))
    return FGB_ERR_INVALID_ARG;
  const link::HandleInfo hi = link::info(h, link::Command::kZipper);
  std::fill(hi.timing, hi.timing + 6, 0.0);
  std::fill(stats, stats + FGB_ZIPPER_NSTATS, 0);
  *out = nullptr;
  *out_len = 0;
  *mapped_consumed = 0;
  std::vector<uint8_t> names;
  if (!tag_lists(*opt, &names)) {
    *hi.last_error = "fgb_zipper_records: a tag list entry is not a two-byte tag name";
    return FGB_ERR_INVALID_ARG;
  }
  if (hi.busy) { *hi.last_error = "fgb_zipper_records: a submit has not been waited on"; return FGB_ERR_BUSY; }
  const Stream us{unmapped, u_off, n_unmapped, 0, false}, ms{mapped, m_off, n_mapped, n_unmapped, true};
  Fail fl;
  const fgb_status st = link::guarded(hi.last_error, "fgb_zipper_records", [&]() -> fgb_status {
    hi.kept->clear();
    return zipper_impl(hi, *opt, us, ms, last_call != 0, mapped_consumed, stats, &fl);
  });
  if (st != FGB_OK) {
    if (fl.bad != kNone) {
      if (bad_record) *bad_record = fl.bad;
      *hi.last_error = "fgb_zipper_records: record " + std::to_string(fl.bad) + " " + fl.why;
    }
    hi.kept->clear();
    std::fill(stats, stats + FGB_ZIPPER_NSTATS, 0);
    *mapped_consumed = 0;
    return st;
  }
  *out = hi.kept->data();
  *out_len = hi.kept->size();
  return FGB_OK;
}

fgb_status fgb_host_zipper_records(const fgb_zipper_options* opt, const uint8_t* unmapped, const uint64_t* u_off,
                                   uint64_t n_unmapped, const uint8_t* mapped, const uint64_t* m_off, uint64_t n_mapped,
                                   int last_call, uint8_t** out, uint64_t* out_len, uint64_t* mapped_consumed,
                                   uint64_t stats[FGB_ZIPPER_NSTATS], uint64_t* bad_record) {
  if (bad_record) *bad_record = kNone;
  if (!args_ok(opt, unmapped, u_off, n_unmapped, mapped, m_off, n_mapped, out, out_len, mapped_consumed, stats))
    return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  *out_len = 0;
  *mapped_consumed = 0;
  std::fill(stats, stats + FGB_ZIPPER_NSTATS, 0);
  std::vector<uint8_t> names;
  if (!tag_lists(*opt, &names)) return FGB_ERR_INVALID_ARG;
  names.resize(names.size() + 2);
  const Stream us{unmapped, u_off, n_unmapped, 0, false}, ms{mapped, m_off, n_mapped, n_unmapped, true};
  Join J;
  Fail fl;
  if (!join(*opt, us, ms, last_call != 0, &J, &fl)) {
    if (bad_record) *bad_record = fl.bad;
    return fl.st;
  }
  const zip::Sets sets = sets_at(*opt, names.data());
  const uint64_t n = J.zr.size(), t = std::max<uint32_t>(opt->n_threads, 1);
  const bool skip = opt->skip_pa_tags != 0;
  auto sum = [](uint32_t v) { return v; };
  struct {
    uint32_t operator()(uint32_t v) const { return v; }
    uint32_t last(uint32_t x) const { return x; }
  } prefix;
  std::vector<uint64_t> off(n + 1, 0);
  fgb_umi::parallel_for(t, opt->n_threads, [&](uint64_t w) {
    for (uint64_t i = n * w / t, e = n * (w + 1) / t; i < e; ++i) {
      const zip::ZRec& z = J.zr[i];
      off[i + 1] = 4 + (z.kind == zip::kPass ? u_off[z.src + 1] - u_off[z.src]
                                             : zip::out_size(zip::plan(z, unmapped, u_off, mapped, m_off, sets, skip,
                                                                       0, 1, sum), sets));
    }
  });
  for (uint64_t i = 0; i < n; ++i) off[i + 1] += off[i];
  uint8_t* buf = static_cast<uint8_t*>(std::malloc(std::max<uint64_t>(off[n], 1)));
  if (!buf) return FGB_ERR_NOMEM;
  fgb_umi::parallel_for(t, opt->n_threads, [&](uint64_t w) {
    for (uint64_t i = n * w / t, e = n * (w + 1) / t; i < e; ++i) {
      const zip::ZRec& z = J.zr[i];
      uint8_t* d = buf + off[i];
      const uint32_t bs = static_cast<uint32_t>(off[i + 1] - off[i] - 4);
      std::memcpy(d, &bs, 4);
      if (z.kind == zip::kPass) std::memcpy(d + 4, unmapped + u_off[z.src], bs);
      else zip::write(d + 4, zip::plan(z, unmapped, u_off, mapped, m_off, sets, skip, 0, 1, sum), sets, 0, 1, prefix);
    }
  });
  *out = buf;
  *out_len = off[n];
  *mapped_consumed = J.consumed;
  stats[FGB_ZSTAT_MERGED] = J.merged;
  stats[FGB_ZSTAT_UNMAPPED_ONLY] = J.passed;
  stats[FGB_ZSTAT_EXCLUDED] = J.excluded;
  stats[FGB_ZSTAT_RECORDS_OUT] = n;
  return FGB_OK;
}

void fgb_host_free_buffer(void* p) { std::free(p); }

fgb_status fgb_zipper_last_timing(const fgb_handle* h, double ms[6]) {
  if (!h || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, link::info(const_cast<fgb_handle*>(h), link::Command::kZipper).timing, 6 * sizeof(double));
  return FGB_OK;
}

}  // extern "C"
