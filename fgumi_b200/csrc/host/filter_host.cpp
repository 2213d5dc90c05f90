// `fgumi filter --ref` from raw BAM records (src/lib/commands/filter.rs:550-905): the resident reference
// (fgb_reference_*) and the driver of the device filter (fgb_filter_records).  The host does the header-level work --
// record checks, the @SQ-to-contig table, QNAME runs and Template::from_records order -- and cuts the call into runs of
// whole templates that fit a device budget; each run crosses the link through page-locked staging and is filtered by
// the kernels of ../filter_records_kernels.cuh behind filter_device.h.  Restated in tests/filter_oracle.py.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "bam.h"
#include "filter_device.h"
#include "group_rules.h"
#include "record_link.h"
#include "umi_host.h"

struct fgb_reference {
  int device = -1;
  std::vector<std::string> names;
  std::vector<uint64_t> off, len;                      // each contig's place in the genome array
  std::unordered_map<std::string, uint64_t> index;     // name -> contig (the later of two with one name)
  uint8_t* d_seq = nullptr;
  uint64_t* d_off = nullptr;
  uint64_t* d_len = nullptr;
};

namespace {

namespace dev = fgb::filterdev;
namespace link = fgb::link;
using link::ms_since;
constexpr uint64_t kNone = UINT64_MAX;

// The sequential FASTA reader's records (reference.rs:229-244): name up to the first whitespace after '>', sequence
// = the following lines up to the next '>' with \n / \r\n removed.  false: not a FASTA image.
bool parse_fasta(const uint8_t* f, size_t n, fgb_reference* r, std::vector<uint8_t>* seq) {
  if (n >= 2 && f[0] == 0x1f && f[1] == 0x8b) return false;   // gzip / BGZF
  bool open = false;
  seq->reserve(n);   // the sequence is at most the image: no doubling growth over a 3 GB genome
  for (size_t p = 0; p < n;) {
    const uint8_t* nl = static_cast<const uint8_t*>(std::memchr(f + p, '\n', n - p));
    const size_t e = nl ? static_cast<size_t>(nl - f) : n;
    size_t le = e;
    if (le > p && f[le - 1] == '\r') --le;
    if (le > p && f[p] == '>') {
      size_t ne = p + 1;
      while (ne < le && f[ne] != ' ' && f[ne] != '\t') ++ne;
      if (open) r->len.push_back(seq->size() - r->off.back());
      r->names.emplace_back(reinterpret_cast<const char*>(f + p + 1), ne - p - 1);
      r->off.push_back(seq->size());
      open = true;
    } else if (le > p) {
      if (!open) return false;
      seq->insert(seq->end(), f + p, f + le);
    }
    p = e + 1;
  }
  if (open) r->len.push_back(seq->size() - r->off.back());
  for (uint64_t i = 0; i < r->names.size(); ++i) r->index[r->names[i]] = i;
  return true;
}

// The checks that need only a record's fixed fields (regenerate_alignment_tags_raw's, alignment_tags.rs:259-291, and
// the command's no-reference check, commands/filter.rs:758-768): "" or why record i fails the call; *layout: the
// record is cut short.
std::string host_check(const uint8_t* r, uint64_t len, bool have_ref, uint64_t n_sq, bool* layout) {
  *layout = true;
  if (len < 32) return "is shorter than 32 bytes";
  const fgb::bam::View v(r, len);
  const uint64_t need = 32ull + v.l_read_name() + 4ull * v.n_cigar() + (v.l_seq() + 1ull) / 2 + v.l_seq();
  if (need > len) return "is truncated: its name, CIGAR, sequence or qualities run past its end";
  *layout = false;
  if (v.flags() & fgb::bam::kUnmapped) return "";
  if (!have_ref) return "is mapped: --ref is required when filtering mapped reads to keep NM/UQ/MD tags consistent";
  if (v.ref_id() < 0) return "";
  if (static_cast<uint64_t>(v.ref_id()) >= n_sq) return "has a reference sequence ID not found in the header";
  if (v.pos() < 0) return "has an invalid alignment start position " + std::to_string(v.pos());
  return "";
}

fgb_status filter_impl(const link::HandleInfo& hi, const fgb_record_filter_options& o, const fgb_reference* ref,
                       std::string_view header, const uint8_t* records, const uint64_t* rec_off, uint64_t n,
                       uint64_t* stats, uint64_t* bad_record) {
  auto fail = [&](cudaError_t e, const char* what) { return link::fail(hi.last_error, "fgb_filter_records", e, what); };
  link::Resources r(hi.stream, o.n_threads);
  double* tm = hi.timing;
  auto t_host = std::chrono::steady_clock::now();
  // header-level checks: the first failing record in input order
  const std::vector<std::string> sq = link::sq_names(header);
  uint64_t hb = n;
  std::string herr;
  fgb_status hst = FGB_OK;
  {
    const uint64_t t = std::max<uint32_t>(o.n_threads, 1);
    std::vector<uint64_t> first(t, n);
    fgb_umi::parallel_for(t, o.n_threads, [&](uint64_t w) {
      bool layout;
      for (uint64_t i = n * w / t, e = n * (w + 1) / t; i < e; ++i)
        if (rec_off[i + 1] < rec_off[i] ||
            !host_check(records + rec_off[i], rec_off[i + 1] - rec_off[i], ref != nullptr, sq.size(), &layout).empty()) {
          first[w] = i;
          break;
        }
    });
    hb = *std::min_element(first.begin(), first.end());
    if (hb < n) {
      bool layout = true;
      herr = rec_off[hb + 1] < rec_off[hb] ? std::string("is shorter than 32 bytes")
                                          : host_check(records + rec_off[hb], rec_off[hb + 1] - rec_off[hb],
                                                       ref != nullptr, sq.size(), &layout);
      hst = layout ? FGB_ERR_LAYOUT : FGB_ERR_INVALID_ARG;
    }
  }
  // templates (Template::from_records order) over the records before the first bad one, so that a second primary R1
  // or R2 before it is found first; order[] holds the output positions' records, tpl[] each template's first position
  std::vector<uint32_t> order, tpl{0};
  order.reserve(hb);
  tpl.reserve(hb + 1);
  if (o.filter_by_template) {
    std::vector<uint64_t> lists[4], ord;
    for (uint64_t i = 0; i < hb;) {
      const fgb::bam::View vi(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
      const std::string_view name = fgb::grp::read_name(vi);
      uint64_t j = i + 1;
      while (j < hb && fgb::grp::read_name(fgb::bam::View(records + rec_off[j], rec_off[j + 1] - rec_off[j])) == name) ++j;
      int64_t r1, r2;
      uint64_t dup;
      ord.clear();
      const std::string err = fgb::grp::template_order(
          i, j, [&](uint64_t k) { return fgb::bam::rd16(records + rec_off[k] + 14); }, name, lists, &ord, &r1, &r2, &dup);
      if (!err.empty()) {
        hb = dup;
        herr = err;
        hst = FGB_ERR_INVALID_ARG;
        break;
      }
      for (uint64_t k : ord) order.push_back(static_cast<uint32_t>(k));
      tpl.push_back(static_cast<uint32_t>(order.size()));
      i = j;
    }
  }
  if (hb < n || !o.filter_by_template) {   // each record alone (the call fails anyway when hb < n)
    order.resize(hb);
    tpl.resize(hb + 1);
    for (uint64_t i = 0; i < hb; ++i) order[i] = static_cast<uint32_t>(i);
    for (uint64_t i = 0; i <= hb; ++i) tpl[i] = static_cast<uint32_t>(i);
  }
  const uint64_t n_tpl = tpl.size() - 1;
  // the @SQ -> FASTA contig table
  std::vector<int32_t> ctg(std::max<size_t>(sq.size(), 1), -1);
  if (ref)
    for (size_t s = 0; s < sq.size(); ++s) {
      const auto it = ref->index.find(sq[s]);
      if (it != ref->index.end()) ctg[s] = static_cast<int32_t>(it->second);
    }
  cudaError_t e = cudaSetDevice(hi.device);
  if (e != cudaSuccess) return fail(e, "cudaSetDevice");
  // runs of whole templates: input bytes, their edited copies in both streams and ~100 bytes of tables per record
  uint64_t budget;
  if ((e = link::device_budget(o.device_bytes, &budget)) != cudaSuccess) return fail(e, "cudaMemGetInfo");
  std::vector<uint64_t> run_tpl{0};
  uint64_t max_n = 0, max_bytes = 0;
  for (uint64_t t = 0; t < n_tpl;) {
    uint64_t u = t + 1;   // at least one template per run
    const uint64_t r0 = tpl[t];
    while (u < n_tpl) {
      const uint64_t recs = tpl[u + 1] - r0, bytes = rec_off[tpl[u + 1]] - rec_off[r0];
      if (3 * bytes + recs * 160 > budget || recs >= INT32_MAX / 2) break;
      ++u;
    }
    max_n = std::max<uint64_t>(max_n, tpl[u] - r0);
    max_bytes = std::max(max_bytes, rec_off[tpl[u]] - rec_off[r0]);
    run_tpl.push_back(u);
    t = u;
  }
  const uint64_t n_runs = run_tpl.size() - 1;
  uint8_t *d_rec = nullptr, *d_temp = nullptr, *d_kept = nullptr, *d_rej = nullptr;
  uint64_t *d_off, *d_ks, *d_rs, *d_koff, *d_roff, *d_ctg_off = ref ? ref->d_off : nullptr,
                                                   *d_ctg_len = ref ? ref->d_len : nullptr;
  uint32_t *d_order, *d_tpl;
  int32_t* d_ctg;
  fgb::FRec* d_fr;
  unsigned long long* d_cnt;
  uint64_t cap_kept = 0, cap_rej = 0;
  size_t t_scan = 0;
  const uint32_t mn = static_cast<uint32_t>(max_n);
  if ((e = dev::offsets(nullptr, &t_scan, nullptr, nullptr, mn, false, nullptr, nullptr, nullptr, nullptr, hi.stream)))
    return fail(e, "CUB temp storage");
  if ((e = r.alloc(&d_rec, max_bytes + 16)) || (e = r.alloc(&d_off, max_n + 1)) || (e = r.alloc(&d_fr, max_n)) ||
      (e = r.alloc(&d_order, max_n)) || (e = r.alloc(&d_tpl, max_n + 1)) || (e = r.alloc(&d_ks, max_n + 1)) ||
      (e = r.alloc(&d_rs, max_n + 1)) || (e = r.alloc(&d_koff, max_n + 1)) || (e = r.alloc(&d_roff, max_n + 1)) ||
      (e = r.alloc(&d_ctg, ctg.size())) || (e = r.alloc(&d_cnt, 3)) || (e = r.alloc(&d_temp, t_scan + 16)))
    return fail(e, "cudaMalloc");
  // FGB_FILTER_STAGE_BYTES (at least 4096) lowers the staging buffers' size, so that small inputs cross several chunks
  uint64_t stage_cap = link::kStageBytes;
  if (const char* env = std::getenv("FGB_FILTER_STAGE_BYTES"))
    stage_cap = std::max<uint64_t>(4096, std::min<uint64_t>(link::kStageBytes, std::strtoull(env, nullptr, 10)));
  const char* what;
  if ((e = r.open(std::min<uint64_t>(stage_cap, std::max<uint64_t>(max_bytes + 64, (max_n + 1) * 8)), &what)))
    return fail(e, what);
  if ((e = cudaMemcpy(d_ctg, ctg.data(), ctg.size() * 4, cudaMemcpyHostToDevice))) return fail(e, "cudaMemcpy");
  tm[5] += ms_since(t_host);   // host work: the checks, templates and contig table, and every allocation of the call
  fgb::FilterCfg cfg{};
  const fgb_duplex_filter_params& p = o.filter;
  cfg.cc = {p.cc.min_reads, p.cc.max_read_error_rate, p.cc.max_base_error_rate};
  cfg.ab = {p.ab_min_reads, p.ab_max_read_error_rate, p.ab_max_base_error_rate};
  cfg.ba = {p.ba_min_reads, p.ba_max_read_error_rate, p.ba_max_base_error_rate};
  cfg.min_mean_q = p.cc.min_mean_base_quality;
  cfg.max_no_call = p.cc.max_no_call_fraction;
  cfg.min_bq = p.cc.min_base_quality;
  cfg.require_ss = p.require_ss_agreement;
  cfg.reverse_tags = o.reverse_per_base_tags;
  cfg.regenerate = ref != nullptr;
  std::vector<uint8_t>& kept = *hi.kept;
  std::vector<uint8_t>& rej = *hi.rejects;
  const bool track = o.track_rejects != 0;
  uint64_t masked = 0, passed = 0;
  std::vector<uint32_t> lorder, ltpl;
  for (uint64_t x = 0; x < n_runs; ++x) {
    t_host = std::chrono::steady_clock::now();
    const uint64_t t0 = run_tpl[x], t1 = run_tpl[x + 1], p0 = tpl[t0], nr64 = tpl[t1] - p0;
    // the run's records are the input range [rb, rb + nr) (templates are consecutive QNAME runs)
    uint64_t rb = n;
    for (uint64_t q = p0; q < p0 + nr64; ++q) rb = std::min<uint64_t>(rb, order[q]);
    const uint32_t nr = static_cast<uint32_t>(nr64);
    lorder.resize(nr);
    ltpl.resize(t1 - t0 + 1);
    for (uint64_t q = 0; q < nr; ++q) lorder[q] = static_cast<uint32_t>(order[p0 + q] - rb);
    for (uint64_t t = t0; t <= t1; ++t) ltpl[t - t0] = static_cast<uint32_t>(tpl[t] - p0);
    tm[5] += ms_since(t_host);
    const uint64_t base = rec_off[rb], bytes = rec_off[rb + nr] - base;
    auto t_up = std::chrono::steady_clock::now();
    const unsigned long long init[3] = {0, 0, ~0ull};
    if ((e = r.upload(d_rec, records + base, bytes)) || (e = r.upload(d_off, rec_off + rb, (nr64 + 1) * 8)) ||
        (e = r.upload(d_order, lorder.data(), nr64 * 4)) || (e = r.upload(d_tpl, ltpl.data(), ltpl.size() * 4)) ||
        (e = cudaMemcpyAsync(d_cnt, init, sizeof(init), cudaMemcpyHostToDevice, hi.stream)) ||
        (e = cudaStreamSynchronize(hi.stream)))
      return fail(e, "upload");
    tm[0] += ms_since(t_up);
    uint64_t tot[2];
    unsigned long long cnt[3];
    size_t tb = t_scan + 16;
    if ((e = cudaEventRecord(r.ev[0], hi.stream)) ||
        (e = dev::pass1(d_rec, d_off, base, nr, cfg, d_ctg, d_ctg_off, d_ctg_len, ref ? ref->d_seq : nullptr, rb, d_fr,
                        d_cnt + 2, d_cnt, hi.sm_count, hi.stream)) ||
        (e = cudaEventRecord(r.ev[1], hi.stream)) ||
        (e = dev::decide(d_fr, d_order, d_tpl, static_cast<uint32_t>(t1 - t0), o.filter_by_template != 0, d_cnt,
                         hi.stream)) ||
        (e = dev::offsets(d_temp, &tb, d_fr, d_order, nr, track, d_ks, d_rs, d_koff, d_roff, hi.stream)) ||
        (e = cudaEventRecord(r.ev[2], hi.stream)) ||
        (e = cudaMemcpyAsync(&tot[0], d_koff + nr, 8, cudaMemcpyDeviceToHost, hi.stream)) ||
        (e = cudaMemcpyAsync(&tot[1], d_roff + nr, 8, cudaMemcpyDeviceToHost, hi.stream)) ||
        (e = cudaMemcpyAsync(cnt, d_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, hi.stream)) ||
        (e = cudaStreamSynchronize(hi.stream)))
      return fail(e, "pass 1");
    if (cnt[2] != ~0ull) {   // a device error: before the first host error by construction
      const uint64_t bi = cnt[2] >> 8;
      const uint8_t code = static_cast<uint8_t>(cnt[2] & 0xFF);
      const int32_t rid = fgb::bam::rdi32(records + rec_off[bi]);
      *bad_record = bi;
      *hi.last_error = "fgb_filter_records: record " + std::to_string(bi) + " " +
                       (code == fgb::kErrContig   ? "is aligned to reference sequence '" + sq[rid] + "', which the FASTA lacks"
                        : code == fgb::kErrPastEnd ? "is aligned past the end of reference sequence '" + sq[rid] + "'"
                                                   : std::string("has a CIGAR that consumes more bases than its sequence"));
      kept.clear();
      rej.clear();
      return FGB_ERR_INVALID_ARG;
    }
    masked += cnt[0];
    passed += cnt[1];
    t_host = std::chrono::steady_clock::now();
    if ((e = r.grow(&d_kept, &cap_kept, tot[0] + 16)) || (e = r.grow(&d_rej, &cap_rej, tot[1] + 16)))
      return fail(e, "cudaMalloc");
    tm[5] += ms_since(t_host);
    if ((e = cudaEventRecord(r.ev[3], hi.stream)) ||
        (e = dev::pass2(d_rec, d_off, base, nr, d_fr, d_order, d_koff, d_roff, track, ref ? ref->d_seq : nullptr,
                        d_kept, d_rej, hi.sm_count, hi.stream)) ||
        (e = cudaEventRecord(r.ev[4], hi.stream)) || (e = cudaStreamSynchronize(hi.stream)))
      return fail(e, "pass 2");
    float a = 0, b = 0, c = 0;
    cudaEventElapsedTime(&a, r.ev[0], r.ev[1]);
    cudaEventElapsedTime(&b, r.ev[1], r.ev[2]);
    cudaEventElapsedTime(&c, r.ev[3], r.ev[4]);
    tm[1] += a; tm[2] += b; tm[3] += c;
    auto t_dn = std::chrono::steady_clock::now();
    const uint64_t k0 = kept.size(), j0 = rej.size();
    kept.resize(k0 + tot[0]);
    rej.resize(j0 + tot[1]);
    if ((e = r.download(kept.data() + k0, d_kept, tot[0])) || (e = r.download(rej.data() + j0, d_rej, tot[1])))
      return fail(e, "download");
    tm[4] += ms_since(t_dn);
  }
  if (hb < n) {
    *bad_record = hb;
    *hi.last_error = "fgb_filter_records: record " + std::to_string(hb) + " " + herr;
    kept.clear();
    rej.clear();
    return hst;
  }
  stats[FGB_FSTAT_TOTAL] = n;
  stats[FGB_FSTAT_PASSED] = passed;
  stats[FGB_FSTAT_FAILED] = n - passed;
  stats[FGB_FSTAT_BASES_MASKED] = masked;
  return FGB_OK;
}

}  // namespace

extern "C" {

fgb_status fgb_reference_create(int device, const uint8_t* fasta, size_t len, fgb_reference** out) {
  if (!out || (len && !fasta)) return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  try {
    std::unique_ptr<fgb_reference> r(new fgb_reference());
    std::vector<uint8_t> seq;
    if (!parse_fasta(fasta, len, r.get(), &seq)) return FGB_ERR_INVALID_ARG;
    if (device == FGB_DEVICE_NONE) {   // parsed only: the contig table without the device copy
      *out = r.release();
      return FGB_OK;
    }
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) {
      cudaGetLastError();
      return FGB_ERR_NO_DEVICE;
    }
    r->device = device;
    const size_t nc = std::max<size_t>(r->names.size(), 1);
    cudaError_t e;
    if ((e = cudaSetDevice(device)) || (e = cudaMalloc(&r->d_seq, std::max<size_t>(seq.size(), 1))) ||
        (e = cudaMalloc(&r->d_off, nc * 8)) || (e = cudaMalloc(&r->d_len, nc * 8)) ||
        (!seq.empty() && (e = cudaMemcpy(r->d_seq, seq.data(), seq.size(), cudaMemcpyHostToDevice))) ||
        (!r->off.empty() && (e = cudaMemcpy(r->d_off, r->off.data(), r->off.size() * 8, cudaMemcpyHostToDevice))) ||
        (!r->len.empty() && (e = cudaMemcpy(r->d_len, r->len.data(), r->len.size() * 8, cudaMemcpyHostToDevice)))) {
      cudaGetLastError();
      fgb_reference_destroy(r.release());
      return e == cudaErrorMemoryAllocation ? FGB_ERR_NOMEM : FGB_ERR_CUDA;
    }
    *out = r.release();
    return FGB_OK;
  } catch (const std::bad_alloc&) {
    return FGB_ERR_NOMEM;
  }
}

void fgb_reference_destroy(fgb_reference* r) {
  if (!r) return;
  if (r->device >= 0) {
    cudaSetDevice(r->device);
    cudaFree(r->d_seq);
    cudaFree(r->d_off);
    cudaFree(r->d_len);
  }
  delete r;
}

uint64_t fgb_reference_contigs(const fgb_reference* r) { return r ? r->names.size() : 0; }

fgb_status fgb_reference_contig(const fgb_reference* r, uint64_t i, const char** name, uint64_t* length) {
  if (!r || i >= r->names.size() || !name || !length) return FGB_ERR_INVALID_ARG;
  *name = r->names[i].c_str();
  *length = r->len[i];
  return FGB_OK;
}

fgb_status fgb_filter_records(fgb_handle* h, const fgb_record_filter_options* opt, const fgb_reference* ref,
                              const char* header_text, size_t header_len, const uint8_t* records,
                              const uint64_t* rec_off, uint64_t n_records, const uint8_t** kept, uint64_t* kept_len,
                              const uint8_t** rejects, uint64_t* rejects_len, uint64_t stats[FGB_FILTER_NSTATS],
                              uint64_t* bad_record) {
  if (!h || !opt || !kept || !kept_len || !rejects || !rejects_len || !stats || !rec_off ||
      (n_records && !records) || (header_len && !header_text))
    return FGB_ERR_INVALID_ARG;
  const link::HandleInfo hi = link::info(h, link::Command::kFilter);
  uint64_t bad = kNone;
  std::fill(hi.timing, hi.timing + 6, 0.0);
  std::fill(stats, stats + FGB_FILTER_NSTATS, 0);
  *kept = *rejects = nullptr;
  *kept_len = *rejects_len = 0;
  if (ref && ref->device != hi.device) {
    *hi.last_error = "fgb_filter_records: the reference lives on another device";
    return FGB_ERR_INVALID_ARG;
  }
  if (hi.busy) { *hi.last_error = "fgb_filter_records: a submit has not been waited on"; return FGB_ERR_BUSY; }
  const fgb_status st = link::guarded(hi.last_error, "fgb_filter_records", [&]() -> fgb_status {
    hi.kept->clear();
    hi.rejects->clear();
    return n_records ? filter_impl(hi, *opt, ref, std::string_view(header_text ? header_text : "", header_len), records,
                                   rec_off, n_records, stats, &bad)
                     : FGB_OK;
  });
  if (bad_record) *bad_record = bad;
  if (st != FGB_OK) {
    hi.kept->clear();
    hi.rejects->clear();
    std::fill(stats, stats + FGB_FILTER_NSTATS, 0);
    return st;
  }
  *kept = hi.kept->data();
  *kept_len = hi.kept->size();
  *rejects = hi.rejects->data();
  *rejects_len = hi.rejects->size();
  return FGB_OK;
}

fgb_status fgb_filter_last_timing(const fgb_handle* h, double ms[6]) {
  if (!h || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, link::info(const_cast<fgb_handle*>(h), link::Command::kFilter).timing, 6 * sizeof(double));
  return FGB_OK;
}

}  // extern "C"
