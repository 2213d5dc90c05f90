// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.  A stand-in for the GPU engine behind the record-level callers,
// so that the callers' flush side (tile planning, submit, record assembly, filter template rule, threaded
// assembly) can run on a machine without a GPU and under sanitizers.  It defines the engine entry points
// caller_host.cpp calls -- fgb_create / fgb_submit / fgb_submit_ex / fgb_wait / fgb_host_alloc ... -- on
// top of the CPU oracle (oracle/fgumi_oracle.cpp), and is linked ONLY into tests/native/caller_e2e.cpp
// (the executable's definitions take precedence over the library's).  The product has no CPU path: libfgumi_b200.so never contains or loads any of this.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/fgumi_b200.h"

extern "C" {
// oracle/oracle_capi.cpp
struct OrcUnit { uint64_t out_off; uint32_t read_begin; uint32_t cons_len; };
int orc_simplex_batch(uint64_t n_units, const OrcUnit* units, const uint64_t* reads, const uint8_t* bases,
                      const uint8_t* quals, uint8_t pre, uint8_t post, uint32_t min_reads, uint8_t min_cons_q,
                      uint8_t* out_base, uint8_t* out_qual, uint16_t* out_depth, uint16_t* out_errors,
                      uint32_t* cons_len_out, int n_threads);
int orc_duplex_job(const uint8_t* ab, const uint8_t* aq, const uint16_t* ad, const uint16_t* ae, size_t la,
                   const uint8_t* bb, const uint8_t* bq, const uint16_t* bd, const uint16_t* be, size_t lb,
                   const uint8_t* const* src_bases, const size_t* src_len, long n_source, uint8_t* ob,
                   uint8_t* oq, uint16_t* oe, size_t* out_len);
int orc_codec_job(const uint8_t* ab, const uint8_t* aq, const uint16_t* ad, const uint16_t* ae, size_t la,
                  const uint8_t* bb, const uint8_t* bq, const uint16_t* bd, const uint16_t* be, size_t lb,
                  int r1_neg, int r2_neg, size_t cons_len, int ss_qual, int outer_qual, size_t outer_len,
                  size_t max_dis, double max_rate, uint8_t* ob, uint8_t* oq, uint16_t* od, uint16_t* oe,
                  uint64_t* duplex_bases, uint64_t* disagreements);
}

struct fgb_handle { fgb_params p; };

namespace {

// bench.py's record-level CPU baseline builds this file with -DFGB_MOCK_THREADS: the vote and the row building
// then run on FGB_CPU_THREADS threads (default 1), like the caller's own host phases.
int mock_threads() {
#ifdef FGB_MOCK_THREADS
  const char* e = std::getenv("FGB_CPU_THREADS");
  const int n = e ? std::atoi(e) : 1;
  return n > 0 ? n : 1;
#else
  return 1;
#endif
}

fgb_status vote(const fgb_handle* h, const fgb_batch* in, const fgb_columns* out) {
  static_assert(sizeof(OrcUnit) == sizeof(fgb_unit), "unit layout");
  if (in->n_units == 0) return FGB_OK;
  int rc = orc_simplex_batch(in->n_units, reinterpret_cast<const OrcUnit*>(in->units),
                             reinterpret_cast<const uint64_t*>(in->reads), in->bases, in->quals,
                             h->p.error_rate_pre_umi, h->p.error_rate_post_umi, h->p.min_reads,
                             h->p.min_consensus_base_quality, out->base, out->qual, out->depth, out->errors,
                             nullptr, mock_threads());
  return rc == 0 ? FGB_OK : FGB_ERR_INVALID_ARG;
}

// filter_kernel.cuh restated on the host columns (filter.rs:453-471, 650-696, commands/filter.rs:909-929)
void filter_units(const fgb_batch* in, const fgb_columns* c, const fgb_filter_params& fp, uint8_t* status,
                  uint32_t* masked) {
  for (uint64_t u = 0; u < in->n_units; ++u) {
    const fgb_unit& un = in->units[u];
    const uint32_t L = un.cons_len;
    if (L == 0) { status[u] = FGB_FILTER_NO_RECORD; if (masked) masked[u] = 0; continue; }
    uint32_t maxd = 0, ncount = 0, newly = 0;
    uint64_t td = 0, te = 0, qsum = 0;
    for (uint32_t p = 0; p < L; ++p) {
      const uint64_t o = un.out_off + p;
      uint32_t b = c->base[o], q = c->qual[o];
      const uint32_t d = c->depth[o], e = c->errors[o];
      maxd = std::max(maxd, d); td += d; te += e;
      const uint32_t dt = fp.per_base_tags ? std::min(d, 32767u) : 0u, et = fp.per_base_tags ? std::min(e, 32767u) : 0u;
      const bool mask = (fp.min_base_quality >= 0 && q < static_cast<uint32_t>(fp.min_base_quality)) || dt < fp.min_reads ||
                        (dt > 0 && static_cast<double>(et) / static_cast<double>(dt) > fp.max_base_error_rate);
      if (mask) { newly += (b != 'N'); b = 'N'; q = 2; c->base[o] = 'N'; c->qual[o] = 2; }
      if (b == 'N') ++ncount; else qsum += q;
    }
    uint32_t st = FGB_FILTER_PASS;
    const float ce = td == 0 ? 0.0f : static_cast<float>(te) / static_cast<float>(td);
    if (maxd < fp.min_reads) st = FGB_FILTER_INSUFFICIENT_READS;
    else if (static_cast<double>(ce) > fp.max_read_error_rate) st = FGB_FILTER_EXCESSIVE_ERROR_RATE;
    else {
      const uint32_t non_n = L - ncount;
      const double mean = non_n ? static_cast<double>(qsum) / static_cast<double>(non_n) : 0.0;
      if (fp.min_mean_base_quality >= 0.0 && mean < fp.min_mean_base_quality) st = FGB_FILTER_LOW_MEAN_QUALITY;
      else if (fp.max_no_call_fraction >= 1.0) { if (static_cast<double>(ncount) > fp.max_no_call_fraction) st = FGB_FILTER_TOO_MANY_NO_CALLS; }
      else if (static_cast<double>(ncount) / static_cast<double>(L) > fp.max_no_call_fraction) st = FGB_FILTER_TOO_MANY_NO_CALLS;
    }
    status[u] = static_cast<uint8_t>(st);
    if (masked) masked[u] = newly;
  }
}

}  // namespace

extern "C" {

fgb_status fgb_create(int device, const fgb_params* params, fgb_handle** out) {
  if (!params || !out || device < 0) return FGB_ERR_INVALID_ARG;
  *out = new fgb_handle{*params};
  return FGB_OK;
}
void fgb_destroy(fgb_handle* h) { delete h; }
size_t fgb_last_error(const fgb_handle*, char* buf, size_t n) { if (buf && n) buf[0] = 0; return 0; }
fgb_status fgb_wait(fgb_handle*) { return FGB_OK; }
fgb_status fgb_host_alloc(void** p, size_t bytes) { *p = std::malloc(bytes ? bytes : 1); return *p ? FGB_OK : FGB_ERR_NOMEM; }
void fgb_host_free(void* p) { std::free(p); }
uint32_t fgb_engine_caps(void) { return 0; }        // no device record assembly here: the callers assemble on the host
int fgb_host_is_pinned(const void*) { return std::getenv("FGB_MOCK_PINNED") != nullptr; }   // lets the CPU harness take the zero-copy path

fgb_status fgb_submit(fgb_handle* h, const fgb_batch* in, const fgb_columns* out) { return vote(h, in, out); }

static void run_duplex_jobs(const fgb_batch* in, const fgb_columns* ss, const fgb_duplex_job* jobs, uint64_t n_jobs,
                            const fgb_duplex_out* out);
static void run_codec_jobs(const fgb_batch* in, const fgb_columns* ss, const fgb_codec_job* jobs, uint64_t n_jobs,
                           const fgb_codec_params* cp, const fgb_codec_out* out);

// FGB_IN_RECORDS restated on the host (unpack_kernels.cuh unpack_records_kernel): row position p is raw base p
// (forward) or l_seq - 1 - p complemented (reverse); q < min_q -> (N, Q2); row padding is zero.
void build_rows(const fgb_batch* in, const fgb_record_columns* rc, std::vector<uint8_t>* bases, std::vector<uint8_t>* quals) {
  static const char* kF = "=ACMGRSVTWYHKDBN";
  static const char* kC = "=TGMCRSVAWYHKDBN";
  bases->assign(in->n_bytes + 16, 0);
  quals->assign(in->n_bytes + 16, 0);
  const int T = mock_threads();
  auto range = [&](uint64_t r_lo, uint64_t r_hi) {
  for (uint64_t r = r_lo; r < r_hi; ++r) {
    const fgb_raw_read& rr = rc->raw_reads[r];
    const uint64_t off = FGB_READ_OFF(in->reads[r]);
    const uint32_t len = FGB_READ_LEN(in->reads[r]);
    const uint8_t* seq = rc->records + rr.src_off;
    const uint8_t* q = seq + (static_cast<uint64_t>(rr.raw_len) + 1) / 2;
    const bool rev = rr.flags & FGB_RAW_REVERSE;
    for (uint32_t p = 0; p < len; ++p) {
      const uint32_t i = rev ? rr.raw_len - 1 - p : p;
      const uint32_t nib = (i & 1) ? (seq[i >> 1] & 15u) : (seq[i >> 1] >> 4);
      uint8_t b = static_cast<uint8_t>(rev ? kC[nib] : kF[nib]), qq = q[i];
      if (qq < rc->min_input_base_quality) { b = 'N'; qq = 2; }
      (*bases)[off + p] = b; (*quals)[off + p] = qq;
    }
  }
  };
  if (T <= 1) { range(0, in->n_reads); return; }
  std::vector<std::thread> th;
  for (int t = 0; t < T; ++t) th.emplace_back(range, in->n_reads * t / T, in->n_reads * (t + 1) / T);
  for (auto& x : th) x.join();
}

// The device's overlapping-bases pre-pass (unpack_kernels.cuh overlap_kernel) restated on a host copy of the blob.
void apply_overlap_runs(std::vector<uint8_t>* blob, const fgb_submit_options* opt) {
  uint64_t st[4] = {0, 0, 0, 0};
  for (uint64_t k = 0; k < opt->n_overlap_runs; ++k) {
    const fgb_overlap_run& r = opt->overlap_runs[k];
    uint8_t* s1 = blob->data() + r.seq1_off; uint8_t* q1 = s1 + (static_cast<uint64_t>(r.l_seq1) + 1) / 2;
    uint8_t* s2 = blob->data() + r.seq2_off; uint8_t* q2 = s2 + (static_cast<uint64_t>(r.l_seq2) + 1) / 2;
    for (uint32_t t = 0; t < r.len; ++t) {
      const uint32_t i1 = r.o1 + t, i2 = r.o2 + t;
      const uint32_t c1 = (i1 & 1) ? (s1[i1 >> 1] & 15u) : (s1[i1 >> 1] >> 4), c2 = (i2 & 1) ? (s2[i2 >> 1] & 15u) : (s2[i2 >> 1] >> 4);
      if (c1 == 15 || c2 == 15) continue;
      ++st[0];
      const uint32_t x = q1[i1], y = q2[i2];
      uint32_t oc1 = c1, oc2 = c2, oq1 = x, oq2 = y;
      if (c1 == c2) {
        ++st[1];
        if (opt->overlap_agreement == FGB_OVERLAP_AGREE_PASS_THROUGH) continue;
        const uint32_t nq = opt->overlap_agreement == FGB_OVERLAP_AGREE_CONSENSUS ? std::min(x + y, 93u) : std::max(x, y);
        oq1 = oq2 = nq;
        if (nq != x || nq != y) ++st[3];
      } else {
        ++st[2];
        if (opt->overlap_disagreement == FGB_OVERLAP_DISAGREE_CONSENSUS) {
          uint32_t code = 15, q = 2;
          if (x > y) { code = c1; q = std::max(x - y, 2u); } else if (y > x) { code = c2; q = std::max(y - x, 2u); }
          oc1 = oc2 = code; oq1 = oq2 = q; st[3] += 2;
        } else if (opt->overlap_disagreement == FGB_OVERLAP_DISAGREE_MASK_BOTH || x == y) {
          oc1 = oc2 = 15; oq1 = oq2 = 2; st[3] += 2;
        } else if (x < y) { oc1 = 15; oq1 = 2; ++st[3]; }
        else { oc2 = 15; oq2 = 2; ++st[3]; }
      }
      auto put = [](uint8_t* s, uint32_t i, uint32_t c) { s[i >> 1] = static_cast<uint8_t>((i & 1) ? ((s[i >> 1] & 0xF0u) | c) : ((c << 4) | (s[i >> 1] & 0x0Fu))); };
      put(s1, i1, oc1); put(s2, i2, oc2);
      q1[i1] = static_cast<uint8_t>(oq1); q2[i2] = static_cast<uint8_t>(oq2);
    }
  }
  if (opt->overlap_stats) for (int i = 0; i < 4; ++i) opt->overlap_stats[i] += st[i];
}

fgb_status fgb_submit_ex(fgb_handle* h, const fgb_batch* in, const fgb_columns* out, const fgb_submit_options* opt) {
  if (!opt) return vote(h, in, out);
  if (opt->input_format != FGB_IN_BYTES && opt->input_format != FGB_IN_RECORDS) return FGB_ERR_INVALID_ARG;   // what the callers use
  fgb_batch b = *in;
  std::vector<uint8_t> rb, rq;
  if (opt->input_format == FGB_IN_RECORDS) {
    if (!opt->records) return FGB_ERR_INVALID_ARG;
    fgb_record_columns rcols = *opt->records;
    std::vector<uint8_t> blob;
    if (opt->n_overlap_runs) {
      blob.assign(rcols.records, rcols.records + rcols.n_bytes);
      apply_overlap_runs(&blob, opt);
      rcols.records = blob.data();
    }
    build_rows(in, &rcols, &rb, &rq);
    b.bases = rb.data(); b.quals = rq.data();
  }
  const bool narrow = opt->output_format == FGB_OUT_U8;
  std::vector<uint16_t> d16, e16;
  fgb_columns cols = *out;
  if (narrow) { d16.assign(in->n_out + 8, 0); e16.assign(in->n_out + 8, 0); cols.depth = d16.data(); cols.errors = e16.data(); }
  fgb_status st = vote(h, &b, &cols);
  if (st != FGB_OK) return st;
  if (opt->filter) {
    if (!opt->unit_status) return FGB_ERR_INVALID_ARG;
    filter_units(&b, &cols, *opt->filter, opt->unit_status, opt->unit_masked);
  }
  if (opt->n_duplex_jobs) run_duplex_jobs(&b, &cols, opt->duplex_jobs, opt->n_duplex_jobs, opt->duplex_out);
  if (opt->n_codec_jobs) run_codec_jobs(&b, &cols, opt->codec_jobs, opt->n_codec_jobs, opt->codec_params, opt->codec_out);
  if (narrow) {
    uint8_t* d8 = reinterpret_cast<uint8_t*>(out->depth);
    uint8_t* e8 = reinterpret_cast<uint8_t*>(out->errors);
    for (uint64_t i = 0; i < in->n_out; ++i) { d8[i] = static_cast<uint8_t>(d16[i]); e8[i] = static_cast<uint8_t>(e16[i]); }
  }
  return FGB_OK;
}

static void run_duplex_jobs(const fgb_batch* in, const fgb_columns* ss, const fgb_duplex_job* jobs, uint64_t n_jobs,
                            const fgb_duplex_out* out) {
  std::vector<const uint8_t*> src; std::vector<size_t> len;
  for (uint64_t j = 0; j < n_jobs; ++j) {
    const fgb_unit &ua = in->units[jobs[j].unit_a], &ub = in->units[jobs[j].unit_b];
    src.clear(); len.clear();
    for (uint32_t u : {jobs[j].unit_a, jobs[j].unit_b})
      for (uint32_t r = in->units[u].read_begin; r < in->units[u + 1].read_begin; ++r) {
        src.push_back(in->bases + FGB_READ_OFF(in->reads[r])); len.push_back(FGB_READ_LEN(in->reads[r]));
      }
    size_t n = 0;
    const uint64_t o = jobs[j].out_off;
    int status = orc_duplex_job(ss->base + ua.out_off, ss->qual + ua.out_off, ss->depth + ua.out_off, ss->errors + ua.out_off,
                                ua.cons_len, ss->base + ub.out_off, ss->qual + ub.out_off, ss->depth + ub.out_off,
                                ss->errors + ub.out_off, ub.cons_len, src.data(), len.data(), static_cast<long>(src.size()),
                                out->base + o, out->qual + o, out->errors + o, &n);
    if (out->status) out->status[j] = static_cast<uint8_t>(status);
  }
}

static void run_codec_jobs(const fgb_batch* in, const fgb_columns* ss, const fgb_codec_job* jobs, uint64_t n_jobs,
                           const fgb_codec_params* cp, const fgb_codec_out* out) {
  for (uint64_t j = 0; j < n_jobs; ++j) {
    const fgb_codec_job& job = jobs[j];
    const fgb_unit &ua = in->units[job.unit_a], &ub = in->units[job.unit_b];
    const bool r1_neg = job.rc_a != 0;
    const bool r2_neg = job.pad_b_left > 0 ? true : (job.len > ub.cons_len ? false : !r1_neg);   // the padding side of R2
    uint64_t dup = 0, dis = 0;
    const uint64_t o = job.out_off;
    int status = orc_codec_job(ss->base + ua.out_off, ss->qual + ua.out_off, ss->depth + ua.out_off, ss->errors + ua.out_off,
                               ua.cons_len, ss->base + ub.out_off, ss->qual + ub.out_off, ss->depth + ub.out_off,
                               ss->errors + ub.out_off, ub.cons_len, r1_neg, r2_neg, job.len, cp->single_strand_qual,
                               cp->outer_bases_qual, cp->outer_bases_length, cp->max_duplex_disagreements,
                               cp->max_duplex_disagreement_rate, out->cols.base + o, out->cols.qual + o,
                               out->cols.depth + o, out->cols.errors + o, &dup, &dis);
    if (out->status) out->status[j] = static_cast<uint8_t>(status);
    if (out->disagreements) out->disagreements[j] = static_cast<uint32_t>(dis);
    if (out->duplex_bases) out->duplex_bases[j] = static_cast<uint32_t>(dup);
  }
}

}  // extern "C"
