// Record-level callers behind fgb_caller_* (product code): the host side of fgumi's
// VanillaUmiConsensusCaller and DuplexConsensusCaller, re-shaped for GPU batches.
//
//   add_group()  everything the reference does BEFORE the vote, per MI group, packing the surviving
//                SourceRead rows into the SoA batch of include/fgumi_b200.h:
//                  simplex  vanilla_caller.rs:1042-1227 (process_group / process_subgroup)
//                  duplex   duplex_caller.rs:576-630 (strand partition), :1719-1942 (process_group)
//   flush()      one vote (+ strand combine) on the GPU for everything packed, then the record
//                assembly, in input order:
//                  simplex  vanilla_caller.rs:1365-1473 (build_consensus_record_into)
//                  duplex   duplex_caller.rs:1944-2202 (arm selection, min-reads re-check) and
//                           :1048-1285 (duplex_read_into)
// There is no CPU vote here: without a device, fgb_caller_create fails.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "bam.h"
#include "overlap.h"
#include "../planner.h"
#include "prep.h"
#include "record_filter.h"

using namespace fgb;
using namespace fgb::prep;

namespace {

enum ReadType : uint8_t { kFragment = 0, kR1 = 1, kR2 = 2 };

struct RxSource {                    // duplex: one surviving raw read's RX + FIRST_SEGMENT flag
  std::string rx;
  bool first;
};

struct Molecule {                    // duplex: one MI group that reached the vote
  std::string base_mi;
  uint32_t n_input = 0;              // a_records.len() + b_records.len() (for rejections)
  bool has_cell = false;
  std::string cell;
  // unit index of AB-R1, AB-R2, BA-R1, BA-R2 (UINT32_MAX = absent)
  uint32_t unit[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
  std::vector<RxSource> rx[4];       // RX sources per sub-family
  int32_t job[2] = {-1, -1};         // duplex combine jobs (R1, R2) when all four are present
  uint8_t pattern = 0;               // 0 full duplex, 1 AB only, 2 BA only
};

struct CodecMolecule {               // CODEC: one MI group that reached the vote
  bool has_umi = false;
  std::string umi;
  uint32_t unit_r1 = 0, unit_r2 = 0;
  uint32_t job = 0;
  bool r1_negative = false;
  uint32_t cons_len = 0;
  bool has_cell = false;
  std::string cell;
  std::vector<std::string> rx;       // RX of ALL records of the group (codec_caller.rs:1340-1349)
};

struct Prepared {
  size_t n = 0;                    // live elements of `srs`; the rest is a pool whose buffers are reused
  std::vector<SourceRead> srs;
};

// The host threads of one caller, started once: fgb_caller_add_groups and the record assembly of a flush
// each fan out several times per batch, and starting 64 threads four times per batch costs more than some
// of the phases they run.  run(n, fn) executes fn(0..n-1): task 0 on the calling thread, task t on helper
// t, and returns when all have finished.  One caller, one user at a time (a caller is not thread-safe).
class WorkerPool {
 public:
  explicit WorkerPool(uint32_t n_threads) {
    for (uint32_t i = 1; i < n_threads; ++i) threads_.emplace_back([this, i]() { loop(i); });
  }
  ~WorkerPool() {
    { std::lock_guard<std::mutex> l(m_); stop_ = true; ++gen_; }
    cv_.notify_all();
    for (auto& t : threads_) t.join();
  }
  uint32_t size() const { return static_cast<uint32_t>(threads_.size()) + 1; }
  // Returns false when a task threw (std::bad_alloc from a growing buffer, typically): the exception is
  // caught on the thread it was raised on, every task is still waited for -- the lambda's captures live on the
  // caller's frame -- and the caller turns the flag into FGB_ERR_NOMEM.
  bool run(uint32_t n, const std::function<void(uint32_t)>& fn) {
    if (n == 0) return true;
    failed_.store(false, std::memory_order_relaxed);
    if (n > 1) {
      { std::lock_guard<std::mutex> l(m_); fn_ = &fn; n_ = n; pending_ = n - 1; ++gen_; }
      cv_.notify_all();
    }
    try { fn(0); } catch (...) { failed_.store(true, std::memory_order_relaxed); }
    if (n > 1) {
      std::unique_lock<std::mutex> l(m_);
      done_.wait(l, [&] { return pending_ == 0; });
    }
    return !failed_.load(std::memory_order_relaxed);
  }

 private:
  void loop(uint32_t idx) {
    uint64_t seen = 0;
    for (;;) {
      const std::function<void(uint32_t)>* fn;
      uint32_t n;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
        fn = fn_; n = n_;
      }
      if (idx < n) {
        try { (*fn)(idx); } catch (...) { failed_.store(true, std::memory_order_relaxed); }
        std::lock_guard<std::mutex> l(m_);
        if (--pending_ == 0) done_.notify_one();
      }
    }
  }
  std::atomic<bool> failed_{false};
  std::vector<std::thread> threads_;
  std::mutex m_;
  std::condition_variable cv_, done_;
  const std::function<void(uint32_t)>* fn_ = nullptr;
  uint32_t n_ = 0, pending_ = 0;
  uint64_t gen_ = 0;
  bool stop_ = false;
};


// ---- direct path (simplex callers) ---------------------------------------------------------------------
// The records of a batch are copied once into page-locked staging memory and shipped as they are
// (FGB_IN_RECORDS); the host keeps only the per-read decisions (survival, row length, strand) and small
// references into the staging copy (UMI, cell barcode, RX values).  Each context -- the caller itself
// and each worker of fgb_caller_add_groups -- appends to its own plan; the parent keeps the order.
struct StrRef { uint64_t off = 0; uint32_t len = 0; };    // bytes inside the record staging

struct DUnit {                       // one unit (consensus read) of a plan
  uint32_t n_reads = 0, cons_len = 0;
  uint32_t rx_begin = 0, rx_n = 0;   // RX values of the surviving reads, in DirectPlan::rx
  StrRef umi, cell;
  uint8_t read_type = 0, has_cell = 0;
  uint32_t rec_size = 0;             // simplex: size of the consensus record incl. its block_size word, 0 = decided after the vote
};

struct DirectPlan {
  std::vector<fgb_raw_read> raws;    // per read: src_off relative to the staging, l_seq, strand
  std::vector<uint16_t> lens;        // per read: SourceRead row length
  std::vector<DUnit> units;
  std::vector<StrRef> rx;
  std::vector<fgb_overlap_run> oruns; // overlapping-bases runs for the device (offsets relative to the staging)
  uint64_t row_bytes = 0;            // sum of round_up(len, 8) over the reads
  uint64_t out_elems = 0;            // sum of round_up(cons_len, 8) over the units
  uint64_t rec_bytes = 0;            // sum of the units' record sizes (units with rec_size 0 add nothing)
  uint64_t str_bytes = 0;            // UMI + cell + RX bytes of the units (device record assembly)
  void clear() { raws.clear(); lens.clear(); units.clear(); rx.clear(); oruns.clear(); row_bytes = out_elems = rec_bytes = str_bytes = 0; }
};

struct DMark { size_t raws, units, rx, oruns; uint64_t row_bytes, out_elems, rec_bytes, str_bytes; size_t rejects; uint64_t reject_count; };   // a plan's size, for roll-back

struct DSeg {                        // units [u0, u1) / reads [r0, r1) of one context's plan, in input order
  struct fgb_caller* ctx;
  uint32_t u0, u1;
  uint64_t r0, r1;
  uint64_t row_bytes, out_elems;
  uint64_t o0, o1;                   // overlap runs [o0, o1) of the plan
  uint64_t rec_bytes, str_bytes;
};

struct PinBuf {                      // grow-only page-locked buffer
  void* p = nullptr;
  size_t cap = 0;
  bool pageable = false;             // the owner has no device (FGB_DEVICE_NONE): ordinary heap memory, fgb_host_alloc needs a GPU
  fgb_status ensure(size_t bytes, size_t keep = 0) {
    if (bytes <= cap) return FGB_OK;
    const size_t ncap = bytes + bytes / 2 + 4096;
    void* np = pageable ? std::malloc(ncap) : nullptr;
    if (pageable ? np == nullptr : fgb_host_alloc(&np, ncap) != FGB_OK) return FGB_ERR_NOMEM;
    if (keep) std::memcpy(np, p, keep);
    release();
    p = np; cap = ncap;
    return FGB_OK;
  }
  void release() {
    if (pageable) std::free(p); else fgb_host_free(p);
    p = nullptr; cap = 0;
  }
};

}  // namespace

struct fgb_caller {
  fgb_caller_options opt{};
  // options.track_rejects: the rejected records (block_size word + bytes) of the add calls since the last take
  std::vector<uint8_t> rejects, rejects_taken;
  uint64_t reject_count = 0, reject_taken_count = 0;
  std::string prefix, rg;
  fgb_handle* h = nullptr;
  UmiBuilder umi_builder;
  PrepOptions prep_opt;
  uint64_t stats[FGB_NSTATS] = {0};
  mutable Packer pack;                   // duplex / CODEC: the queued batch; planning-only simplex: what fgb_caller_pending laid out
  std::vector<Molecule> molecules;       // duplex
  std::vector<fgb_duplex_job> jobs;      // duplex
  uint64_t n_duplex_out = 0;
  std::vector<CodecMolecule> codec_molecules;   // CODEC
  std::vector<fgb_codec_job> codec_jobs;
  uint64_t n_codec_out = 0;
  uint64_t consensus_counter = 0;        // codec_caller.rs:1236
  std::vector<uint8_t> out;              // output of the last flush
  uint64_t out_count = 0;
  mutable std::string last_error;        // (fgb_caller_pending, const, reports through it too)
  std::vector<uint32_t> ops;             // scratch
  Prepared prepared[2];                  // simplex: [0] the alignment filter's pool; duplex: the X / Y pools; buffers reused across groups
  std::vector<uint32_t> scratch_idx[5];  // simplex: kept / fragment / R1 / R2 record indices, [4] the alignment filter's survivors (track_rejects)
  overlap::Caller overlap{overlap::kAgreeConsensus, overlap::kDisagreeConsensus};   // simplex.rs:384-387
  std::vector<uint8_t> group_copy;       // mutable copy of a group for the overlap pre-pass
  std::vector<std::unique_ptr<fgb_caller>> workers;   // per-thread prep state of fgb_caller_add_groups (no GPU handle)
  mutable std::unique_ptr<WorkerPool> pool;            // the threads themselves, started on first use
  // flush scratch that outlives a flush, so steady-state flushes neither page-fault nor zero-fill:
  uint8_t* joined = nullptr;                 // output stream of a flush (page-locked, grow-only)
  size_t joined_cap = 0, joined_len = 0;
  bool out_is_joined = false;
  void* pinned[4] = {nullptr, nullptr, nullptr, nullptr};   // consensus columns, page-locked (fgb_host_alloc)
  size_t pinned_cap = 0;                     // capacity in elements (same for the four columns)
  // ---- direct path (see DirectPlan) ----
  DirectPlan dplan;                          // what THIS context queued (the caller itself or a worker)
  std::vector<DSeg> segs;                    // parent: ranges of the plans in input order
  PinBuf stage;                              // parent: the staged records
  size_t stage_len = 0;
  const uint8_t* zc_base = nullptr;          // parent: zero-copy batch (options.zero_copy_records): the caller's own page-locked blob
  mutable PinBuf d_reads, d_raws, d_units;   // parent: descriptor arrays handed to the engine (fgb_caller_pending lays them out too)
  PinBuf px[12];                             // duplex / CODEC: page-locked result columns of a flush (grow-only)
  std::vector<View> views;                   // scratch: the records of the group being planned
  std::vector<uint64_t> rel_off;             // scratch: record offsets relative to the group
  std::vector<overlap::Run> group_runs;      // scratch: the overlap runs of the group being planned (device pre-pass)
  PinBuf d_oruns;                            // parent: the batch's runs for the engine
  PinBuf d_recjobs, d_recstr;                // parent: device record assembly (jobs, string blob)
};

namespace {

// The flush's output stream lives in page-locked memory that outlives the flush (the device writes finished
// records into it when it assembles them; the host assembly writes at final offsets).
bool ensure_joined(fgb_caller* c, size_t total) {
  if (c->joined_cap >= total + 64) return true;
  fgb_host_free(c->joined);
  c->joined = nullptr;
  c->joined_cap = total + total / 4 + 4096;
  void* p = nullptr;
  if (fgb_host_alloc(&p, c->joined_cap) != FGB_OK) { c->joined_cap = 0; c->last_error = "out of page-locked memory"; return false; }
  c->joined = static_cast<uint8_t*>(p);
  return true;
}

// fn(0..T-1) on the caller's pool (T <= options.n_threads).
void run_parallel(const fgb_caller* c, uint32_t T, const std::function<void(uint32_t)>& fn) {
  if (T <= 1) { if (T) fn(0); return; }
  if (!c->pool || c->pool->size() < T) c->pool.reset(new WorkerPool(std::max<uint32_t>(T, c->opt.n_threads)));
  if (!c->pool->run(T, fn)) throw std::bad_alloc();   // re-raised on the calling thread once every task has finished;
}                                                      // the extern "C" entry points turn it into FGB_ERR_NOMEM

void reject(fgb_caller* c, int reason, uint64_t n) {
  c->stats[FGB_STAT_FILTERED_READS] += n;
  c->stats[reason] += n;
}

bool get_string_tag(const View& v, const char tag[2], std::string* out) {
  const uint8_t* val; size_t n;
  if (!bam::find_string_tag(v, tag, &val, &n)) return false;
  out->assign(reinterpret_cast<const char*>(val), n);
  return true;
}

// ------------------------------------------------------------------------------------------------
// simplex: the group rules on record headers only (no read is decoded here; the device -- or
// fgb_caller_pending of a planning-only caller -- builds the SourceRead rows from the staged records)
// ------------------------------------------------------------------------------------------------
// vanilla_caller.rs:752-754, 1061-1063, ...: the raw bytes of a rejected read, kept as a BAM record (block_size first).
inline void keep_reject(fgb_caller* c, const View& v) {
  if (!c->opt.track_rejects) return;
  const uint32_t n = static_cast<uint32_t>(v.n);
  const size_t o = c->rejects.size();
  c->rejects.resize(o + 4 + n);
  std::memcpy(c->rejects.data() + o, &n, 4);
  std::memcpy(c->rejects.data() + o + 4, v.b, n);
  ++c->reject_count;
}

struct DRead {                       // one record of a sub-group that yields a source read
  uint32_t rec;                      // index into the group's records
  uint32_t final_len;
  const uint8_t* rx;                 // RX value inside the staged record (nullptr: none)
  uint32_t rx_len;
};

// process_subgroup up to the vote (vanilla_caller.rs:1124-1227).  True when the sub-group yields a unit;
// `out` then lists its surviving reads in order.
bool plan_subgroup(fgb_caller* c, const std::vector<View>& recs, const std::vector<uint32_t>& members,
                   std::vector<DRead>* out, size_t* surviving) {
  out->clear();
  *surviving = 0;
  const size_t min_reads = c->opt.min_reads;
  if (members.empty()) return false;
  const bool track = c->opt.track_rejects != 0;
  if (members.size() < min_reads) {
    reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, members.size());
    if (track) for (uint32_t m : members) keep_reject(c, recs[m]);                     // :1137-1142
    return false;
  }
  static const char kWant[2][2] = {{'M', 'C'}, {'R', 'X'}};
  size_t zero = 0;
  for (uint32_t k = 0; k < members.size(); ++k) {
    const View& v = recs[members[k]];
    bam::cigar_ops(v, &c->ops);
    const uint8_t* val[2]; size_t len[2];
    bam::find_string_tags(v, kWant, 2, val, len);
    const size_t clip = bam::num_bases_extending_past_mate_mc(v, c->ops, val[0], len[0]);
    uint32_t fl;
    if (c->group_runs.empty()) {
      fl = plan_read_len(c->prep_opt, v, clip);
    } else {
      // the device will have co-called the mates' overlap before it builds the rows: what the row's tail looks like
      // afterwards decides its length, so evaluate the rule for the positions the strip looks at
      const uint32_t me = members[k];
      fl = plan_read_len_eff(c->prep_opt, v, clip, [&](size_t j, uint8_t* nib, uint8_t* qq) {
        for (const overlap::Run& r : c->group_runs) {
          const bool first = r.rec1 == me && j >= r.o1 && j < static_cast<size_t>(r.o1) + r.len;
          const bool second = !first && r.rec2 == me && j >= r.o2 && j < static_cast<size_t>(r.o2) + r.len;
          if (!first && !second) continue;
          const View& o = recs[first ? r.rec2 : r.rec1];
          const size_t jo = first ? r.o2 + (j - r.o1) : r.o1 + (j - r.o2);
          const uint8_t* os = o.b + o.seq_off();
          const uint8_t oc = static_cast<uint8_t>((jo & 1) ? (os[jo >> 1] & 15u) : (os[jo >> 1] >> 4));
          const uint8_t oq = o.b[o.qual_off() + jo];
          uint8_t c1, q1, c2, q2;
          if (first) c->overlap.position_rule(*nib, oc, *qq, oq, &c1, &q1, &c2, &q2);
          else c->overlap.position_rule(oc, *nib, oq, *qq, &c2, &q2, &c1, &q1);
          *nib = c1; *qq = q1;
          return;
        }
      });
    }
    if (fl) out->push_back(DRead{members[k], fl, val[1], static_cast<uint32_t>(len[1])});
    else { ++zero; keep_reject(c, v); }                                                // :1170-1174
  }
  if (zero) reject(c, FGB_STAT_REJ_ZERO_LENGTH, zero);
  size_t n = out->size();
  if (n < min_reads) {
    if (n) {
      reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, n);
      if (track) for (const DRead& r : *out) keep_reject(c, recs[r.rec]);              // :1180-1184
    }
    return false;
  }
  // filter_source_reads_by_alignment (vanilla_caller.rs:961-1013).  Reads with the same CIGAR on the same
  // strand all join the group of the longest one (a truncated copy of a CIGAR is a prefix of the copy that
  // was truncated later, clipper.rs:2425-2448), so nothing is dropped; anything else takes the grouping code.
  bool same = true;
  {
    const View& v0 = recs[(*out)[0].rec];
    const uint32_t nc = v0.n_cigar();
    const bool rev0 = v0.flags() & bam::kReverse;
    for (size_t i = 1; i < n && same; ++i) {
      const View& v = recs[(*out)[i].rec];
      same = v.n_cigar() == nc && ((v.flags() & bam::kReverse) != 0) == rev0 && v0.cigar_in_bounds() && v.cigar_in_bounds() &&
             std::memcmp(v.b + v.cigar_off(), v0.b + v0.cigar_off(), 4 * static_cast<size_t>(nc)) == 0;
    }
  }
  if (!same) {
    Prepared& pool = c->prepared[0];
    pool.n = 0;
    for (size_t i = 0; i < n; ++i) {
      const View& v = recs[(*out)[i].rec];
      if (pool.n == pool.srs.size()) pool.srs.emplace_back();
      SourceRead& sr = pool.srs[pool.n++];
      sr.bases.resize((*out)[i].final_len);                  // only the length and the CIGAR take part
      bam::cigar_ops(v, &c->ops);
      bam::simplify_cigar(c->ops, &sr.cigar);
      if (v.flags() & bam::kReverse) std::reverse(sr.cigar.begin(), sr.cigar.end());
      bam::truncate_cigar(&sr.cigar, (*out)[i].final_len);
      sr.original_idx = static_cast<uint32_t>(i);
      sr.flags = v.flags();
    }
    const size_t kept = filter_by_alignment_n(&pool.srs, pool.n);
    if (kept != n) {
      reject(c, FGB_STAT_REJ_MINORITY_ALIGNMENT, n - kept);
      if (track) {                                                                     // :1193-1197, ascending input order
        std::vector<uint32_t>& alive = c->scratch_idx[4];
        alive.assign(n, 0u);
        for (size_t i = 0; i < kept; ++i) alive[pool.srs[i].original_idx] = 1u;
        for (size_t i = 0; i < n; ++i) if (!alive[i]) keep_reject(c, recs[(*out)[i].rec]);
      }
      static thread_local std::vector<DRead> tmp;
      tmp.clear();
      for (size_t i = 0; i < kept; ++i) tmp.push_back((*out)[pool.srs[i].original_idx]);
      out->assign(tmp.begin(), tmp.end());
      n = kept;
    }
    if (n < min_reads) {
      if (n) {
        reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, n);
        if (track) for (const DRead& r : *out) keep_reject(c, recs[r.rec]);            // :1205-1209
      }
      return false;
    }
  }
  *surviving = n;
  return true;
}

inline uint32_t int_tag_width(uint32_t v) { return v <= 255u ? 1u : (v <= 65535u ? 2u : 4u); }   // tags.rs:533-553, v >= 0

// Size of the simplex consensus record write_simplex_record_at produces (block_size word included).
inline uint32_t simplex_record_size(const fgb_caller* c, uint32_t L, uint32_t umi_len, bool has_cell, uint32_t cell_len,
                                    bool has_rx, uint32_t rx_len, uint32_t w_cd, uint32_t w_cm) {
  const uint32_t name = static_cast<uint32_t>(c->prefix.size()) + 1u + umi_len;
  uint32_t n = 4u + 32u + name + 1u + (L + 1u) / 2u + L;
  n += 3u + static_cast<uint32_t>(c->rg.size()) + 1u;          // RG
  n += 3u + w_cd + 3u + w_cm + 3u + 4u;                        // cD cM cE
  if (c->opt.produce_per_base_tags) n += 2u * (3u + 1u + 4u + 2u * L);
  n += 3u + umi_len + 1u;                                      // MI
  if (has_cell) n += 3u + cell_len + 1u;
  if (has_rx) n += 3u + rx_len + 1u;
  return n;
}

void pack_direct_unit(fgb_caller* c, const uint8_t* stage, const std::vector<View>& recs, const std::vector<DRead>& rd,
                      uint8_t read_type, StrRef umi) {
  DirectPlan& P = c->dplan;
  DUnit u;
  u.n_reads = static_cast<uint32_t>(rd.size());
  u.read_type = read_type;
  u.umi = umi;
  u.rx_begin = static_cast<uint32_t>(P.rx.size());
  static thread_local std::vector<uint32_t> lens;
  lens.clear();
  for (const DRead& r : rd) {
    const View& v = recs[r.rec];
    fgb_raw_read rr;
    rr.src_off = static_cast<uint64_t>(v.b - stage) + v.seq_off();
    rr.raw_len = v.l_seq();
    rr.flags = (v.flags() & bam::kReverse) ? FGB_RAW_REVERSE : 0u;
    P.raws.push_back(rr);
    P.lens.push_back(static_cast<uint16_t>(r.final_len));
    P.row_bytes += round_up(r.final_len, FGB_READ_ALIGN);
    lens.push_back(r.final_len);
    if (r.rx) P.rx.push_back(StrRef{static_cast<uint64_t>(r.rx - stage), r.rx_len});
  }
  u.rx_n = static_cast<uint32_t>(P.rx.size()) - u.rx_begin;
  if (u.rx_n > 1) {
    // The usual family: every RX value identical and free of lower-case bases.  Its consensus is the value itself
    // (consensus_umis_refs' first case); deciding that HERE, while the tag bytes of the group's records are in cache,
    // leaves the flush one reference to follow instead of rx_n cold ones.
    const StrRef* rf = P.rx.data() + u.rx_begin;
    const uint8_t* f = stage + rf[0].off;
    bool same = true;
    for (uint32_t k = 1; k < u.rx_n && same; ++k) same = rf[k].len == rf[0].len && std::memcmp(stage + rf[k].off, f, rf[0].len) == 0;
    for (uint32_t i = 0; i < rf[0].len && same; ++i) { const uint8_t ch = f[i]; same = !(ch == 'a' || ch == 'c' || ch == 'g' || ch == 't' || ch == 'n'); }
    if (same) { P.rx.resize(u.rx_begin + 1u); u.rx_n = 1; }
  }
  const size_t kth = c->opt.min_reads - 1;                      // vanilla_caller.rs:1269-1277
  std::nth_element(lens.begin(), lens.begin() + kth, lens.end(), std::greater<uint32_t>());
  u.cons_len = lens[kth];
  P.out_elems += round_up(u.cons_len, FGB_OUT_ALIGN);
  if (c->opt.cell_tag[0] && !rd.empty()) {
    const uint8_t* val; size_t n;
    if (bam::find_string_tag(recs[rd[0].rec], c->opt.cell_tag, &val, &n)) {
      u.has_cell = 1;
      u.cell = StrRef{static_cast<uint64_t>(val - stage), static_cast<uint32_t>(n)};
    }
  }
  if (u.n_reads <= 255u)                                        // cD / cM fit one byte whatever the vote says
    u.rec_size = simplex_record_size(c, u.cons_len, umi.len, u.has_cell, u.cell.len, u.rx_n > 0,
                                     u.rx_n ? P.rx[u.rx_begin].len : 0u, 1u, 1u);
  P.rec_bytes += u.rec_size;
  P.str_bytes += umi.len + (u.has_cell ? u.cell.len : 0u) + (u.rx_n ? P.rx[u.rx_begin].len : 0u);
  P.units.push_back(u);
}

// consensus_reads for one MI group (vanilla_caller.rs:1477-1499 + process_group :1042-1114); `recs` are
// views of the STAGED records.
fgb_status direct_group_simplex(fgb_caller* c, const uint8_t* stage, const std::vector<View>& recs) {
  const uint32_t n_records = static_cast<uint32_t>(recs.size());
  const uint8_t* uv; size_t un;
  if (!bam::find_string_tag(recs[0], c->opt.tag, &uv, &un)) {   // vanilla_caller.rs:1493-1496
    c->last_error = std::string("Missing UMI tag '") + c->opt.tag[0] + c->opt.tag[1] + "'";
    return FGB_ERR_MISSING_TAG;
  }
  const StrRef umi{static_cast<uint64_t>(uv - stage), static_cast<uint32_t>(un)};
  for (const View& v : recs)
    if (v.l_seq() > FGB_MAX_READ_LEN) {
      c->last_error = "a read is longer than 65535 bases (FGB_MAX_READ_LEN)";
      return FGB_ERR_UNIT_TOO_LARGE;
    }
  c->stats[FGB_STAT_TOTAL_READS] += n_records;
  std::vector<uint32_t>&kept = c->scratch_idx[0], &frag = c->scratch_idx[1], &r1 = c->scratch_idx[2], &r2 = c->scratch_idx[3];
  kept.clear(); frag.clear(); r1.clear(); r2.clear();
  for (uint32_t i = 0; i < n_records; ++i) {
    const uint16_t f = recs[i].flags();
    if (!(f & bam::kSecondary) && !(f & bam::kSupplementary)) kept.push_back(i);
  }
  if (kept.size() != n_records) {
    reject(c, FGB_STAT_REJ_SECONDARY_SUPPLEMENTARY, n_records - kept.size());
    if (c->opt.track_rejects)                                                          // filter_reads, :745-757
      for (uint32_t i = 0; i < n_records; ++i)
        if (recs[i].flags() & (bam::kSecondary | bam::kSupplementary)) keep_reject(c, recs[i]);
  }
  if (kept.empty()) return FGB_OK;
  if (kept.size() < c->opt.min_reads) {
    reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, kept.size());
    for (uint32_t i : kept) keep_reject(c, recs[i]);                                   // :1061-1063
    return FGB_OK;
  }
  for (uint32_t i : kept) {   // subgroup_reads, vanilla_caller.rs:1018-1039
    const uint16_t f = recs[i].flags();
    if (!(f & bam::kPaired)) frag.push_back(i);
    else if (f & bam::kFirst) r1.push_back(i);
    else if (f & bam::kLast) r2.push_back(i);
  }
  if (frag.size() > 0xFFFFu || r1.size() > 0xFFFFu || r2.size() > 0xFFFFu) {   // u16 observation counters, base_builder.rs:236
    c->last_error = "a sub-group (fragment / R1 / R2 reads of one MI) has more than 65535 reads";
    return FGB_ERR_UNIT_TOO_LARGE;
  }
  static thread_local std::vector<DRead> df, d1, d2;
  size_t sf, s1, s2;
  if (plan_subgroup(c, recs, frag, &df, &sf)) { pack_direct_unit(c, stage, recs, df, kFragment, umi); c->stats[FGB_STAT_CONSENSUS_READS] += 1; }
  const bool ok1 = plan_subgroup(c, recs, r1, &d1, &s1);
  const bool ok2 = plan_subgroup(c, recs, r2, &d2, &s2);
  if (ok1 && ok2) {   // orphan rule, vanilla_caller.rs:1089-1108
    pack_direct_unit(c, stage, recs, d1, kR1, umi);
    pack_direct_unit(c, stage, recs, d2, kR2, umi);
    c->stats[FGB_STAT_CONSENSUS_READS] += 2;
  } else if (ok1) {
    reject(c, FGB_STAT_REJ_ORPHAN_CONSENSUS, s1);
    for (const DRead& r : d1) keep_reject(c, recs[r.rec]);                             // :1095-1099
  } else if (ok2) {
    reject(c, FGB_STAT_REJ_ORPHAN_CONSENSUS, s2);
    for (const DRead& r : d2) keep_reject(c, recs[r.rec]);                             // :1101-1105
  }
  return FGB_OK;
}

float error_rate(uint64_t errors, uint64_t depth) {
  return depth > 0 ? static_cast<float>(errors) / static_cast<float>(depth) : 0.0f;
}

fgb_status append_rx(fgb_caller* c, bam::Writer* w, const std::vector<std::string>& umis) {
  if (umis.empty()) return FGB_OK;
  std::string rx;
  if (!consensus_umis(c->umi_builder, umis, &rx)) {
    c->last_error = "RX values of a family have different lengths or mix DNA and non-DNA characters";
    return FGB_ERR_INVALID_ARG;   // the reference panics here (simple_umi.rs:78-116)
  }
  w->str("RX", rx.data(), rx.size());
  return FGB_OK;
}

// FGB_CALLER_TRACE=1 prints the phases of a flush to stderr (diagnostics only).
struct PhaseTrace {
  bool on = std::getenv("FGB_CALLER_TRACE") != nullptr;
  std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
  void mark(const char* what) {
    if (!on) return;
    auto n = std::chrono::steady_clock::now();
    std::fprintf(stderr, "fgb_caller flush: %-22s %8.2f ms\n", what,
                 std::chrono::duration<double, std::milli>(n - t).count());
    t = n;
  }
};

// ------------------------------------------------------------------------------------------------
// simplex, direct path: flush
// ------------------------------------------------------------------------------------------------
// consensus_umis (simple_umi.rs:65-122, 236-245) over references into the staged records.
bool consensus_umis_refs(const UmiBuilder& builder, const uint8_t* base, const StrRef* refs, uint32_t n, std::string* out) {
  out->clear();
  if (n == 0) return true;
  if (n == 1) { out->assign(reinterpret_cast<const char*>(base + refs[0].off), refs[0].len); return true; }
  const uint32_t len = refs[0].len;
  for (uint32_t k = 1; k < n; ++k) if (refs[k].len != len) return false;
  {
    // Every value identical (the usual family) and free of lower-case bases: each DNA column is unanimous and calls
    // its own base (UmiBuilder::call: no tie, no rounding can touch a unanimous column; an all-N column calls N),
    // each non-DNA column passes its character through -- the consensus is the value itself.
    const uint8_t* f = base + refs[0].off;
    bool same = true;
    for (uint32_t k = 1; k < n && same; ++k) same = std::memcmp(base + refs[k].off, f, len) == 0;
    if (same) {
      bool plain = true;
      for (uint32_t i = 0; i < len && plain; ++i) { const uint8_t ch = f[i]; plain = !(ch == 'a' || ch == 'c' || ch == 'g' || ch == 't' || ch == 'n'); }
      if (plain) { out->assign(reinterpret_cast<const char*>(f), len); return true; }
    }
  }
  auto is_dna = [](uint8_t ch) {
    switch (ch) { case 'A': case 'C': case 'G': case 'T': case 'N':
                  case 'a': case 'c': case 'g': case 't': case 'n': return true; default: return false; }
  };
  static thread_local std::vector<uint8_t> col;
  col.resize(n);
  const uint8_t* first = base + refs[0].off;
  for (uint32_t i = 0; i < len; ++i) {
    size_t non_dna = 0;
    for (uint32_t k = 0; k < n; ++k) {
      col[k] = base[refs[k].off + i];
      if (!is_dna(col[k])) {
        ++non_dna;
        if (col[k] != first[i]) return false;
      }
    }
    if (non_dna == 0) out->push_back(static_cast<char>(builder.call(col)));
    else if (non_dna == n) out->push_back(static_cast<char>(first[i]));
    else return false;
  }
  return true;
}

// Record encoder over a raw buffer whose size is known up front (UnmappedSamBuilder + tag encoders,
// raw-bam builder.rs:90-230, tags.rs:512-667; the vector-backed twin is bam::Writer).
struct RawWriter {
  uint8_t* p;
  void put(const void* s, size_t n) { std::memcpy(p, s, n); p += n; }
  template <class T> void le(T v) { std::memcpy(p, &v, sizeof(T)); p += sizeof(T); }
  void tag(const char t[2], char type) { p[0] = static_cast<uint8_t>(t[0]); p[1] = static_cast<uint8_t>(t[1]); p[2] = static_cast<uint8_t>(type); p += 3; }
  void str(const char t[2], const void* v, size_t n) { tag(t, 'Z'); put(v, n); *p++ = 0; }
  void integer(const char t[2], int32_t v) {
    if (v >= -128 && v <= 127) { tag(t, 'c'); *p++ = static_cast<uint8_t>(static_cast<int8_t>(v)); }
    else if (v >= 0 && v <= 255) { tag(t, 'C'); *p++ = static_cast<uint8_t>(v); }
    else if (v >= 0 && v <= 65535) { tag(t, 'S'); le<uint16_t>(static_cast<uint16_t>(v)); }
    else if (v >= -32768 && v <= 32767) { tag(t, 's'); le<int16_t>(static_cast<int16_t>(v)); }
    else { tag(t, 'i'); le<int32_t>(v); }
  }
  void real(const char t[2], float v) { tag(t, 'f'); le<float>(v); }
  template <class D> void i16_array(const char t[2], const D* v, uint32_t n) {   // values clamp to i16::MAX
    tag(t, 'B'); *p++ = 's'; le<uint32_t>(n);
    for (uint32_t i = 0; i < n; ++i) { const uint16_t x = v[i] > 32767 ? 32767 : static_cast<uint16_t>(v[i]); std::memcpy(p + 2 * i, &x, 2); }
    p += 2 * static_cast<size_t>(n);
  }
};

// build_consensus_record_into (vanilla_caller.rs:1365-1473) at `dst`; returns the bytes written (block_size
// word included), 0 with *err set when the reference would have failed.
template <class D>
size_t write_simplex_record_at(const fgb_caller* c, uint8_t* dst, const DUnit& u, const StrRef* rx, const uint8_t* stage,
                               const uint8_t* bases, const uint8_t* quals, const D* depths, const D* errors,
                               std::string* rx_scratch, std::string* err) {
  static const bam::Writer::CodeTable kCodes;
  const uint32_t L = u.cons_len;
  const size_t name_len = c->prefix.size() + 1 + u.umi.len;
  if (name_len >= 255) { *err = "read name too long"; return 0; }
  uint16_t flag = bam::kUnmapped;
  if (u.read_type == kR1) flag |= bam::kPaired | bam::kFirst | bam::kMateUnmapped;
  else if (u.read_type == kR2) flag |= bam::kPaired | bam::kLast | bam::kMateUnmapped;
  RawWriter w{dst + 4};
  w.le<int32_t>(-1); w.le<int32_t>(-1);
  *w.p++ = static_cast<uint8_t>(name_len + 1);
  *w.p++ = 0;
  w.le<uint16_t>(4680); w.le<uint16_t>(0); w.le<uint16_t>(flag); w.le<uint32_t>(L);
  w.le<int32_t>(-1); w.le<int32_t>(-1); w.le<int32_t>(0);
  w.put(c->prefix.data(), c->prefix.size());
  *w.p++ = ':';
  w.put(stage + u.umi.off, u.umi.len);
  *w.p++ = 0;
  {
    uint8_t* sp = w.p;
    for (uint32_t i = 0; i + 1 < L; i += 2) sp[i >> 1] = static_cast<uint8_t>((kCodes.t[bases[i]] << 4) | kCodes.t[bases[i + 1]]);
    if (L & 1) sp[L >> 1] = static_cast<uint8_t>(kCodes.t[bases[L - 1]] << 4);
    w.p += (static_cast<size_t>(L) + 1) / 2;
    if (L) w.put(quals, L);
  }
  w.str("RG", c->rg.data(), c->rg.size());
  uint32_t max_d = 0, min_d = L ? 0xFFFFFFFFu : 0;
  uint64_t tot_e = 0, tot_d = 0;
  for (uint32_t k = 0; k < L; ++k) {
    const uint32_t d = depths[k];
    max_d = d > max_d ? d : max_d;
    min_d = d < min_d ? d : min_d;
    tot_e += errors[k];
    tot_d += d;
  }
  w.integer("cD", static_cast<int32_t>(max_d));
  w.integer("cM", static_cast<int32_t>(min_d));
  w.real("cE", error_rate(tot_e, tot_d));
  if (c->opt.produce_per_base_tags) {
    w.i16_array("cd", depths, L);
    w.i16_array("ce", errors, L);
  }
  w.str("MI", stage + u.umi.off, u.umi.len);
  if (u.has_cell) w.str(c->opt.cell_tag, stage + u.cell.off, u.cell.len);
  if (u.rx_n) {
    if (!consensus_umis_refs(c->umi_builder, stage, rx, u.rx_n, rx_scratch)) {   // the reference panics here (simple_umi.rs:78-116)
      *err = "RX values of a family have different lengths or mix DNA and non-DNA characters";
      return 0;
    }
    w.str("RX", rx_scratch->data(), rx_scratch->size());
  }
  const size_t total = static_cast<size_t>(w.p - dst);
  const uint32_t bs = static_cast<uint32_t>(total - 4);
  std::memcpy(dst, &bs, 4);
  return total;
}

// fn(i) for every segment i of the queued batch, on up to options.n_threads of the caller's threads.
void for_segs(const fgb_caller* c, const std::function<void(size_t)>& fn) {
  const size_t NS = c->segs.size();
  const uint32_t T = std::max<uint32_t>(1u, std::min<uint32_t>(std::max<uint32_t>(c->opt.n_threads, 1u), static_cast<uint32_t>(NS)));
  if (T <= 1) { for (size_t i = 0; i < NS; ++i) fn(i); return; }
  run_parallel(c, T, [&](uint32_t t) { for (size_t i = t; i < NS; i += T) fn(i); });
}

// The queued plans laid out as one batch (the flush's, and fgb_caller_pending's on a planning-only caller): prefix sums
// over the segments, then every segment's descriptors at their global places in d_reads / d_raws / d_units, the
// sentinel unit and two zero row descriptors behind them.
struct DLayout {
  std::vector<uint64_t> ub, rbase, bb, ob;   // per segment (and one past the last): first unit, read, row byte, output element
  uint64_t U = 0, R = 0, n_bytes = 0, n_out = 0;
  uint32_t max_reads = 0;                    // reads of the deepest unit
  uint64_t* reads = nullptr;
  fgb_raw_read* raws = nullptr;
  fgb_unit* units = nullptr;
};

fgb_status lay_out_direct(const fgb_caller* c, DLayout* L) {
  const size_t NS = c->segs.size();
  std::vector<uint64_t> &ub = L->ub, &rbase = L->rbase, &bb = L->bb, &ob = L->ob;
  ub.assign(NS + 1, 0); rbase.assign(NS + 1, 0); bb.assign(NS + 1, 0); ob.assign(NS + 1, 0);
  for (size_t i = 0; i < NS; ++i) {
    const DSeg& sg = c->segs[i];
    ub[i + 1] = ub[i] + (sg.u1 - sg.u0);
    rbase[i + 1] = rbase[i] + (sg.r1 - sg.r0);
    bb[i + 1] = bb[i] + sg.row_bytes;
    ob[i + 1] = ob[i] + sg.out_elems;
  }
  const uint64_t U = ub[NS], R = rbase[NS];
  L->U = U; L->R = R; L->n_bytes = bb[NS]; L->n_out = ob[NS];
  if (!U) return FGB_OK;
  if (U >= 0xFFFFFFFFull || R >= 0xFFFFFFFFull) { c->last_error = "batch too large"; return FGB_ERR_INVALID_ARG; }
  if (c->d_reads.ensure((R + 2) * sizeof(uint64_t)) != FGB_OK || c->d_raws.ensure((R + 1) * sizeof(fgb_raw_read)) != FGB_OK ||
      c->d_units.ensure((U + 1) * sizeof(fgb_unit)) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
  uint64_t* g_reads = L->reads = static_cast<uint64_t*>(c->d_reads.p);
  fgb_raw_read* g_raws = L->raws = static_cast<fgb_raw_read*>(c->d_raws.p);
  fgb_unit* g_units = L->units = static_cast<fgb_unit*>(c->d_units.p);
  std::vector<uint32_t> seg_max(NS, 0);
  for_segs(c, [&](size_t i) {    // descriptors of segment i at their global places
    const DSeg& sg = c->segs[i];
    const DirectPlan& P = sg.ctx->dplan;
    uint64_t off = bb[i], oo = ob[i], r = rbase[i];
    uint64_t lr = sg.r0;
    uint32_t mx = 0;
    for (uint32_t u = sg.u0; u < sg.u1; ++u) {
      const DUnit& du = P.units[u];
      fgb_unit gu;
      gu.out_off = oo; gu.read_begin = static_cast<uint32_t>(r); gu.cons_len = du.cons_len;
      g_units[ub[i] + (u - sg.u0)] = gu;
      oo += round_up(du.cons_len, FGB_OUT_ALIGN);
      mx = du.n_reads > mx ? du.n_reads : mx;
      for (uint32_t k = 0; k < du.n_reads; ++k, ++lr, ++r) {
        const uint32_t len = P.lens[lr];
        g_reads[r] = FGB_READ_DESC(off, len);
        g_raws[r] = P.raws[lr];
        off += round_up(len, FGB_READ_ALIGN);
      }
    }
    seg_max[i] = mx;
  });
  {
    fgb_unit sentinel;
    sentinel.out_off = L->n_out; sentinel.read_begin = static_cast<uint32_t>(R); sentinel.cons_len = 0;
    g_units[U] = sentinel;
    g_reads[R] = 0; g_reads[R + 1] = 0;
  }
  for (uint32_t m : seg_max) L->max_reads = m > L->max_reads ? m : L->max_reads;
  return FGB_OK;
}

fgb_status flush_simplex_direct(fgb_caller* c) {
  PhaseTrace trace;
  DLayout L;
  const fgb_status lst = lay_out_direct(c, &L);
  if (lst != FGB_OK) return lst;
  if (!L.U) {
    // Nothing to vote, so nothing goes to the device.  The queued overlap runs (pairs the group rules rejected)
    // still count, as the reference co-calls every pair (simplex.rs:395-398); their rewritten bases would feed no
    // row, so the counters come from a read-only pass over the staged records (or the caller's own blob).
    const uint8_t* const stage0 = c->zc_base ? c->zc_base : static_cast<const uint8_t*>(c->stage.p);
    for (const DSeg& sg : c->segs)
      for (uint64_t k = sg.o0; k < sg.o1; ++k) {
        const fgb_overlap_run& r = sg.ctx->dplan.oruns[k];
        const uint8_t* s1 = stage0 + r.seq1_off; const uint8_t* s2 = stage0 + r.seq2_off;
        c->overlap.count_run(s1, s1 + (r.l_seq1 + 1ull) / 2, r.o1, s2, s2 + (r.l_seq2 + 1ull) / 2, r.o2, r.len);
      }
    return FGB_OK;
  }
  const size_t NS = c->segs.size();
  const std::vector<uint64_t> &ub = L.ub, &bb = L.bb;
  const uint64_t U = L.U, R = L.R, n_bytes = L.n_bytes, no = L.n_out;
  const uint32_t max_reads = L.max_reads;
  uint64_t* const g_reads = L.reads;
  fgb_raw_read* const g_raws = L.raws;
  fgb_unit* const g_units = L.units;
  trace.mark("descriptors");
  // ---- tiles: every segment plans its own range (a tile never spans two segments) ----
  std::vector<std::vector<fgb_tile>> seg_tiles(NS);
  std::vector<fgb_status> seg_st(NS, FGB_OK);
  for_segs(c, [&](size_t i) {
    uint64_t prev_end = bb[i];
    seg_tiles[i].clear();
    seg_st[i] = plan_tiles_range(g_units, ub[i], ub[i + 1], g_reads, R, &prev_end, [&](const fgb_tile& t) { seg_tiles[i].push_back(t); });
  });
  size_t n_tiles = 0;
  for (size_t i = 0; i < NS; ++i) {
    if (seg_st[i] != FGB_OK) { c->last_error = "tile planning failed"; return seg_st[i]; }
    n_tiles += seg_tiles[i].size();
  }
  std::vector<fgb_tile> tiles;
  tiles.reserve(n_tiles + 1);
  for (size_t i = 0; i < NS; ++i) tiles.insert(tiles.end(), seg_tiles[i].begin(), seg_tiles[i].end());
  trace.mark("tiles");
  // ---- record assembly on the device (K5) when the engine offers it, every record's size is known up front (no
  //      unit deeper than 255 reads) and no filter decides what is emitted: the host supplies the strings only ----
  if (!c->opt.filter_enabled && max_reads <= 255u && (fgb_engine_caps() & FGB_CAP_RECORD_ASSEMBLY)) {
    std::vector<uint64_t> rb_(NS + 1, 0), sb_(NS + 1, 0);
    const uint64_t head = c->prefix.size() + c->rg.size();
    sb_[0] = head;
    for (size_t i = 0; i < NS; ++i) { rb_[i + 1] = rb_[i] + c->segs[i].rec_bytes; sb_[i + 1] = sb_[i] + c->segs[i].str_bytes; }
    const uint64_t total = rb_[NS], n_str = sb_[NS];
    if (n_str >= 0xFFFFFFFFull) { c->last_error = "batch too large"; return FGB_ERR_INVALID_ARG; }
    if (c->d_recjobs.ensure((U + 1) * sizeof(fgb_record_job)) != FGB_OK || c->d_recstr.ensure(n_str + 64) != FGB_OK || !ensure_joined(c, total)) {
      c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM;
    }
    fgb_record_job* jobs = static_cast<fgb_record_job*>(c->d_recjobs.p);
    uint8_t* strs = static_cast<uint8_t*>(c->d_recstr.p);
    std::memcpy(strs, c->prefix.data(), c->prefix.size());
    std::memcpy(strs + c->prefix.size(), c->rg.data(), c->rg.size());
    const uint8_t* const stage0 = c->zc_base ? c->zc_base : static_cast<const uint8_t*>(c->stage.p);
    std::vector<int> bad(NS, 0);
    for_segs(c, [&](size_t i) {       // jobs and strings of segment i; the RX consensus (simple_umi.rs:236-245) is computed here
      const DSeg& sg = c->segs[i];
      const DirectPlan& P = sg.ctx->dplan;
      uint64_t ro = rb_[i], so_ = sb_[i];
      static thread_local std::string rx;
      for (uint32_t u = sg.u0; u < sg.u1; ++u) {
        const DUnit& du = P.units[u];
        fgb_record_job j;
        j.out_off = ro; j.str_off = static_cast<uint32_t>(so_); j.size = du.rec_size;
        j.umi_len = static_cast<uint16_t>(du.umi.len); j.cell_len = du.has_cell ? static_cast<uint16_t>(du.cell.len) : 0;
        j.rx_len = 0; j.read_type = du.read_type;
        j.flags = (du.has_cell ? FGB_RECJOB_HAS_CELL : 0) | (du.rx_n ? FGB_RECJOB_HAS_RX : 0);
        if (c->prefix.size() + 1 + du.umi.len >= 255 || du.umi.len > 0xFFFFu || du.cell.len > 0xFFFFu) { bad[i] = 1; return; }
        std::memcpy(strs + so_, stage0 + du.umi.off, du.umi.len); so_ += du.umi.len;
        if (du.has_cell) { std::memcpy(strs + so_, stage0 + du.cell.off, du.cell.len); so_ += du.cell.len; }
        if (du.rx_n) {
          const uint32_t want = P.rx[du.rx_begin].len;
          if (!consensus_umis_refs(c->umi_builder, stage0, P.rx.data() + du.rx_begin, du.rx_n, &rx) || rx.size() != want || want > 0xFFFFu) { bad[i] = 2; return; }
          std::memcpy(strs + so_, rx.data(), want); so_ += want;
          j.rx_len = static_cast<uint16_t>(want);
        }
        jobs[ub[i] + (u - sg.u0)] = j;
        ro += du.rec_size;
      }
    });
    for (size_t i = 0; i < NS; ++i)
      if (bad[i]) {
        c->last_error = bad[i] == 1 ? "read name too long"
                                    : "RX values of a family have different lengths or mix DNA and non-DNA characters";
        return FGB_ERR_INVALID_ARG;
      }
    std::memset(&jobs[U], 0, sizeof(fgb_record_job));
    jobs[U].out_off = total;
    trace.mark("record jobs");
    fgb_batch b;
    std::memset(&b, 0, sizeof(b));
    b.n_units = U; b.n_reads = R; b.n_bytes = n_bytes; b.n_out = no; b.n_tiles = n_tiles;
    b.reads = g_reads; b.units = g_units; b.tiles = tiles.data();
    fgb_columns none{nullptr, nullptr, nullptr, nullptr};
    fgb_record_columns rc;
    std::memset(&rc, 0, sizeof(rc));
    rc.n_bytes = c->stage_len; rc.records = stage0; rc.raw_reads = g_raws;
    rc.min_input_base_quality = c->prep_opt.min_input_base_quality;
    fgb_submit_options so;
    std::memset(&so, 0, sizeof(so));
    so.input_format = FGB_IN_RECORDS; so.output_format = FGB_OUT_U16;
    so.records = &rc;
    uint64_t n_runs = 0;
    for (const DSeg& sg : c->segs) n_runs += sg.o1 - sg.o0;
    if (n_runs) {
      if (c->d_oruns.ensure(n_runs * sizeof(fgb_overlap_run)) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
      fgb_overlap_run* dst = static_cast<fgb_overlap_run*>(c->d_oruns.p);
      for (const DSeg& sg : c->segs) {
        const size_t k = sg.o1 - sg.o0;
        if (k) std::memcpy(dst, sg.ctx->dplan.oruns.data() + sg.o0, k * sizeof(fgb_overlap_run));
        dst += k;
      }
      so.overlap_runs = static_cast<const fgb_overlap_run*>(c->d_oruns.p);
      so.n_overlap_runs = n_runs;
      so.overlap_stats = &c->overlap.stats.overlapping_bases;
      so.overlap_agreement = static_cast<uint8_t>(c->overlap.agreement());
      so.overlap_disagreement = static_cast<uint8_t>(c->overlap.disagreement());
    }
    so.rec_jobs = jobs; so.rec_strings = strs; so.n_rec_string_bytes = n_str;
    so.rec_prefix_len = static_cast<uint32_t>(c->prefix.size()); so.rec_rg_len = static_cast<uint32_t>(c->rg.size());
    so.rec_cell_tag[0] = static_cast<uint8_t>(c->opt.cell_tag[0]); so.rec_cell_tag[1] = static_cast<uint8_t>(c->opt.cell_tag[1]);
    so.rec_per_base_tags = c->opt.produce_per_base_tags;
    so.rec_out = c->joined; so.n_rec_out_bytes = total;
    fgb_status st = fgb_submit_ex(c->h, &b, &none, &so);
    if (st == FGB_OK) st = fgb_wait(c->h);
    if (st != FGB_OK) {
      char buf[256];
      fgb_last_error(c->h, buf, sizeof(buf));
      c->last_error = buf;
      return st;
    }
    trace.mark("submit + wait (records assembled on the device)");
    c->out_count += U;
    c->joined_len = total;
    c->out_is_joined = true;
    return FGB_OK;
  }
  // ---- output columns (page-locked, grow-only); depth / errors travel as bytes when no unit is deeper than 255 ----
  const bool narrow = max_reads <= 255u;
  if (c->pinned_cap < no + 8) {
    for (void*& p : c->pinned) { fgb_host_free(p); p = nullptr; }
    c->pinned_cap = 0;
    const size_t cap = (no + 8) + (no + 8) / 4;
    const size_t bytes[4] = {cap, cap, cap * 2, cap * 2};
    for (int i = 0; i < 4; ++i)
      if (fgb_host_alloc(&c->pinned[i], bytes[i]) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
    c->pinned_cap = cap;
  }
  uint8_t* const o_base = static_cast<uint8_t*>(c->pinned[0]);
  uint8_t* const o_qual = static_cast<uint8_t*>(c->pinned[1]);
  fgb_batch b;
  std::memset(&b, 0, sizeof(b));
  b.n_units = U; b.n_reads = R; b.n_bytes = n_bytes; b.n_out = no; b.n_tiles = n_tiles;
  b.reads = g_reads; b.units = g_units; b.tiles = tiles.data();
  fgb_columns cols{o_base, o_qual, static_cast<uint16_t*>(c->pinned[2]), static_cast<uint16_t*>(c->pinned[3])};
  fgb_record_columns rc;
  std::memset(&rc, 0, sizeof(rc));
  rc.n_bytes = c->stage_len; rc.records = c->zc_base ? c->zc_base : static_cast<const uint8_t*>(c->stage.p); rc.raw_reads = g_raws;
  rc.min_input_base_quality = c->prep_opt.min_input_base_quality;
  std::vector<uint8_t> fstatus;
  std::vector<uint32_t> fmasked;
  fgb_filter_params fp = c->opt.filter;
  fgb_submit_options so;
  std::memset(&so, 0, sizeof(so));
  so.input_format = FGB_IN_RECORDS; so.output_format = narrow ? FGB_OUT_U8 : FGB_OUT_U16;
  so.records = &rc;
  {
    uint64_t n_runs = 0;
    for (const DSeg& sg : c->segs) n_runs += sg.o1 - sg.o0;
    if (n_runs) {                // the overlapping-bases pre-pass, on the device (K0o)
      if (c->d_oruns.ensure(n_runs * sizeof(fgb_overlap_run)) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
      fgb_overlap_run* dst = static_cast<fgb_overlap_run*>(c->d_oruns.p);
      for (const DSeg& sg : c->segs) {
        const size_t k = sg.o1 - sg.o0;
        if (k) std::memcpy(dst, sg.ctx->dplan.oruns.data() + sg.o0, k * sizeof(fgb_overlap_run));
        dst += k;
      }
      so.overlap_runs = static_cast<const fgb_overlap_run*>(c->d_oruns.p);
      so.n_overlap_runs = n_runs;
      so.overlap_stats = &c->overlap.stats.overlapping_bases;      // four consecutive u64 counters
      so.overlap_agreement = static_cast<uint8_t>(c->overlap.agreement());
      so.overlap_disagreement = static_cast<uint8_t>(c->overlap.disagreement());
    }
  }
  if (c->opt.filter_enabled) {   // `fgumi filter` as an epilogue of the vote (commands/filter.rs:738-905)
    fstatus.assign(U + 1, FGB_FILTER_PASS);
    fmasked.assign(U + 1, 0);
    fp.per_base_tags = c->opt.produce_per_base_tags;
    so.filter = &fp; so.unit_status = fstatus.data(); so.unit_masked = fmasked.data();
  }
  fgb_status st = fgb_submit_ex(c->h, &b, &cols, &so);
  if (st == FGB_OK) st = fgb_wait(c->h);
  if (st != FGB_OK) {
    char buf[256];
    fgb_last_error(c->h, buf, sizeof(buf));
    c->last_error = buf;
    return st;
  }
  trace.mark("submit + wait");
  const uint8_t* const stage = c->zc_base ? c->zc_base : static_cast<const uint8_t*>(c->stage.p);
  // ---- which units are emitted (template rule of the filter, commands/filter.rs:640-672: the consecutive
  //      units of one MI are emitted only if every one of them passed) ----
  std::vector<char> emit;
  auto unit_at = [&](uint64_t g, const DirectPlan** P) -> const DUnit& {
    const size_t i = static_cast<size_t>(std::upper_bound(ub.begin(), ub.end(), g) - ub.begin()) - 1;
    *P = &c->segs[i].ctx->dplan;
    return (*P)->units[c->segs[i].u0 + (g - ub[i])];
  };
  if (c->opt.filter_enabled) {
    emit.assign(U, 1);
    for (uint64_t i = 0; i < U;) {
      const DirectPlan* P0; const DUnit& u0 = unit_at(i, &P0);
      uint64_t j = i;
      bool pass = true;
      while (j < U) {
        const DirectPlan* Pj; const DUnit& uj = unit_at(j, &Pj);
        if (uj.umi.len != u0.umi.len || std::memcmp(stage + uj.umi.off, stage + u0.umi.off, u0.umi.len) != 0) break;
        pass = pass && fstatus[j] == FGB_FILTER_PASS;
        ++j;
      }
      for (uint64_t k = i; k < j; ++k) {
        emit[k] = pass;
        c->stats[FGB_STAT_FILTER_RECORDS] += 1;
        c->stats[FGB_STAT_FILTER_BASES_MASKED] += fmasked[k];
        if (pass) c->stats[FGB_STAT_FILTER_PASSED] += 1;
      }
      i = j;
    }
  }
  // ---- build_consensus_record_into (vanilla_caller.rs:1365-1473): pieces of segments, sized first, then
  //      written at their final place in one output buffer ----
  struct Piece { size_t seg; uint32_t u0, u1; uint64_t g0; size_t bytes; uint64_t count; };
  std::vector<Piece> pieces;
  {
    const uint64_t want = std::max<uint64_t>(256, U / (std::max<uint32_t>(c->opt.n_threads, 1u) * 4u) + 1);
    for (size_t i = 0; i < NS; ++i) {
      const DSeg& sg = c->segs[i];
      for (uint32_t u = sg.u0; u < sg.u1;) {
        const uint32_t e = static_cast<uint32_t>(std::min<uint64_t>(sg.u1, static_cast<uint64_t>(u) + want));
        pieces.push_back(Piece{i, u, e, ub[i] + (u - sg.u0), 0, 0});
        u = e;
      }
    }
  }
  const uint32_t TP = std::max<uint32_t>(1u, std::min<uint32_t>(std::max<uint32_t>(c->opt.n_threads, 1u), static_cast<uint32_t>(pieces.size())));
  auto for_pieces = [&](const std::function<void(size_t)>& fn) {
    if (TP <= 1) { for (size_t i = 0; i < pieces.size(); ++i) fn(i); return; }
    run_parallel(c, TP, [&](uint32_t t) {       // contiguous runs of pieces per thread
      const size_t a = pieces.size() * t / TP, e = pieces.size() * (t + 1) / TP;
      for (size_t i = a; i < e; ++i) fn(i);
    });
  };
  auto depth_stats = [&](uint64_t out_off, uint32_t L, uint32_t* mx, uint32_t* mn) {
    uint32_t a = 0, m = L ? 0xFFFFFFFFu : 0;
    if (narrow) { const uint8_t* d = static_cast<const uint8_t*>(c->pinned[2]) + out_off; for (uint32_t k = 0; k < L; ++k) { a = d[k] > a ? d[k] : a; m = d[k] < m ? d[k] : m; } }
    else { const uint16_t* d = static_cast<const uint16_t*>(c->pinned[2]) + out_off; for (uint32_t k = 0; k < L; ++k) { a = d[k] > a ? d[k] : a; m = d[k] < m ? d[k] : m; } }
    *mx = a; *mn = m;
  };
  for_pieces([&](size_t pi) {                     // pass 1: sizes
    Piece& pc = pieces[pi];
    const DirectPlan& P = c->segs[pc.seg].ctx->dplan;
    size_t bytes = 0; uint64_t count = 0;
    for (uint32_t u = pc.u0; u < pc.u1; ++u) {
      const uint64_t g = pc.g0 + (u - pc.u0);
      if (!emit.empty() && !emit[g]) continue;
      const DUnit& du = P.units[u];
      uint32_t sz = du.rec_size;
      if (!sz) {
        uint32_t mx, mn;
        depth_stats(g_units[g].out_off, du.cons_len, &mx, &mn);
        sz = simplex_record_size(c, du.cons_len, du.umi.len, du.has_cell, du.cell.len, du.rx_n > 0,
                                 du.rx_n ? P.rx[du.rx_begin].len : 0u, int_tag_width(mx), int_tag_width(mn));
      }
      bytes += sz; ++count;
    }
    pc.bytes = bytes; pc.count = count;
  });
  size_t total = 0;
  std::vector<size_t> at(pieces.size() + 1, 0);
  for (size_t i = 0; i < pieces.size(); ++i) { at[i] = total; total += pieces[i].bytes; c->out_count += pieces[i].count; }
  if (!ensure_joined(c, total)) return FGB_ERR_NOMEM;
  std::vector<fgb_status> pst(pieces.size(), FGB_OK);
  std::vector<std::string> perr(TP);
  trace.mark("sizes");
  for_pieces([&](size_t pi) {                     // pass 2: the records
    const Piece& pc = pieces[pi];
    const DirectPlan& P = c->segs[pc.seg].ctx->dplan;
    static thread_local std::string rx, err;
    uint8_t* dst = c->joined + at[pi];
    uint8_t* const end = dst + pc.bytes;
    for (uint32_t u = pc.u0; u < pc.u1; ++u) {
      const uint64_t g = pc.g0 + (u - pc.u0);
      if (!emit.empty() && !emit[g]) continue;
      const DUnit& du = P.units[u];
      const uint64_t oo = g_units[g].out_off;
      size_t n;
      if (narrow) n = write_simplex_record_at<uint8_t>(c, dst, du, P.rx.data() + du.rx_begin, stage, o_base + oo, o_qual + oo,
                                                       static_cast<const uint8_t*>(c->pinned[2]) + oo,
                                                       static_cast<const uint8_t*>(c->pinned[3]) + oo, &rx, &err);
      else n = write_simplex_record_at<uint16_t>(c, dst, du, P.rx.data() + du.rx_begin, stage, o_base + oo, o_qual + oo,
                                                 static_cast<const uint16_t*>(c->pinned[2]) + oo,
                                                 static_cast<const uint16_t*>(c->pinned[3]) + oo, &rx, &err);
      if (!n) { pst[pi] = FGB_ERR_INVALID_ARG; return; }
      dst += n;
      if (dst > end) { pst[pi] = FGB_ERR_INVALID_ARG; return; }      // cannot happen: sizes come from the same formula
    }
    if (dst != end) pst[pi] = FGB_ERR_INVALID_ARG;
  });
  for (size_t i = 0; i < pieces.size(); ++i)
    if (pst[i] != FGB_OK) {
      c->last_error = "consensus record assembly failed (read name too long, or RX values of a family have different "
                      "lengths or mix DNA and non-DNA characters)";
      return pst[i];
    }
  c->joined_len = total;
  c->out_is_joined = true;
  trace.mark("assemble");
  return FGB_OK;
}

// ------------------------------------------------------------------------------------------------
// threaded record assembly (duplex, CODEC)
// ------------------------------------------------------------------------------------------------
void ensure_workers(fgb_caller* c, uint32_t T) {
  while (c->workers.size() < T) {
    std::unique_ptr<fgb_caller> w(new fgb_caller());
    w->opt = c->opt; w->prefix = c->prefix; w->rg = c->rg; w->prep_opt = c->prep_opt;
    w->h = nullptr;                    // workers prepare and assemble; the vote happens in the parent
    c->workers.push_back(std::move(w));
  }
}

// Runs body(ctx, i0, i1) over [0, n): on the caller itself when one thread is enough, else on worker
// contexts (own record buffer, counters, error text) over contiguous ranges; buffers are joined in
// order, counters summed, and the first error in input order wins.
template <class Body>
fgb_status parallel_records(fgb_caller* c, uint64_t n, uint64_t min_per_thread, Body body) {
  const uint32_t T = static_cast<uint32_t>(std::min<uint64_t>(std::max<uint32_t>(c->opt.n_threads, 1u),
                                                               (n + min_per_thread - 1) / min_per_thread));
  if (T <= 1) return body(c, static_cast<uint64_t>(0), n);
  ensure_workers(c, T);
  std::vector<fgb_status> sts(T, FGB_OK);
  run_parallel(c, T, [&](uint32_t t) {
    fgb_caller* w = c->workers[t].get();
    w->out.clear(); w->out_count = 0; w->last_error.clear();
    sts[t] = body(w, n * t / T, n * (t + 1) / T);
  });
  size_t total = 0;
  std::vector<size_t> at(T, 0);
  fgb_status first = FGB_OK;
  for (uint32_t t = 0; t < T; ++t) {
    fgb_caller* w = c->workers[t].get();
    if (first == FGB_OK && sts[t] != FGB_OK) { first = sts[t]; c->last_error = w->last_error; }
    at[t] = total;
    total += w->out.size();
    c->out_count += w->out_count;
    for (int i = 0; i < FGB_NSTATS; ++i) { c->stats[i] += w->stats[i]; w->stats[i] = 0; }
  }
  if (first != FGB_OK) return first;
  if (!ensure_joined(c, total)) return FGB_ERR_NOMEM;
  run_parallel(c, T, [&](uint32_t t) {
    const auto& o = c->workers[t]->out;
    if (!o.empty()) std::memcpy(c->joined + at[t], o.data(), o.size());
  });
  c->joined_len = total;
  c->out_is_joined = true;
  return FGB_OK;
}

// ------------------------------------------------------------------------------------------------
// duplex
// ------------------------------------------------------------------------------------------------
bool paired_r1(const View& v) { return (v.flags() & bam::kPaired) && (v.flags() & bam::kFirst); }
bool paired_r2(const View& v) { return (v.flags() & bam::kPaired) && (v.flags() & bam::kLast); }

// has_minimum_number_of_reads / duplex_consensus_has_minimum_reads, duplex_caller.rs:731-769
bool min_reads_ok(const fgb_caller* c, size_t na, size_t nb) {
  size_t xy = na >= nb ? na : nb, yx = na >= nb ? nb : na;
  return c->opt.min_reads <= xy + yx && c->opt.min_xy_reads <= xy && c->opt.min_yx_reads <= yx;
}

bool all_same_strand(const std::vector<View>& recs, const std::vector<uint32_t>& a,
                     const std::vector<uint32_t>& b) {
  bool have = false, rev = false;
  for (const auto* grp : {&a, &b})
    for (uint32_t i : *grp) {
      bool r = recs[i].flags() & bam::kReverse;
      if (!have) { have = true; rev = r; }
      else if (r != rev) return false;
    }
  return true;
}

// duplex_caller.rs:2206-2250 (consensus_reads) + :576-630 + process_group :1719-1942
fgb_status add_group_duplex(fgb_caller* c, const std::vector<View>& recs) {
  const uint32_t n = static_cast<uint32_t>(recs.size());
  c->stats[FGB_STAT_TOTAL_READS] += n;
  std::vector<uint32_t> a, b;
  std::string base_mi, mi;
  bool have_mi = false;
  for (uint32_t i = 0; i < n; ++i) {   // partition_records_by_strand
    if (!get_string_tag(recs[i], "MI", &mi)) {
      c->last_error = "read is missing the MI tag (duplex requires 'group --strategy paired' input)";
      return FGB_ERR_MISSING_TAG;
    }
    if (!have_mi) { base_mi = mi.size() >= 2 ? mi.substr(0, mi.size() - 2) : mi; have_mi = true; }
    if (mi.size() >= 2 && mi[mi.size() - 2] == '/' && mi.back() == 'A') a.push_back(i);
    else if (mi.size() >= 2 && mi[mi.size() - 2] == '/' && mi.back() == 'B') b.push_back(i);
    else {
      c->last_error = "MI tag '" + mi + "' has no /A or /B suffix (duplex requires paired grouping)";
      return FGB_ERR_INVALID_ARG;
    }
  }
  if (a.empty() && b.empty()) return FGB_OK;
  const uint64_t n_input = a.size() + b.size();
  size_t na = 0, nb = 0;
  for (uint32_t i : a) na += paired_r1(recs[i]);
  for (uint32_t i : b) nb += paired_r1(recs[i]);
  if (!min_reads_ok(c, na, nb)) { reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, n_input); return FGB_OK; }
  Molecule m;
  m.base_mi = base_mi;
  m.n_input = static_cast<uint32_t>(n_input);
  if (c->opt.cell_tag[0]) {
    const View& first = !a.empty() ? recs[a[0]] : recs[b[0]];
    m.has_cell = get_string_tag(first, c->opt.cell_tag, &m.cell);
  }
  std::vector<uint32_t> ab_r1, ab_r2, ba_r1, ba_r2;
  for (uint32_t i : a) { if (paired_r1(recs[i])) ab_r1.push_back(i); if (paired_r2(recs[i])) ab_r2.push_back(i); }
  for (uint32_t i : b) { if (paired_r1(recs[i])) ba_r1.push_back(i); if (paired_r2(recs[i])) ba_r2.push_back(i); }
  if (!a.empty() && !b.empty()) {   // strand-orientation sanity, duplex_caller.rs:1799-1823
    if (!all_same_strand(recs, ab_r1, ba_r2) || !all_same_strand(recs, ab_r2, ba_r1)) {
      reject(c, FGB_STAT_REJ_POTENTIAL_COLLISION, n_input);
      return FGB_OK;
    }
  }
  // X = AB-R1 + BA-R2, Y = AB-R2 + BA-R1: pooled CIGAR filter, then split back (:1844-1892)
  // (the SourceRead buffers live in two pools that persist across groups: Prepared::srs / n)
  auto pooled = [&](const std::vector<uint32_t>& p, const std::vector<uint32_t>& q,
                    std::vector<uint32_t>* raws, Prepared* pool) {
    raws->clear(); pool->n = 0;
    raws->insert(raws->end(), p.begin(), p.end());
    raws->insert(raws->end(), q.begin(), q.end());
    for (uint32_t k = 0; k < raws->size(); ++k) {
      const View& v = recs[(*raws)[k]];
      bam::cigar_ops(v, &c->ops);
      size_t clip = bam::num_bases_extending_past_mate(v, c->ops);
      if (pool->n == pool->srs.size()) pool->srs.emplace_back();
      if (make_source_read(c->prep_opt, v, k, clip, &c->ops, &pool->srs[pool->n])) ++pool->n;
    }
    pool->n = filter_by_alignment_n(&pool->srs, pool->n);   // MinorityAlignment is counted by the ss caller, not the duplex stats
  };
  std::vector<uint32_t>&x_raws = c->scratch_idx[0], &y_raws = c->scratch_idx[1];
  Prepared &fx = c->prepared[0], &fy = c->prepared[1];
  pooled(ab_r1, ba_r2, &x_raws, &fx);
  pooled(ab_r2, ba_r1, &y_raws, &fy);
  // AB-R1, AB-R2, BA-R1, BA-R2 (per-thread scratch: eight heap vectors per group otherwise)
  static thread_local std::vector<const SourceRead*> grp[4];
  static thread_local std::vector<uint32_t> grp_raw[4];
  for (int g = 0; g < 4; ++g) { grp[g].clear(); grp_raw[g].clear(); }
  for (size_t i = 0; i < fx.n; ++i) { const SourceRead& sr = fx.srs[i]; int g = (sr.flags & bam::kFirst) ? 0 : 3; grp_raw[g].push_back(x_raws[sr.original_idx]); grp[g].push_back(&sr); }
  for (size_t i = 0; i < fy.n; ++i) { const SourceRead& sr = fy.srs[i]; int g = (sr.flags & bam::kFirst) ? 2 : 1; grp_raw[g].push_back(y_raws[sr.original_idx]); grp[g].push_back(&sr); }
  const bool have[4] = {!grp[0].empty(), !grp[1].empty(), !grp[2].empty(), !grp[3].empty()};
  // consensus_call succeeds iff the group is non-empty (min_reads = 1); arm selection :1986-2190
  if (have[0] && have[1] && have[2] && have[3]) m.pattern = 0;
  else if (have[0] && have[1] && !have[2] && !have[3] && c->opt.min_yx_reads == 0) m.pattern = 1;
  else if (!have[0] && !have[1] && have[2] && have[3] && c->opt.min_yx_reads == 0) m.pattern = 2;
  else { reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, n_input); return FGB_OK; }
  std::string rx;
  for (int g = 0; g < 4; ++g) {
    if (!have[g]) continue;
    m.unit[g] = c->pack.add_unit(grp[g], 1);
    for (uint32_t ri : grp_raw[g])
      if (get_string_tag(recs[ri], "RX", &rx)) m.rx[g].push_back(RxSource{rx, (recs[ri].flags() & bam::kFirst) != 0});
  }
  if (m.pattern == 0) {
    auto add_job = [&](uint32_t ua, uint32_t ub) {
      fgb_duplex_job j;
      j.unit_a = ua; j.unit_b = ub; j.out_off = c->n_duplex_out;
      uint32_t cap = std::max(c->pack.units[ua].cons_len, c->pack.units[ub].cons_len);
      c->n_duplex_out += round_up(cap, FGB_OUT_ALIGN);
      c->jobs.push_back(j);
      return static_cast<int32_t>(c->jobs.size() - 1);
    };
    m.job[0] = add_job(m.unit[0], m.unit[3]);   // duplex R1 = AB-R1 (+) BA-R2, :1999-2004
    m.job[1] = add_job(m.unit[1], m.unit[2]);   // duplex R2 = AB-R2 (+) BA-R1, :2008-2012
  }
  c->molecules.push_back(std::move(m));
  return FGB_OK;
}

// One strand's columns as seen by duplex_read_into (ab_consensus / ba_consensus).
struct Strand {
  const uint8_t* bases = nullptr;
  const uint8_t* quals = nullptr;
  const uint16_t* depths = nullptr;
  const uint16_t* errors = nullptr;
  uint32_t len = 0;
  bool present = false;
};

struct DuplexRead {
  const uint8_t* bases; const uint8_t* quals; const uint16_t* errors; uint32_t len;
  Strand ab, ba;
};

uint32_t max_depth(const Strand& s) {
  uint32_t m = 0;
  for (uint32_t i = 0; i < s.len; ++i) m = std::max<uint32_t>(m, s.depths[i]);
  return m;
}

// duplex_read_into, duplex_caller.rs:1048-1285 (methylation off)
fgb_status write_duplex_record(fgb_caller* c, bam::Writer* w, const DuplexRead& d, bool r1,
                               const Molecule& m, const std::vector<RxSource>& src_a,
                               const std::vector<RxSource>& src_b) {
  uint16_t flag = bam::kUnmapped | bam::kPaired | bam::kMateUnmapped | (r1 ? bam::kFirst : bam::kLast);
  std::string name = c->prefix + ":" + m.base_mi;
  if (name.size() >= 255) { c->last_error = "read name too long"; return FGB_ERR_INVALID_ARG; }
  w->begin(name, flag, d.bases, d.quals, d.len);
  w->str("MI", m.base_mi.data(), m.base_mi.size());
  if (m.has_cell) w->str(c->opt.cell_tag, m.cell.data(), m.cell.size());
  w->str("RG", c->rg.data(), c->rg.size());
  auto metrics = [](const Strand& s, int32_t* mx, int32_t* mn, float* er) {
    *mx = 0; *mn = 0; *er = 0.0f;
    if (!s.present) return;
    uint32_t lo = s.len ? 0xFFFFFFFFu : 0, hi = 0;
    uint64_t td = 0, te = 0;
    for (uint32_t i = 0; i < s.len; ++i) {
      hi = std::max<uint32_t>(hi, s.depths[i]); lo = std::min<uint32_t>(lo, s.depths[i]);
      td += s.depths[i]; te += s.errors[i];
    }
    *mx = static_cast<int32_t>(hi); *mn = static_cast<int32_t>(lo); *er = error_rate(te, td);
  };
  int32_t mx, mn; float er;
  metrics(d.ab, &mx, &mn, &er);
  w->integer("aD", mx); w->real("aE", er); w->integer("aM", mn);
  if (c->opt.produce_per_base_tags) {
    w->str("ac", d.ab.bases, d.ab.len);
    w->i16_array("ad", d.ab.depths, d.ab.len);
    w->i16_array("ae", d.ab.errors, d.ab.len);
    w->phred33("aq", d.ab.quals, d.ab.len);
  }
  metrics(d.ba, &mx, &mn, &er);
  w->integer("bD", mx); w->real("bE", er); w->integer("bM", mn);
  if (c->opt.produce_per_base_tags && d.ba.present) {
    w->str("bc", d.ba.bases, d.ba.len);
    w->i16_array("bd", d.ba.depths, d.ba.len);
    w->i16_array("be", d.ba.errors, d.ba.len);
    w->phred33("bq", d.ba.quals, d.ba.len);
  }
  int32_t cmx = 0, cmn = d.len ? 0x7FFFFFFF : 0;
  uint64_t td = 0, te = 0;
  for (uint32_t i = 0; i < d.len; ++i) {
    int32_t v = (i < d.ab.len ? d.ab.depths[i] : 0) + ((d.ba.present && i < d.ba.len) ? d.ba.depths[i] : 0);
    cmx = std::max(cmx, v); cmn = std::min(cmn, v);
    td += static_cast<uint64_t>(v); te += d.errors[i];
  }
  w->integer("cD", cmx); w->real("cE", error_rate(te, td)); w->integer("cM", cmn);
  // RX: orientation-aware reversal of the '-'-separated halves, :1187-1211
  std::vector<std::string> umis;
  auto collect = [&](const std::vector<RxSource>& src) {
    for (const auto& s : src) {
      if (s.first == r1) { umis.push_back(s.rx); continue; }
      std::vector<std::string> parts;
      size_t start = 0;
      for (;;) {
        size_t p = s.rx.find('-', start);
        if (p == std::string::npos) { parts.push_back(s.rx.substr(start)); break; }
        parts.push_back(s.rx.substr(start, p - start));
        start = p + 1;
      }
      std::string rev;
      for (size_t k = parts.size(); k-- > 0;) { rev += parts[k]; if (k) rev += '-'; }
      umis.push_back(rev);
    }
  };
  collect(src_a);
  collect(src_b);
  fgb_status st = append_rx(c, w, umis);
  if (st != FGB_OK) return st;
  w->end();
  ++c->out_count;
  return FGB_OK;
}

// `fgumi duplex | fgumi filter`, template mode (commands/filter.rs:640-672): the two records of the
// molecule start at `mark` in ctx->out; both are masked, and both are dropped unless both pass.
void filter_duplex_template(fgb_caller* ctx, size_t mark) {
  bool pass = true;
  size_t p = mark;
  while (p + 4 <= ctx->out.size()) {
    const uint32_t bs = bam::rd32(ctx->out.data() + p);
    uint32_t masked = 0;
    const int st = rfilter::filter_record(ctx->out.data() + p + 4, bs, ctx->opt.duplex_filter, &masked);
    ctx->stats[FGB_STAT_FILTER_RECORDS] += 1;
    ctx->stats[FGB_STAT_FILTER_BASES_MASKED] += masked;
    if (st != FGB_FILTER_PASS) pass = false;
    p += 4 + static_cast<size_t>(bs);
  }
  if (pass) ctx->stats[FGB_STAT_FILTER_PASSED] += 2;
  else { ctx->out.resize(mark); ctx->out_count -= 2; }
}

fgb_status flush_duplex(fgb_caller* c) {
  const uint64_t U = c->pack.units.size();
  if (!U) return FGB_OK;
  PhaseTrace trace;
  uint64_t n_bytes, R;
  c->pack.seal(&n_bytes, &R);
  uint64_t n_tiles = 0;
  fgb_status st = fgb_plan_tiles(c->pack.units.data(), U, c->pack.reads.data(), R, nullptr, 0, &n_tiles);
  if (st != FGB_OK) { c->last_error = "fgb_plan_tiles failed"; return st; }
  std::vector<fgb_tile> tiles(n_tiles ? n_tiles : 1);
  if ((st = fgb_plan_tiles(c->pack.units.data(), U, c->pack.reads.data(), R, tiles.data(), n_tiles, &n_tiles)) != FGB_OK) return st;
  const uint64_t no = c->pack.n_out, nd = c->n_duplex_out, nj = c->jobs.size();
  // result columns in page-locked memory that outlives the flush (no zero-fill, asynchronous copies back)
  const size_t want[8] = {no + 8, no + 8, 2 * (no + 8), 2 * (no + 8), nd + 8, nd + 8, 2 * (nd + 8), nj + 8};
  for (int i = 0; i < 8; ++i)
    if (c->px[i].ensure(want[i]) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
  struct P8 { uint8_t* p; uint8_t* data() const { return p; } uint8_t& operator[](size_t i) const { return p[i]; } };
  struct P16 { uint16_t* p; uint16_t* data() const { return p; } };
  const P8 sb{static_cast<uint8_t*>(c->px[0].p)}, sq{static_cast<uint8_t*>(c->px[1].p)};
  const P16 sd{static_cast<uint16_t*>(c->px[2].p)}, se{static_cast<uint16_t*>(c->px[3].p)};
  const P8 db{static_cast<uint8_t*>(c->px[4].p)}, dq{static_cast<uint8_t*>(c->px[5].p)};
  const P16 de{static_cast<uint16_t*>(c->px[6].p)};
  const P8 dst{static_cast<uint8_t*>(c->px[7].p)};
  fgb_batch b;
  std::memset(&b, 0, sizeof(b));
  b.n_units = U; b.n_reads = R; b.n_bytes = n_bytes; b.n_out = no; b.n_tiles = n_tiles;
  b.bases = c->pack.bases.data(); b.quals = c->pack.quals.data(); b.reads = c->pack.reads.data();
  b.units = c->pack.units.data(); b.tiles = tiles.data();
  fgb_columns ss{sb.data(), sq.data(), sd.data(), se.data()};
  fgb_duplex_out dout{db.data(), dq.data(), de.data(), dst.data()};
  if (nj) {                        // vote + strand combine in one call, buffers owned by the engine's slots
    fgb_submit_options so;
    std::memset(&so, 0, sizeof(so));
    so.input_format = FGB_IN_BYTES; so.output_format = FGB_OUT_U16;
    so.duplex_jobs = c->jobs.data(); so.n_duplex_jobs = nj; so.n_duplex_out = nd; so.duplex_out = &dout;
    st = fgb_submit_ex(c->h, &b, &ss, &so);
  } else {
    st = fgb_submit(c->h, &b, &ss);
  }
  trace.mark("seal + tiles + submit");
  if (st == FGB_OK) st = fgb_wait(c->h);
  trace.mark("wait");
  if (st != FGB_OK) {
    char buf[256];
    fgb_last_error(c->h, buf, sizeof(buf));
    c->last_error = buf;
    return st;
  }
  auto strand_of = [&](uint32_t unit, uint32_t len) {
    Strand s;
    const fgb_unit& u = c->pack.units[unit];
    s.bases = sb.data() + u.out_off; s.quals = sq.data() + u.out_off;
    s.depths = sd.data() + u.out_off; s.errors = se.data() + u.out_off;
    s.len = len; s.present = true;
    return s;
  };
  const fgb_status rst = parallel_records(c, c->molecules.size(), 128, [&](fgb_caller* ctx, uint64_t m0, uint64_t m1) -> fgb_status {
  // `ctx` owns the record buffer, the counters and the error text of this range; the voted columns,
  // jobs and molecules are the parent's (read-only here)
  fgb_status st = FGB_OK;
  bam::Writer w(&ctx->out);
  for (uint64_t mi = m0; mi < m1; ++mi) {
    const Molecule& m = c->molecules[mi];
    DuplexRead d[2];
    bool ok = true;
    if (m.pattern == 0) {
      const uint32_t ua[2] = {m.unit[0], m.unit[1]}, ub[2] = {m.unit[3], m.unit[2]};
      for (int k = 0; k < 2 && ok; ++k) {
        const fgb_duplex_job& j = c->jobs[m.job[k]];
        const uint32_t la = c->pack.units[ua[k]].cons_len, lb = c->pack.units[ub[k]].cons_len;
        const uint8_t status = dst[m.job[k]];
        DuplexRead& r = d[k];
        r.bases = db.data() + j.out_off; r.quals = dq.data() + j.out_off; r.errors = de.data() + j.out_off;
        if (status == FGB_DUPLEX_BOTH) {            // ab/ba truncated to the duplex length, :972-991
          r.len = std::min(la, lb);
          r.ab = strand_of(ua[k], r.len); r.ba = strand_of(ub[k], r.len);
        } else if (status == FGB_DUPLEX_A_ONLY) {   // :855-868
          r.len = la; r.ab = strand_of(ua[k], la); r.ba = Strand();
        } else if (status == FGB_DUPLEX_B_ONLY) {   // :869-882 (is_ba_only: BA sits in the ab slot)
          r.len = lb; r.ab = strand_of(ub[k], lb); r.ba = Strand();
        } else {
          ok = false;                               // duplex_consensus returned None
        }
      }
      if (ok) {   // duplex_consensus_has_minimum_reads on both reads, :2036-2047
        for (int k = 0; k < 2; ++k)
          if (!min_reads_ok(ctx, max_depth(d[k].ab), d[k].ba.present ? max_depth(d[k].ba) : 0)) ok = false;
      }
      if (!ok) { reject(ctx, FGB_STAT_REJ_INSUFFICIENT_READS, m.n_input); continue; }
      const size_t mark = ctx->out.size();
      if ((st = write_duplex_record(ctx, &w, d[0], true, m, m.rx[0], m.rx[3])) != FGB_OK) return st;
      if ((st = write_duplex_record(ctx, &w, d[1], false, m, m.rx[1], m.rx[2])) != FGB_OK) return st;
      ctx->stats[FGB_STAT_CONSENSUS_READS] += 1;
      if (c->opt.filter_enabled) filter_duplex_template(ctx, mark);
    } else {
      // single-strand molecule (min_yx_reads == 0): duplex_consensus(Some, None) keeps the strand
      // only if it has depth somewhere (:852-853)
      const uint32_t u1 = m.pattern == 1 ? m.unit[0] : m.unit[3];   // R1 from AB-R1 / BA-R2
      const uint32_t u2 = m.pattern == 1 ? m.unit[1] : m.unit[2];   // R2 from AB-R2 / BA-R1
      const uint32_t us[2] = {u1, u2};
      for (int k = 0; k < 2 && ok; ++k) {
        Strand s = strand_of(us[k], c->pack.units[us[k]].cons_len);
        if (max_depth(s) == 0) { ok = false; break; }
        d[k].bases = s.bases; d[k].quals = s.quals; d[k].errors = s.errors; d[k].len = s.len;
        d[k].ab = s; d[k].ba = Strand();
      }
      if (!ok) { reject(ctx, FGB_STAT_REJ_INSUFFICIENT_READS, m.n_input); continue; }
      static const std::vector<RxSource> kNone;
      const size_t mark = ctx->out.size();
      if (m.pattern == 1) {
        if ((st = write_duplex_record(ctx, &w, d[0], true, m, m.rx[0], kNone)) != FGB_OK) return st;
        if ((st = write_duplex_record(ctx, &w, d[1], false, m, m.rx[1], kNone)) != FGB_OK) return st;
      } else {
        if ((st = write_duplex_record(ctx, &w, d[0], true, m, kNone, m.rx[3])) != FGB_OK) return st;
        if ((st = write_duplex_record(ctx, &w, d[1], false, m, kNone, m.rx[2])) != FGB_OK) return st;
      }
      ctx->stats[FGB_STAT_CONSENSUS_READS] += 1;
      if (c->opt.filter_enabled) filter_duplex_template(ctx, mark);
    }
  }
  return FGB_OK;
  });
  trace.mark("records");
  return rst;
}


// ------------------------------------------------------------------------------------------------
// CODEC
// ------------------------------------------------------------------------------------------------
struct ClippedInfo {                 // ClippedRecordInfo, codec_caller.rs
  uint32_t raw_idx;
  size_t clip_amount;
  bool clip_from_start;
  size_t clipped_seq_len;
  std::vector<uint32_t> clipped_cigar;
  size_t adjusted_pos;
  uint16_t flags;
};

// build_clipped_info, codec_caller.rs:817-851
ClippedInfo clipped_info(fgb_caller* c, const View& v, uint32_t idx) {
  ClippedInfo ci;
  bam::cigar_ops(v, &c->ops);
  ci.clip_amount = bam::num_bases_extending_past_mate(v, c->ops);
  ci.raw_idx = idx;
  ci.flags = v.flags();
  ci.clip_from_start = v.flags() & bam::kReverse;
  size_t ref_consumed = 0;
  ci.clipped_cigar = bam::clip_cigar_ops(c->ops, ci.clip_amount, ci.clip_from_start, &ref_consumed);
  ci.clipped_seq_len = v.l_seq() > ci.clip_amount ? v.l_seq() - ci.clip_amount : 0;
  ci.adjusted_pos = static_cast<size_t>(v.pos() + 1) + (ci.clip_from_start ? ref_consumed : 0);
  return ci;
}

// filter_to_most_common_alignment_raw, codec_caller.rs:867-909
void codec_filter(fgb_caller* c, std::vector<ClippedInfo>* infos) {
  if (infos->size() < 2) return;
  std::vector<SourceRead> proxy(infos->size());   // reuse the shared grouping on (length, cigar)
  for (size_t i = 0; i < infos->size(); ++i) {
    bam::simplify_cigar((*infos)[i].clipped_cigar, &proxy[i].cigar);
    if ((*infos)[i].flags & bam::kReverse) std::reverse(proxy[i].cigar.begin(), proxy[i].cigar.end());
    proxy[i].bases.resize((*infos)[i].clipped_seq_len);
    proxy[i].original_idx = static_cast<uint32_t>(i);
  }
  size_t rejected = filter_by_alignment(&proxy);
  if (rejected) reject(c, FGB_STAT_REJ_MINORITY_ALIGNMENT, rejected);
  std::vector<ClippedInfo> kept;
  for (auto& p : proxy) kept.push_back(std::move((*infos)[p.original_idx]));
  infos->swap(kept);
}

// to_source_read_for_codec_raw, codec_caller.rs:414-469 (no masking, no trimming)
void codec_source_read(const View& v, const ClippedInfo& ci, SourceRead* sr) {
  // to_source_read_for_codec_raw, codec_caller.rs:414-469: decode, drop the virtual clip from one end,
  // reverse-complement negative-strand reads -- produced in one pass over the kept record positions
  const size_t l = v.l_seq();
  const size_t clip = std::min<size_t>(ci.clip_amount, l);
  const size_t lo = ci.clip_from_start ? clip : 0, hi = ci.clip_from_start ? l : l - clip;
  const size_t n = hi - lo;
  sr->bases.resize(n);
  sr->quals.resize(n);
  const uint8_t* s = v.b + v.seq_off();
  const uint8_t* q = v.b + v.qual_off();
  if (!(v.flags() & bam::kReverse)) {
    for (size_t i = 0; i < n; ++i) {
      const size_t j = lo + i;
      const uint8_t byte = s[j >> 1];
      sr->bases[i] = static_cast<uint8_t>(prep::kFwd[(j & 1) ? (byte & 0xF) : (byte >> 4)]);
    }
    if (n) std::memcpy(sr->quals.data(), q + lo, n);
  } else {
    for (size_t i = 0; i < n; ++i) {
      const size_t j = hi - 1 - i;
      const uint8_t byte = s[j >> 1];
      sr->bases[i] = static_cast<uint8_t>(prep::kRev[(j & 1) ? (byte & 0xF) : (byte >> 4)]);
    }
    std::reverse_copy(q + lo, q + hi, sr->quals.begin());
  }
  sr->flags = v.flags();
}

bool strict_utf8_string_tag(const View& v, const char tag[2], std::string* out) {
  const uint8_t* val; size_t n;
  if (!bam::find_string_tag(v, tag, &val, &n)) return false;
  if (!bam::valid_utf8(val, n)) return false;   // String::from_utf8(..).ok()
  out->assign(reinterpret_cast<const char*>(val), n);
  return true;
}

// consensus_reads_raw up to the vote, codec_caller.rs:531-745
fgb_status add_group_codec(fgb_caller* c, const std::vector<View>& recs) {
  const uint32_t n = static_cast<uint32_t>(recs.size());
  c->stats[FGB_STAT_TOTAL_READS] += n;
  CodecMolecule m;
  m.has_umi = get_string_tag(recs[0], "MI", &m.umi);
  std::vector<uint32_t> paired;
  size_t frag = 0;
  std::vector<uint32_t> ops;
  for (uint32_t i = 0; i < n; ++i) {   // phase 1
    const uint16_t f = recs[i].flags();
    if (!(f & bam::kPaired)) { ++frag; continue; }
    if (f & (bam::kSecondary | bam::kSupplementary | bam::kUnmapped)) continue;
    bam::cigar_ops(recs[i], &ops);
    if (!bam::is_fr_pair(recs[i], ops)) continue;
    paired.push_back(i);
  }
  if (frag) reject(c, FGB_STAT_REJ_FRAGMENT_READ, frag);
  if (paired.empty()) return FGB_OK;
  // phase 2: pair by read name in first-seen order
  struct NameGroup { const uint8_t* name; size_t len; std::vector<uint32_t> idx; };
  std::vector<NameGroup> groups;
  for (uint32_t i : paired) {
    const uint8_t* nm = recs[i].b + 32;
    size_t ln = recs[i].l_read_name() > 1 ? recs[i].l_read_name() - 1 : 0;
    bool found = false;
    for (auto& g : groups)
      if (g.len == ln && std::memcmp(g.name, nm, ln) == 0) { g.idx.push_back(i); found = true; break; }
    if (!found) groups.push_back(NameGroup{nm, ln, {i}});
  }
  std::vector<ClippedInfo> r1s, r2s;
  for (auto& g : groups) {
    if (g.idx.size() != 2) continue;
    uint32_t i1 = g.idx[0], i2 = g.idx[1];
    if (!(recs[i1].flags() & bam::kFirst)) std::swap(i1, i2);
    r1s.push_back(clipped_info(c, recs[i1], i1));
    r2s.push_back(clipped_info(c, recs[i2], i2));
  }
  if (r1s.empty()) return FGB_OK;
  const size_t min_reads = c->opt.min_reads;
  if (r1s.size() < min_reads) { reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, r1s.size() + r2s.size()); return FGB_OK; }
  codec_filter(c, &r1s);   // phase 3
  codec_filter(c, &r2s);
  if (r1s.empty() || r2s.empty()) return FGB_OK;
  if (r1s.size() < min_reads || r2s.size() < min_reads) {
    reject(c, FGB_STAT_REJ_INSUFFICIENT_READS, r1s.size() + r2s.size());
    return FGB_OK;
  }
  // phase 4: overlap / phase on the longest R1 and R2 (first maximum wins)
  auto longest = [](const std::vector<ClippedInfo>& v) {
    const ClippedInfo* best = nullptr;
    int32_t best_len = 0;
    for (const auto& ci : v) {
      int32_t rl = bam::reference_length(ci.clipped_cigar);
      if (!best || rl > best_len) { best = &ci; best_len = rl; }
    }
    return best;
  };
  const ClippedInfo* l1 = longest(r1s);
  const ClippedInfo* l2 = longest(r2s);
  const bool r1_neg = l1->flags & bam::kReverse;
  const ClippedInfo* lpos = r1_neg ? l2 : l1;
  const ClippedInfo* lneg = r1_neg ? l1 : l2;
  const size_t neg_start = lneg->adjusted_pos, pos_start = lpos->adjusted_pos;
  const int32_t prl = bam::reference_length(lpos->clipped_cigar);
  const size_t pos_ref_len = prl > 0 ? static_cast<size_t>(prl) : 0;
  const size_t pos_end = pos_start + (pos_ref_len > 0 ? pos_ref_len - 1 : 0);
  const size_t ov_start = neg_start, ov_end = pos_end;
  const int64_t duplex_length = static_cast<int64_t>(ov_end) - static_cast<int64_t>(ov_start) + 1;
  const uint64_t n_pairs = r1s.size() + r2s.size();
  if (duplex_length < static_cast<int64_t>(c->opt.min_duplex_length)) {
    reject(c, FGB_STAT_REJ_INSUFFICIENT_OVERLAP, n_pairs);
    return FGB_OK;
  }
  size_t a, b, cc, d;
  bool ok = bam::read_pos_at_ref_pos(l1->clipped_cigar, l1->adjusted_pos, ov_start, true, &a) &&
            bam::read_pos_at_ref_pos(l2->clipped_cigar, l2->adjusted_pos, ov_start, true, &b) &&
            bam::read_pos_at_ref_pos(l1->clipped_cigar, l1->adjusted_pos, ov_end, true, &cc) &&
            bam::read_pos_at_ref_pos(l2->clipped_cigar, l2->adjusted_pos, ov_end, true, &d);
  if (!ok || (static_cast<int64_t>(a) - static_cast<int64_t>(b)) != (static_cast<int64_t>(cc) - static_cast<int64_t>(d))) {
    reject(c, FGB_STAT_REJ_INDEL_ERROR, n_pairs);
    return FGB_OK;
  }
  const bool r2_neg = l2->flags & bam::kReverse;
  size_t pp, nn;
  if (!bam::read_pos_at_ref_pos(lpos->clipped_cigar, lpos->adjusted_pos, ov_end, false, &pp) ||
      !bam::read_pos_at_ref_pos(lneg->clipped_cigar, lneg->adjusted_pos, ov_end, false, &nn)) {
    reject(c, FGB_STAT_REJ_INDEL_ERROR, n_pairs);
    return FGB_OK;
  }
  const size_t cons_len = pp + lneg->clipped_seq_len - nn;
  // phase 5: the two single-strand units.  Their consensus length (min_reads = 1 -> longest row)
  // is known now, so the `consensus_length < ss length` rejection (:738-744) happens here.
  std::vector<SourceRead> s1(r1s.size()), s2(r2s.size());
  size_t len1 = 0, len2 = 0;
  for (size_t i = 0; i < r1s.size(); ++i) { codec_source_read(recs[r1s[i].raw_idx], r1s[i], &s1[i]); len1 = std::max(len1, s1[i].bases.size()); }
  for (size_t i = 0; i < r2s.size(); ++i) { codec_source_read(recs[r2s[i].raw_idx], r2s[i], &s2[i]); len2 = std::max(len2, s2[i].bases.size()); }
  for (const auto& sr : s1) if (sr.bases.empty()) { c->last_error = "CODEC read fully clipped"; return FGB_ERR_INVALID_ARG; }
  for (const auto& sr : s2) if (sr.bases.empty()) { c->last_error = "CODEC read fully clipped"; return FGB_ERR_INVALID_ARG; }
  if (cons_len < len1 || cons_len < len2) { reject(c, FGB_STAT_REJ_INDEL_ERROR, n_pairs); return FGB_OK; }
  if (cons_len > FGB_MAX_READ_LEN) { c->last_error = "CODEC consensus longer than 65535"; return FGB_ERR_UNIT_TOO_LARGE; }
  m.unit_r1 = c->pack.add_unit(s1, 1);
  m.unit_r2 = c->pack.add_unit(s2, 1);
  m.r1_negative = r1_neg;
  m.cons_len = static_cast<uint32_t>(cons_len);
  fgb_codec_job j;
  std::memset(&j, 0, sizeof(j));
  j.unit_a = m.unit_r1; j.unit_b = m.unit_r2;
  j.out_off = c->n_codec_out;
  j.len = m.cons_len;
  j.rc_a = r1_neg; j.rc_b = !r1_neg; j.rc_out = r1_neg;            // :746-750, :757-758
  j.pad_a_left = r1_neg ? static_cast<uint32_t>(cons_len - len1) : 0;   // pad_consensus(.., r1_is_negative)
  j.pad_b_left = r2_neg ? static_cast<uint32_t>(cons_len - len2) : 0;
  c->n_codec_out += round_up(cons_len, FGB_OUT_ALIGN);
  m.job = static_cast<uint32_t>(c->codec_jobs.size());
  c->codec_jobs.push_back(j);
  if (c->opt.cell_tag[0]) {   // first source read with a non-empty cell barcode, :1322-1332
    auto scan = [&](const std::vector<ClippedInfo>& v) {
      for (const auto& ci : v) {
        if (m.has_cell) return;
        std::string val;
        if (get_string_tag(recs[ci.raw_idx], c->opt.cell_tag, &val) && !val.empty()) { m.has_cell = true; m.cell = val; }
      }
    };
    scan(r1s); scan(r2s);
  }
  std::string rx;
  for (uint32_t i = 0; i < n; ++i) if (strict_utf8_string_tag(recs[i], "RX", &rx)) m.rx.push_back(rx);
  c->codec_molecules.push_back(std::move(m));
  return FGB_OK;
}

// One padded, oriented single strand as the record builder sees it (ss_for_ac / ss_for_bc).
struct PaddedStrand {
  std::vector<uint8_t> bases, quals;
  std::vector<uint16_t> depths, errors;
};

// reverse_complement_ss + pad_consensus (+ reverse_complement_ss again when R1 is negative),
// codec_caller.rs:507-520, 980-1023, 760-766
void padded_strand(const uint8_t* b, const uint8_t* q, const uint16_t* d, const uint16_t* e, uint32_t len,
                   bool rc_first, uint32_t pad_left, uint32_t total, bool rc_again, PaddedStrand* out) {
  out->bases.assign(total, 'n'); out->quals.assign(total, 0);
  out->depths.assign(total, 0); out->errors.assign(total, 0);
  for (uint32_t i = 0; i < len; ++i) {
    uint32_t s = rc_first ? len - 1 - i : i;
    out->bases[pad_left + i] = rc_first ? bam::complement(b[s]) : b[s];
    out->quals[pad_left + i] = q[s]; out->depths[pad_left + i] = d[s]; out->errors[pad_left + i] = e[s];
  }
  if (rc_again) {
    std::reverse(out->bases.begin(), out->bases.end());
    for (auto& x : out->bases) x = bam::complement(x);
    std::reverse(out->quals.begin(), out->quals.end());
    std::reverse(out->depths.begin(), out->depths.end());
    std::reverse(out->errors.begin(), out->errors.end());
  }
}

fgb_status flush_codec(fgb_caller* c) {
  const uint64_t U = c->pack.units.size();
  if (!U) return FGB_OK;
  uint64_t n_bytes, R;
  c->pack.seal(&n_bytes, &R);
  uint64_t n_tiles = 0;
  fgb_status st = fgb_plan_tiles(c->pack.units.data(), U, c->pack.reads.data(), R, nullptr, 0, &n_tiles);
  if (st != FGB_OK) { c->last_error = "fgb_plan_tiles failed"; return st; }
  std::vector<fgb_tile> tiles(n_tiles ? n_tiles : 1);
  if ((st = fgb_plan_tiles(c->pack.units.data(), U, c->pack.reads.data(), R, tiles.data(), n_tiles, &n_tiles)) != FGB_OK) return st;
  const uint64_t no = c->pack.n_out, nc = c->n_codec_out, nj = c->codec_jobs.size();
  const size_t want[11] = {no + 8, no + 8, 2 * (no + 8), 2 * (no + 8), nc + 8, nc + 8, 2 * (nc + 8), 2 * (nc + 8),
                           nj + 8, 4 * (nj + 2), 4 * (nj + 2)};
  for (int i = 0; i < 11; ++i)
    if (c->px[i].ensure(want[i]) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
  struct P8 { uint8_t* p; uint8_t* data() const { return p; } uint8_t& operator[](size_t i) const { return p[i]; } };
  struct P16 { uint16_t* p; uint16_t* data() const { return p; } };
  struct P32 { uint32_t* p; uint32_t* data() const { return p; } uint32_t& operator[](size_t i) const { return p[i]; } };
  const P8 sb{static_cast<uint8_t*>(c->px[0].p)}, sq{static_cast<uint8_t*>(c->px[1].p)};
  const P16 sd{static_cast<uint16_t*>(c->px[2].p)}, se{static_cast<uint16_t*>(c->px[3].p)};
  const P8 cb{static_cast<uint8_t*>(c->px[4].p)}, cq{static_cast<uint8_t*>(c->px[5].p)};
  const P16 cd{static_cast<uint16_t*>(c->px[6].p)}, ce{static_cast<uint16_t*>(c->px[7].p)};
  const P8 cst{static_cast<uint8_t*>(c->px[8].p)};
  const P32 dis{static_cast<uint32_t*>(c->px[9].p)}, dup{static_cast<uint32_t*>(c->px[10].p)};
  fgb_batch b;
  std::memset(&b, 0, sizeof(b));
  b.n_units = U; b.n_reads = R; b.n_bytes = n_bytes; b.n_out = no; b.n_tiles = n_tiles;
  b.bases = c->pack.bases.data(); b.quals = c->pack.quals.data(); b.reads = c->pack.reads.data();
  b.units = c->pack.units.data(); b.tiles = tiles.data();
  fgb_columns ss{sb.data(), sq.data(), sd.data(), se.data()};
  fgb_codec_out cout;
  cout.cols = fgb_columns{cb.data(), cq.data(), cd.data(), ce.data()};
  cout.status = cst.data(); cout.disagreements = dis.data(); cout.duplex_bases = dup.data();
  if (nj) {
    fgb_submit_options so;
    std::memset(&so, 0, sizeof(so));
    so.input_format = FGB_IN_BYTES; so.output_format = FGB_OUT_U16;
    so.codec_jobs = c->codec_jobs.data(); so.n_codec_jobs = nj; so.n_codec_out = nc;
    so.codec_params = &c->opt.codec; so.codec_out = &cout;
    st = fgb_submit_ex(c->h, &b, &ss, &so);
  } else {
    st = fgb_submit(c->h, &b, &ss);
  }
  if (st == FGB_OK) st = fgb_wait(c->h);
  if (st != FGB_OK) {
    char buf[256];
    fgb_last_error(c->h, buf, sizeof(buf));
    c->last_error = buf;
    return st;
  }
  // the record counter behind `prefix:<n>` names (codec_caller.rs:1236-1242) counts emitted records in
  // input order: number the survivors up front so that ranges can be assembled independently
  const uint64_t NM = c->codec_molecules.size();
  std::vector<uint64_t> ordinal(NM + 1, 0);
  for (uint64_t i = 0; i < NM; ++i)
    ordinal[i + 1] = ordinal[i] + (cst[c->codec_molecules[i].job] == FGB_CODEC_OK);
  const uint64_t counter0 = c->consensus_counter;
  c->consensus_counter += ordinal[NM];
  return parallel_records(c, NM, 128, [&](fgb_caller* ctx, uint64_t m0, uint64_t m1) -> fgb_status {
  bam::Writer w(&ctx->out);
  PaddedStrand sa, sbb;
  for (uint64_t mi = m0; mi < m1; ++mi) {
    const CodecMolecule& m = c->codec_molecules[mi];
    const fgb_codec_job& j = c->codec_jobs[m.job];
    if (dup[m.job] > 0) {   // counted before the gate, codec_caller.rs:1155-1158
      ctx->stats[FGB_STAT_DUPLEX_BASES] += dup[m.job];
      ctx->stats[FGB_STAT_DUPLEX_DISAGREEMENTS] += dis[m.job];
    }
    if (cst[m.job] != FGB_CODEC_OK) continue;   // "High duplex disagreement": the group is dropped
    const fgb_unit& u1 = c->pack.units[m.unit_r1];
    const fgb_unit& u2 = c->pack.units[m.unit_r2];
    const uint32_t L = m.cons_len;
    padded_strand(sb.data() + u1.out_off, sq.data() + u1.out_off, sd.data() + u1.out_off, se.data() + u1.out_off,
                  u1.cons_len, j.rc_a, j.pad_a_left, L, m.r1_negative, &sa);
    padded_strand(sb.data() + u2.out_off, sq.data() + u2.out_off, sd.data() + u2.out_off, se.data() + u2.out_off,
                  u2.cons_len, j.rc_b, j.pad_b_left, L, m.r1_negative, &sbb);
    // build_output_record_into, codec_caller.rs:1226-1368
    std::string name = c->prefix + ":" + (m.has_umi ? m.umi : std::to_string(counter0 + ordinal[mi] + 1));
    if (name.size() >= 255) { ctx->last_error = "read name too long"; return FGB_ERR_INVALID_ARG; }
    const uint8_t* bases = cb.data() + j.out_off;
    const uint8_t* quals = cq.data() + j.out_off;
    const uint16_t* errors = ce.data() + j.out_off;
    w.begin(name, bam::kUnmapped, bases, quals, L);
    w.str("RG", c->rg.data(), c->rg.size());
    if (m.has_umi) w.str("MI", m.umi.data(), m.umi.size());
    int32_t tmax = 0, tmin = L ? 0x7FFFFFFF : 0;
    int64_t tbases = 0; uint64_t terr = 0;
    for (uint32_t i = 0; i < L; ++i) {
      int32_t t = static_cast<int32_t>(sa.depths[i]) + static_cast<int32_t>(sbb.depths[i]);
      tmax = std::max(tmax, t); tmin = std::min(tmin, t); tbases += t; terr += errors[i];
    }
    w.integer("cD", tmax); w.integer("cM", tmin);
    w.real("cE", tbases > 0 ? static_cast<float>(terr) / static_cast<float>(static_cast<int32_t>(tbases)) : 0.0f);
    auto strand_tags = [&](const PaddedStrand& s, const char* dt, const char* mt, const char* et) {
      int32_t mx = 0, mn = L ? 0x7FFFFFFF : 0;
      uint64_t te = 0, tb = 0;
      for (uint32_t i = 0; i < L; ++i) {
        mx = std::max<int32_t>(mx, s.depths[i]); mn = std::min<int32_t>(mn, s.depths[i]);
        te += s.errors[i]; tb += s.depths[i];
      }
      w.integer(dt, mx); w.integer(mt, mn); w.real(et, error_rate(te, tb));
    };
    strand_tags(sa, "aD", "aM", "aE");
    strand_tags(sbb, "bD", "bM", "bE");
    if (c->opt.produce_per_base_tags) {   // `d as i16`: wrapping, not clamping (:1299-1309)
      w.i16_array_wrap("ad", sa.depths.data(), L); w.i16_array_wrap("bd", sbb.depths.data(), L);
      w.i16_array_wrap("ae", sa.errors.data(), L); w.i16_array_wrap("be", sbb.errors.data(), L);
      w.str("ac", sa.bases.data(), L); w.str("bc", sbb.bases.data(), L);
      w.phred33("aq", sa.quals.data(), L); w.phred33("bq", sbb.quals.data(), L);
    }
    if (m.has_cell) w.str(c->opt.cell_tag, m.cell.data(), m.cell.size());
    if (!m.rx.empty()) {
      std::string rx;
      if (!consensus_umis(c->umi_builder, m.rx, &rx)) {
        ctx->last_error = "RX values of a family have different lengths or mix DNA and non-DNA characters";
        return FGB_ERR_INVALID_ARG;
      }
      if (!rx.empty()) w.str("RX", rx.data(), rx.size());
    }
    w.end();
    ++ctx->out_count;
    ctx->stats[FGB_STAT_CONSENSUS_READS] += 1;
  }
  return FGB_OK;
  });
}

}  // namespace

namespace {
fgb_status direct_add(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off, const uint64_t* group_rec,
                      uint64_t n_groups);
}

extern "C" {

static fgb_status caller_create_impl(int device, const fgb_caller_options* opt, fgb_caller** out) {
  if (!opt || !out || !opt->read_name_prefix || !opt->read_group_id) return FGB_ERR_INVALID_ARG;
  *out = nullptr;
  if (opt->mode > FGB_MODE_CODEC) return FGB_ERR_INVALID_ARG;
  if (opt->mode != FGB_MODE_DUPLEX && opt->min_reads == 0) return FGB_ERR_INVALID_ARG;
  if (opt->filter_enabled && opt->mode == FGB_MODE_CODEC) return FGB_ERR_INVALID_ARG;
  if (opt->track_rejects && opt->mode != FGB_MODE_SIMPLEX) return FGB_ERR_INVALID_ARG;   // the simplex caller's reject sites only
  if (opt->filter_enabled && opt->mode == FGB_MODE_DUPLEX) {
    const fgb_duplex_filter_params& f = opt->duplex_filter;
    const double rates[] = {f.cc.max_read_error_rate, f.cc.max_base_error_rate, f.ab_max_read_error_rate,
                            f.ab_max_base_error_rate, f.ba_max_read_error_rate, f.ba_max_base_error_rate};
    for (double r : rates) if (!(r >= 0.0 && r <= 1.0)) return FGB_ERR_INVALID_ARG;     // commands/filter.rs:975-1000
    if (!(f.cc.max_no_call_fraction >= 0.0) || f.cc.min_base_quality > 255 || f.cc.min_base_quality < -1)
      return FGB_ERR_INVALID_ARG;
    // stringency order (commands/filter.rs:965-972): min-reads ba <= ab <= cc, error rates ab <= ba
    if (f.ba_min_reads > f.ab_min_reads || f.ab_min_reads > f.cc.min_reads ||
        f.ab_max_read_error_rate > f.ba_max_read_error_rate || f.ab_max_base_error_rate > f.ba_max_base_error_rate)
      return FGB_ERR_INVALID_ARG;
  }
  if (opt->mode == FGB_MODE_CODEC && opt->consensus_call_overlapping_bases)
    return FGB_ERR_INVALID_ARG;   // "CODEC does not support overlapping consensus", commands/codec.rs:257
  if (opt->mode == FGB_MODE_DUPLEX &&
      (opt->min_xy_reads > opt->min_reads || opt->min_yx_reads > opt->min_xy_reads))
    return FGB_ERR_INVALID_ARG;   // "min-reads values must be specified high to low", duplex_caller.rs:385-395
  std::unique_ptr<fgb_caller> c(new fgb_caller());
  c->opt = *opt;
  c->prefix = opt->read_name_prefix;
  c->rg = opt->read_group_id;
  c->opt.read_name_prefix = nullptr;
  c->opt.read_group_id = nullptr;
  c->prep_opt.min_input_base_quality = opt->min_input_base_quality;
  c->prep_opt.trim = opt->trim != 0;
  fgb_params p;
  p.error_rate_pre_umi = opt->error_rate_pre_umi;
  p.error_rate_post_umi = opt->error_rate_post_umi;
  p.reserved0 = 0;
  if (opt->mode == FGB_MODE_SIMPLEX) {
    p.min_consensus_base_quality = opt->min_consensus_base_quality;
    p.min_reads = opt->min_reads;
  } else if (opt->mode == FGB_MODE_DUPLEX) {   // single-strand caller of the duplex caller, duplex_caller.rs:397-412
    p.min_consensus_base_quality = 2;
    p.min_reads = 1;
  } else {   // single-strand caller of the CODEC caller, codec_caller.rs:326-339
    p.min_consensus_base_quality = 0;
    p.min_reads = 1;
  }
  if (device != FGB_DEVICE_NONE) {       // FGB_DEVICE_NONE: planning only, flush refuses (no CPU fallback)
    fgb_status st = fgb_create(device, &p, &c->h);
    if (st != FGB_OK) return st;
  } else {                               // what a planning-only simplex caller stages and lays out lives on the heap
    for (PinBuf* b : {&c->stage, &c->d_reads, &c->d_raws, &c->d_units}) b->pageable = true;
  }
  *out = c.release();
  return FGB_OK;
}

fgb_status fgb_caller_take_rejects(fgb_caller* c, const uint8_t** data, uint64_t* len, uint64_t* count) {
  if (!c || !data || !len || !count) return FGB_ERR_INVALID_ARG;
  c->rejects_taken.swap(c->rejects);
  c->rejects.clear();
  c->reject_taken_count = c->reject_count;
  c->reject_count = 0;
  *data = c->rejects_taken.data();
  *len = c->rejects_taken.size();
  *count = c->reject_taken_count;
  return FGB_OK;
}

static fgb_status caller_pending_impl(const fgb_caller* c, fgb_batch* batch, const fgb_duplex_job** duplex_jobs,
                                      uint64_t* n_duplex_jobs, const fgb_codec_job** codec_jobs,
                                      uint64_t* n_codec_jobs) {
  if (!c || !batch) return FGB_ERR_INVALID_ARG;
  if (c->opt.mode == FGB_MODE_SIMPLEX && !c->h) {
    // planning only: the queued plans laid out as the flush lays them out, each row decoded from its staged record
    // the way the device builds it (a caller with a device reports the empty Packer: its rows exist on the device only)
    DLayout L;
    const fgb_status st = lay_out_direct(c, &L);
    if (st != FGB_OK) return st;
    Packer& pk = c->pack;
    pk.reads.assign(L.reads, L.reads + L.R);
    pk.units.assign(L.units, L.units + L.U);
    pk.n_out = L.n_out;
    pk.bases.assign(L.n_bytes, 0);
    pk.quals.assign(L.n_bytes, 0);
    const uint8_t* const stage = static_cast<const uint8_t*>(c->stage.p);
    for (uint64_t r = 0; r < L.R; ++r) {
      const uint64_t off = FGB_READ_OFF(L.reads[r]);
      decode_source_row(stage + L.raws[r].src_off, L.raws[r].raw_len, L.raws[r].flags & FGB_RAW_REVERSE, FGB_READ_LEN(L.reads[r]),
                        c->prep_opt.min_input_base_quality, pk.bases.data() + off, pk.quals.data() + off);
    }
  }
  std::memset(batch, 0, sizeof(*batch));
  batch->n_units = c->pack.units.size();
  batch->n_reads = c->pack.reads.size();
  batch->n_bytes = c->pack.bases.size();
  batch->n_out = c->pack.n_out;
  batch->bases = c->pack.bases.data();
  batch->quals = c->pack.quals.data();
  batch->reads = c->pack.reads.data();
  batch->units = c->pack.units.data();
  if (duplex_jobs) *duplex_jobs = c->jobs.data();
  if (n_duplex_jobs) *n_duplex_jobs = c->jobs.size();
  if (codec_jobs) *codec_jobs = c->codec_jobs.data();
  if (n_codec_jobs) *n_codec_jobs = c->codec_jobs.size();
  return FGB_OK;
}

void fgb_caller_destroy(fgb_caller* c) {
  if (!c) return;
  for (void* p : c->pinned) fgb_host_free(p);
  c->stage.release(); c->d_reads.release(); c->d_raws.release(); c->d_units.release(); c->d_oruns.release(); c->d_recjobs.release(); c->d_recstr.release();
  for (PinBuf& b : c->px) b.release();
  fgb_host_free(c->joined);
  fgb_destroy(c->h);
  delete c;
}

size_t fgb_caller_last_error(const fgb_caller* c, char* buf, size_t buf_len) {
  if (!c) return 0;
  if (buf && buf_len) {
    size_t n = std::min(buf_len - 1, c->last_error.size());
    std::memcpy(buf, c->last_error.data(), n);
    buf[n] = 0;
  }
  return c->last_error.size();
}

static fgb_status caller_add_group_impl(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off,
                                uint32_t n_records) {
  if (!c || (n_records && (!records || !rec_off))) return FGB_ERR_INVALID_ARG;
  if (n_records == 0) return FGB_OK;
  if (c->opt.mode == FGB_MODE_SIMPLEX) {
    const uint64_t grp[2] = {0, n_records};
    return direct_add(c, records, rec_off, grp, 1);
  }
  std::vector<View> recs;
  recs.reserve(n_records);
  for (uint32_t i = 0; i < n_records; ++i) {
    if (rec_off[i + 1] < rec_off[i]) { c->last_error = "record offsets must ascend"; return FGB_ERR_LAYOUT; }
    size_t len = static_cast<size_t>(rec_off[i + 1] - rec_off[i]);
    if (len < 32) { c->last_error = "BAM record shorter than its fixed header"; return FGB_ERR_INVALID_ARG; }
    recs.emplace_back(records + rec_off[i], len);
    if (recs.back().aux_off() > len) { c->last_error = "truncated BAM record"; return FGB_ERR_INVALID_ARG; }
    if (recs.back().l_seq() > FGB_MAX_READ_LEN) {      // a row descriptor holds 16 bits of length
      c->last_error = "a read is longer than 65535 bases (FGB_MAX_READ_LEN)";
      return FGB_ERR_UNIT_TOO_LARGE;
    }
  }
  if (n_records > 0xFFFFu) {                                        // u16 observation counters (base_builder.rs:236): say so
    c->last_error = "an MI group has more than 65535 reads";       // now, not at flush time with every other group queued
    return FGB_ERR_UNIT_TOO_LARGE;
  }
  if (c->opt.consensus_call_overlapping_bases) {   // simplex.rs:395-398, duplex.rs:464-467
    const uint64_t base = rec_off[0], total = rec_off[n_records] - base;
    c->group_copy.assign(records + base, records + base + total);
    std::vector<uint64_t> off(n_records + 1);
    for (uint32_t i = 0; i <= n_records; ++i) off[i] = rec_off[i] - base;
    c->overlap.apply_group(c->group_copy.data(), off.data(), n_records);
    for (uint32_t i = 0; i < n_records; ++i) recs[i] = View(c->group_copy.data() + off[i], off[i + 1] - off[i]);
  }
  if (c->opt.mode == FGB_MODE_DUPLEX) return add_group_duplex(c, recs);
  return add_group_codec(c, recs);
}

}  // extern "C"

namespace {

// Below this many column bytes the serial merge is cheaper than starting threads for it
// (FGB_PARALLEL_MERGE_BYTES overrides: tests set it to 0 to exercise the threaded merge on small inputs).
const size_t kParallelMergeBytes = []() { const char* e = std::getenv("FGB_PARALLEL_MERGE_BYTES"); return e ? static_cast<size_t>(std::strtoull(e, nullptr, 10)) : (size_t{4} << 20); }();

// Appends everything a worker queued to the parent, in order, fixing up the offsets and indices that
// are relative to the worker's own batch.
void merge_worker(fgb_caller* c, fgb_caller* w) {
  const uint64_t byte_base = c->pack.bases.size();
  const uint32_t read_base = static_cast<uint32_t>(c->pack.reads.size());
  const uint32_t unit_base = static_cast<uint32_t>(c->pack.units.size());
  const uint64_t out_base = c->pack.n_out;
  c->pack.bases.insert(c->pack.bases.end(), w->pack.bases.begin(), w->pack.bases.end());
  c->pack.quals.insert(c->pack.quals.end(), w->pack.quals.begin(), w->pack.quals.end());
  for (uint64_t d : w->pack.reads) c->pack.reads.push_back(FGB_READ_DESC(FGB_READ_OFF(d) + byte_base, FGB_READ_LEN(d)));
  for (fgb_unit u : w->pack.units) { u.out_off += out_base; u.read_begin += read_base; c->pack.units.push_back(u); }
  c->pack.n_out += w->pack.n_out;
  // duplex
  const int32_t job_base = static_cast<int32_t>(c->jobs.size());
  for (fgb_duplex_job j : w->jobs) { j.unit_a += unit_base; j.unit_b += unit_base; j.out_off += c->n_duplex_out; c->jobs.push_back(j); }
  c->n_duplex_out += w->n_duplex_out;
  for (auto& m : w->molecules) {
    for (auto& u : m.unit) if (u != 0xFFFFFFFFu) u += unit_base;
    for (auto& j : m.job) if (j >= 0) j += job_base;
    c->molecules.push_back(std::move(m));
  }
  // CODEC
  const uint32_t cjob_base = static_cast<uint32_t>(c->codec_jobs.size());
  for (fgb_codec_job j : w->codec_jobs) { j.unit_a += unit_base; j.unit_b += unit_base; j.out_off += c->n_codec_out; c->codec_jobs.push_back(j); }
  c->n_codec_out += w->n_codec_out;
  for (auto& m : w->codec_molecules) { m.unit_r1 += unit_base; m.unit_r2 += unit_base; m.job += cjob_base; c->codec_molecules.push_back(std::move(m)); }
  for (int i = 0; i < FGB_NSTATS; ++i) c->stats[i] += w->stats[i];
  c->overlap.stats.overlapping_bases += w->overlap.stats.overlapping_bases;
  c->overlap.stats.bases_agreeing += w->overlap.stats.bases_agreeing;
  c->overlap.stats.bases_disagreeing += w->overlap.stats.bases_disagreeing;
  c->overlap.stats.bases_corrected += w->overlap.stats.bases_corrected;
  c->rejects.insert(c->rejects.end(), w->rejects.begin(), w->rejects.end());
  c->reject_count += w->reject_count;
  w->rejects.clear(); w->reject_count = 0;
  w->pack.clear(); w->molecules.clear(); w->jobs.clear();
  w->codec_molecules.clear(); w->codec_jobs.clear();
  w->n_duplex_out = 0; w->n_codec_out = 0;
  std::memset(w->stats, 0, sizeof(w->stats));
  w->overlap.stats = overlap::Stats();
}

// merge_worker for all workers at once, with the big copies on the workers' own threads: the parent's
// containers are sized once (the byte columns without zero-fill), every worker then writes its slice at
// a precomputed offset with the same fix-ups merge_worker applies.  Byte-identical to the serial merge.
void merge_workers_parallel(fgb_caller* c, uint32_t T) {
  struct Base { size_t bytes, reads, units, jobs, mols, cjobs, cmols; uint64_t out, dout, cout; };
  std::vector<Base> b(T + 1);
  b[0] = Base{c->pack.bases.size(), c->pack.reads.size(), c->pack.units.size(), c->jobs.size(),
              c->molecules.size(), c->codec_jobs.size(), c->codec_molecules.size(), c->pack.n_out,
              c->n_duplex_out, c->n_codec_out};
  for (uint32_t t = 0; t < T; ++t) {
    const fgb_caller* w = c->workers[t].get();
    b[t + 1] = Base{b[t].bytes + w->pack.bases.size(), b[t].reads + w->pack.reads.size(), b[t].units + w->pack.units.size(),
                    b[t].jobs + w->jobs.size(), b[t].mols + w->molecules.size(),
                    b[t].cjobs + w->codec_jobs.size(), b[t].cmols + w->codec_molecules.size(),
                    b[t].out + w->pack.n_out, b[t].dout + w->n_duplex_out, b[t].cout + w->n_codec_out};
  }
  c->pack.bases.resize(b[T].bytes);
  c->pack.quals.resize(b[T].bytes);
  c->pack.reads.resize(b[T].reads);
  c->pack.units.resize(b[T].units);
  c->jobs.resize(b[T].jobs);
  c->molecules.resize(b[T].mols);
  c->codec_jobs.resize(b[T].cjobs);
  c->codec_molecules.resize(b[T].cmols);
  auto copy_one = [&](uint32_t t) {
    fgb_caller* w = c->workers[t].get();
    const Base& o = b[t];
    if (!w->pack.bases.empty()) {
      std::memcpy(c->pack.bases.data() + o.bytes, w->pack.bases.data(), w->pack.bases.size());
      std::memcpy(c->pack.quals.data() + o.bytes, w->pack.quals.data(), w->pack.quals.size());
    }
    for (size_t i = 0; i < w->pack.reads.size(); ++i) {
      const uint64_t d = w->pack.reads[i];
      c->pack.reads[o.reads + i] = FGB_READ_DESC(FGB_READ_OFF(d) + o.bytes, FGB_READ_LEN(d));
    }
    for (size_t i = 0; i < w->pack.units.size(); ++i) {
      fgb_unit u = w->pack.units[i];
      u.out_off += o.out; u.read_begin += static_cast<uint32_t>(o.reads);
      c->pack.units[o.units + i] = u;
    }
    for (size_t i = 0; i < w->jobs.size(); ++i) {
      fgb_duplex_job j = w->jobs[i];
      j.unit_a += static_cast<uint32_t>(o.units); j.unit_b += static_cast<uint32_t>(o.units); j.out_off += o.dout;
      c->jobs[o.jobs + i] = j;
    }
    for (size_t i = 0; i < w->molecules.size(); ++i) {
      Molecule& m = w->molecules[i];
      for (auto& u : m.unit) if (u != 0xFFFFFFFFu) u += static_cast<uint32_t>(o.units);
      for (auto& j : m.job) if (j >= 0) j += static_cast<int32_t>(o.jobs);
      c->molecules[o.mols + i] = std::move(m);
    }
    for (size_t i = 0; i < w->codec_jobs.size(); ++i) {
      fgb_codec_job j = w->codec_jobs[i];
      j.unit_a += static_cast<uint32_t>(o.units); j.unit_b += static_cast<uint32_t>(o.units); j.out_off += o.cout;
      c->codec_jobs[o.cjobs + i] = j;
    }
    for (size_t i = 0; i < w->codec_molecules.size(); ++i) {
      CodecMolecule& m = w->codec_molecules[i];
      m.unit_r1 += static_cast<uint32_t>(o.units); m.unit_r2 += static_cast<uint32_t>(o.units);
      m.job += static_cast<uint32_t>(o.cjobs);
      c->codec_molecules[o.cmols + i] = std::move(m);
    }
  };
  run_parallel(c, T, copy_one);
  c->pack.n_out = b[T].out;
  c->n_duplex_out = b[T].dout;
  c->n_codec_out = b[T].cout;
  for (uint32_t t = 0; t < T; ++t) {          // counters, then reset the worker like merge_worker does
    fgb_caller* w = c->workers[t].get();
    for (int i = 0; i < FGB_NSTATS; ++i) c->stats[i] += w->stats[i];
    c->overlap.stats.overlapping_bases += w->overlap.stats.overlapping_bases;
    c->overlap.stats.bases_agreeing += w->overlap.stats.bases_agreeing;
    c->overlap.stats.bases_disagreeing += w->overlap.stats.bases_disagreeing;
    c->overlap.stats.bases_corrected += w->overlap.stats.bases_corrected;
    c->rejects.insert(c->rejects.end(), w->rejects.begin(), w->rejects.end());
    c->reject_count += w->reject_count;
    w->rejects.clear(); w->reject_count = 0;
    w->pack.clear(); w->molecules.clear(); w->jobs.clear();
    w->codec_molecules.clear(); w->codec_jobs.clear();
    w->n_duplex_out = 0; w->n_codec_out = 0;
    std::memset(w->stats, 0, sizeof(w->stats));
    w->overlap.stats = overlap::Stats();
  }
}

}  // namespace

namespace {

// The simplex caller's add: stages the records of groups [0, n_groups) (one contiguous slice of the blob) in
// page-locked memory (ordinary heap memory without a device) and plans them, on options.n_threads threads over
// contiguous ranges of groups.  All or nothing: on an error nothing of this call stays queued (the same for one
// thread and for many).
fgb_status direct_add(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off, const uint64_t* group_rec,
                      uint64_t n_groups) {
  const uint64_t rec0 = group_rec[0], rec1 = group_rec[n_groups];
  if (rec1 < rec0) { c->last_error = "bad group_rec table"; return FGB_ERR_INVALID_ARG; }
  const uint64_t b0 = rec_off[rec0], b1 = rec_off[rec1];
  if (b1 < b0) { c->last_error = "record offsets must ascend"; return FGB_ERR_LAYOUT; }
  // zero-copy batches: the records are shipped from the caller's own page-locked blob (decided by the first add
  // of a batch); otherwise this call's slice of the blob is staged in page-locked memory owned by the caller object
  if (c->h && c->opt.zero_copy_records && c->segs.empty() && c->stage_len == 0 && !c->zc_base && fgb_host_is_pinned(records) &&
      !(c->opt.consensus_call_overlapping_bases && (c->prep_opt.trim || c->opt.track_rejects)))   // those run the pre-pass on the host, in the staged copy
    c->zc_base = records;
  const bool zc = c->zc_base != nullptr;
  if (zc && records != c->zc_base) {
    c->last_error = "zero_copy_records: every add call of a batch must pass the same records pointer";
    return FGB_ERR_INVALID_ARG;
  }
  const size_t dst0 = zc ? static_cast<size_t>(b0) : round_up(c->stage_len, 64);
  if (!zc && c->stage.ensure(dst0 + (b1 - b0) + 256, c->stage_len) != FGB_OK) { c->last_error = "out of page-locked memory"; return FGB_ERR_NOMEM; }
  uint8_t* const stage = zc ? const_cast<uint8_t*>(c->zc_base) : static_cast<uint8_t*>(c->stage.p);   // never written in zero-copy mode
  const uint64_t n_rec = rec1 - rec0;
  const uint32_t T = static_cast<uint32_t>(std::min<uint64_t>(std::max<uint32_t>(c->opt.n_threads, 1u), (n_groups + 63) / 64));
  if (T > 1) ensure_workers(c, T);
  std::vector<uint64_t> cut(T + 1, n_groups);
  cut[0] = 0;
  for (uint32_t t = 1; t < T; ++t) {          // contiguous ranges balanced by record count
    const uint64_t target = rec0 + n_rec * t / T;
    cut[t] = static_cast<uint64_t>(std::lower_bound(group_rec, group_rec + n_groups, target) - group_rec);
    if (cut[t] < cut[t - 1]) cut[t] = cut[t - 1];
  }
  std::vector<fgb_caller*> ctx(T);
  std::vector<DMark> mark(T);
  for (uint32_t t = 0; t < T; ++t) {
    ctx[t] = T > 1 ? c->workers[t].get() : c;
    const DirectPlan& P = ctx[t]->dplan;
    mark[t] = DMark{P.raws.size(), P.units.size(), P.rx.size(), P.oruns.size(), P.row_bytes, P.out_elems, P.rec_bytes, P.str_bytes,
                    ctx[t]->rejects.size(), ctx[t]->reject_count};
  }
  uint64_t stats0[FGB_NSTATS];
  std::memcpy(stats0, c->stats, sizeof(stats0));
  const overlap::Stats ostats0 = c->overlap.stats;
  std::vector<fgb_status> sts(T, FGB_OK);
  auto run = [&](uint32_t t) {
    fgb_caller* x = ctx[t];
    const uint64_t g0 = cut[t], g1 = cut[t + 1];
    if (g0 >= g1) return;
    const uint64_t s0 = rec_off[group_rec[g0]], s1 = rec_off[group_rec[g1]];
    if (s1 < s0 || s0 < b0 || s1 > b1) { x->last_error = "record offsets must ascend"; sts[t] = FGB_ERR_LAYOUT; return; }
    if (!zc) std::memcpy(stage + dst0 + (s0 - b0), records + s0, s1 - s0);
    for (uint64_t g = g0; g < g1; ++g) {
      const uint64_t r0 = group_rec[g], r1 = group_rec[g + 1];
      if (r1 < r0 || r1 - r0 > 0xFFFFFFFFull || r1 > rec1) { x->last_error = "bad group_rec table"; sts[t] = FGB_ERR_INVALID_ARG; return; }
      const uint32_t n = static_cast<uint32_t>(r1 - r0);
      if (n == 0) continue;
      // The group rules read a record's fixed header, the start of its name / CIGAR and, at its end, the quality tail
      // and the aux area: three or four cache lines ~300 bytes apart per record, a miss each at DRAM latency.  Ask for
      // those lines of the NEXT group's records now (offsets beyond this worker's slice are simply not asked for).
      if (g + 1 < g1) {
        const uint64_t p0 = r1, p1 = std::min<uint64_t>(std::min<uint64_t>(group_rec[g + 2], p0 + 32), rec1);   // (r1 <= rec1 was checked)
        for (uint64_t r = p0; r < p1 && rec_off[r + 1] <= s1 && rec_off[r] >= s0; ++r) {
          const uint8_t* const rp = stage + dst0 + (rec_off[r] - b0);
          const uint8_t* const re = stage + dst0 + (rec_off[r + 1] - b0);
          __builtin_prefetch(rp, 0, 3);
          __builtin_prefetch(rp + 64, 0, 3);
          if (re - rp > 192) { __builtin_prefetch(re - 64, 0, 3); __builtin_prefetch(re - 128, 0, 3); }
        }
      }
      x->views.clear();
      for (uint64_t r = r0; r < r1; ++r) {
        if (rec_off[r + 1] < rec_off[r] || rec_off[r + 1] > s1) { x->last_error = "record offsets must ascend"; sts[t] = FGB_ERR_LAYOUT; return; }
        const size_t len = static_cast<size_t>(rec_off[r + 1] - rec_off[r]);
        if (len < 32) { x->last_error = "BAM record shorter than its fixed header"; sts[t] = FGB_ERR_INVALID_ARG; return; }
        x->views.emplace_back(stage + dst0 + (rec_off[r] - b0), len);
        if (x->views.back().aux_off() > len) { x->last_error = "truncated BAM record"; sts[t] = FGB_ERR_INVALID_ARG; return; }
      }
      x->group_runs.clear();
      if (c->opt.consensus_call_overlapping_bases) {   // simplex.rs:395-398
        x->rel_off.resize(n + 1);
        for (uint32_t i = 0; i <= n; ++i) x->rel_off[i] = rec_off[r0 + i] - rec_off[r0];
        uint8_t* const gbase = stage + dst0 + (rec_off[r0] - b0);
        // The device co-calls the overlaps on the uploaded records (the host only plans the runs) unless there is no
        // device, the quality trim needs whole rewritten reads or a mate has no qualities (0xFF): then in place, here.
        bool on_device = c->h && !c->prep_opt.trim && !c->opt.track_rejects;   // (rejected reads are kept as the pre-pass leaves them: on the host then)
        if (on_device) {
          x->overlap.plan_group(gbase, x->rel_off.data(), n, &x->group_runs);
          for (const overlap::Run& r : x->group_runs) {
            const View &v1 = x->views[r.rec1], &v2 = x->views[r.rec2];
            if (v1.l_seq() == 0 || v2.l_seq() == 0 || v1.b[v1.qual_off()] == 0xFF || v2.b[v2.qual_off()] == 0xFF ||
                v1.qual_off() + v1.l_seq() > v1.n || v2.qual_off() + v2.l_seq() > v2.n) { on_device = false; break; }
          }
        }
        if (!on_device) {
          if (zc) {   // the host pre-pass rewrites records in place: not on the caller's own blob
            x->last_error = "zero_copy_records: a mate pair without qualities needs the host overlapping-bases pre-pass; pass this batch without the flag";
            sts[t] = FGB_ERR_INVALID_ARG;
            return;
          }
          x->group_runs.clear();
          x->overlap.apply_group(gbase, x->rel_off.data(), n);
        } else {
          for (size_t k = 0; k < x->group_runs.size(); ++k) {
            const overlap::Run& r = x->group_runs[k];
            const View &v1 = x->views[r.rec1], &v2 = x->views[r.rec2];
            fgb_overlap_run g;
            g.seq1_off = static_cast<uint64_t>(v1.b - stage) + v1.seq_off();
            g.seq2_off = static_cast<uint64_t>(v2.b - stage) + v2.seq_off();
            g.l_seq1 = v1.l_seq(); g.l_seq2 = v2.l_seq();
            g.o1 = r.o1; g.o2 = r.o2; g.len = r.len;
            g.flags = (k > 0 && x->group_runs[k - 1].rec1 == r.rec1 && x->group_runs[k - 1].rec2 == r.rec2) ? FGB_RUN_CONTINUES : 0u;
            x->dplan.oruns.push_back(g);
          }
        }
      }
      const fgb_status st = direct_group_simplex(x, stage, x->views);
      if (st != FGB_OK) { sts[t] = st; return; }
    }
  };
  if (T > 1) run_parallel(c, T, run); else run(0);
  fgb_status first = FGB_OK;
  for (uint32_t t = 0; t < T && first == FGB_OK; ++t)
    if (sts[t] != FGB_OK) { first = sts[t]; if (ctx[t] != c) c->last_error = ctx[t]->last_error; }
  if (first != FGB_OK) {                      // roll everything of this call back
    for (uint32_t t = 0; t < T; ++t) {
      DirectPlan& P = ctx[t]->dplan;
      P.raws.resize(mark[t].raws); P.lens.resize(mark[t].raws); P.units.resize(mark[t].units); P.rx.resize(mark[t].rx);
      P.oruns.resize(mark[t].oruns);
      P.row_bytes = mark[t].row_bytes; P.out_elems = mark[t].out_elems; P.rec_bytes = mark[t].rec_bytes; P.str_bytes = mark[t].str_bytes;
      ctx[t]->rejects.resize(mark[t].rejects); ctx[t]->reject_count = mark[t].reject_count;
      if (ctx[t] != c) { std::memset(ctx[t]->stats, 0, sizeof(ctx[t]->stats)); ctx[t]->overlap.stats = overlap::Stats(); }
    }
    std::memcpy(c->stats, stats0, sizeof(stats0));
    c->overlap.stats = ostats0;
    if (c->segs.empty() && c->stage_len == 0) c->zc_base = nullptr;
    return first;
  }
  for (uint32_t t = 0; t < T; ++t) {
    fgb_caller* x = ctx[t];
    const DirectPlan& P = x->dplan;
    if (P.units.size() > mark[t].units || P.oruns.size() > mark[t].oruns) {
      DSeg sg{x, static_cast<uint32_t>(mark[t].units), static_cast<uint32_t>(P.units.size()), mark[t].raws, P.raws.size(),
              P.row_bytes - mark[t].row_bytes, P.out_elems - mark[t].out_elems, mark[t].oruns, P.oruns.size(),
              P.rec_bytes - mark[t].rec_bytes, P.str_bytes - mark[t].str_bytes};
      if (!c->segs.empty() && c->segs.back().ctx == x && c->segs.back().u1 == sg.u0 && c->segs.back().o1 == sg.o0) {   // serial add_group calls
        DSeg& l = c->segs.back();
        l.u1 = sg.u1; l.r1 = sg.r1; l.row_bytes += sg.row_bytes; l.out_elems += sg.out_elems; l.o1 = sg.o1;
        l.rec_bytes += sg.rec_bytes; l.str_bytes += sg.str_bytes;
      } else {
        c->segs.push_back(sg);
      }
    }
    if (x != c) {
      if (!x->rejects.empty()) {               // the workers' ranges are contiguous and in input order
        c->rejects.insert(c->rejects.end(), x->rejects.begin(), x->rejects.end());
        c->reject_count += x->reject_count;
        x->rejects.clear(); x->reject_count = 0;
      }
      for (int i = 0; i < FGB_NSTATS; ++i) { c->stats[i] += x->stats[i]; x->stats[i] = 0; }
      c->overlap.stats.overlapping_bases += x->overlap.stats.overlapping_bases;
      c->overlap.stats.bases_agreeing += x->overlap.stats.bases_agreeing;
      c->overlap.stats.bases_disagreeing += x->overlap.stats.bases_disagreeing;
      c->overlap.stats.bases_corrected += x->overlap.stats.bases_corrected;
      x->overlap.stats = overlap::Stats();
    }
  }
  c->stage_len = std::max<size_t>(c->stage_len, dst0 + (b1 - b0));
  return FGB_OK;
}

}  // namespace

extern "C" {

static fgb_status caller_add_groups_impl(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off,
                                 const uint64_t* group_rec, uint64_t n_groups) {
  if (!c || (n_groups && (!records || !rec_off || !group_rec))) return FGB_ERR_INVALID_ARG;
  if (n_groups == 0) return FGB_OK;
  if (c->opt.mode == FGB_MODE_SIMPLEX) return direct_add(c, records, rec_off, group_rec, n_groups);
  const uint64_t n_rec = group_rec[n_groups] - group_rec[0];
  uint32_t T = static_cast<uint32_t>(std::min<uint64_t>(std::max<uint32_t>(c->opt.n_threads, 1u), (n_groups + 63) / 64));
  auto run = [&](fgb_caller* dst, uint64_t g0, uint64_t g1, uint64_t* bad_group) -> fgb_status {
    for (uint64_t g = g0; g < g1; ++g) {
      const uint64_t r0 = group_rec[g], r1 = group_rec[g + 1];
      if (r1 < r0 || r1 - r0 > 0xFFFFFFFFull) { dst->last_error = "bad group_rec table"; *bad_group = g; return FGB_ERR_INVALID_ARG; }
      fgb_status st = caller_add_group_impl(dst, records, rec_off + r0, static_cast<uint32_t>(r1 - r0));
      if (st != FGB_OK) { *bad_group = g; return st; }
    }
    return FGB_OK;
  };
  if (T <= 1) {
    // one thread: the call still goes to a worker context first, so that a failing call leaves nothing of itself
    // queued -- the same outcome as with several threads (and as the direct path's roll-back)
    ensure_workers(c, 1);
    fgb_caller* w = c->workers[0].get();
    uint64_t bg = 0;
    const fgb_status st = run(w, 0, n_groups, &bg);
    if (st != FGB_OK) {
      c->last_error = w->last_error;
      fgb_caller scratch;
      merge_worker(&scratch, w);
      return st;
    }
    merge_worker(c, w);
    return FGB_OK;
  }
  ensure_workers(c, T);
  // contiguous ranges balanced by record count
  std::vector<uint64_t> cut(T + 1, n_groups);
  cut[0] = 0;
  for (uint32_t t = 1; t < T; ++t) {
    const uint64_t target = group_rec[0] + n_rec * t / T;
    cut[t] = static_cast<uint64_t>(std::lower_bound(group_rec, group_rec + n_groups, target) - group_rec);
    if (cut[t] < cut[t - 1]) cut[t] = cut[t - 1];
  }
  std::vector<fgb_status> sts(T, FGB_OK);
  std::vector<uint64_t> bad(T, 0);
  run_parallel(c, T, [&](uint32_t t) { sts[t] = run(c->workers[t].get(), cut[t], cut[t + 1], &bad[t]); });
  for (uint32_t t = 0; t < T; ++t) {
    if (sts[t] != FGB_OK) {           // report the first failing group in input order; drop the partial work
      c->last_error = c->workers[t]->last_error;
      for (auto& w : c->workers) { fgb_caller scratch; merge_worker(&scratch, w.get()); }
      return sts[t];
    }
  }
  size_t worker_bytes = 0;
  for (uint32_t t = 0; t < T; ++t) worker_bytes += c->workers[t]->pack.bases.size();
  if (worker_bytes >= kParallelMergeBytes) merge_workers_parallel(c, T);
  else for (uint32_t t = 0; t < T; ++t) merge_worker(c, c->workers[t].get());
  return FGB_OK;
}

static fgb_status caller_flush_impl(fgb_caller* c, const uint8_t** out_data, uint64_t* out_len,
                            uint64_t* out_count) {
  if (!c || !out_data || !out_len || !out_count) return FGB_ERR_INVALID_ARG;
  c->out.clear();
  c->out_count = 0;
  c->out_is_joined = false;
  if (!c->h) {
    c->last_error = "planning-only caller (FGB_DEVICE_NONE): flushing needs a GPU, there is no CPU fallback";
    return FGB_ERR_NO_DEVICE;
  }
  fgb_status st = c->opt.mode == FGB_MODE_DUPLEX ? flush_duplex(c)
                  : c->opt.mode == FGB_MODE_CODEC ? flush_codec(c)
                  : flush_simplex_direct(c);
  c->dplan.clear();
  for (auto& w : c->workers) w->dplan.clear();
  c->segs.clear();
  c->stage_len = 0;
  c->zc_base = nullptr;
  c->pack.clear(); c->molecules.clear(); c->jobs.clear();
  c->codec_molecules.clear(); c->codec_jobs.clear();
  c->n_duplex_out = 0; c->n_codec_out = 0;
  if (st != FGB_OK) return st;
  *out_data = c->out_is_joined ? c->joined : c->out.data();
  *out_len = c->out_is_joined ? c->joined_len : c->out.size();
  *out_count = c->out_count;
  return FGB_OK;
}

fgb_status fgb_overlap_apply_group(uint8_t* records, const uint64_t* rec_off, uint32_t n_records,
                                   uint8_t agreement, uint8_t disagreement, uint64_t stats[4]) {
  if (agreement > 2 || disagreement > 2 || (n_records && (!records || !rec_off))) return FGB_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n_records; ++i) {
    if (rec_off[i + 1] < rec_off[i] + 32) return FGB_ERR_INVALID_ARG;
    View v(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
    if (v.aux_off() > v.n) return FGB_ERR_INVALID_ARG;
  }
  overlap::Caller oc(static_cast<overlap::Agreement>(agreement), static_cast<overlap::Disagreement>(disagreement));
  oc.apply_group(records, rec_off, n_records);
  if (stats) {
    stats[0] += oc.stats.overlapping_bases; stats[1] += oc.stats.bases_agreeing;
    stats[2] += oc.stats.bases_disagreeing; stats[3] += oc.stats.bases_corrected;
  }
  return FGB_OK;
}

fgb_status fgb_host_group_by_mi(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                const char tag[2], int strip_strand_suffix, const char* cell_tag,
                                uint8_t* keep, uint64_t* group_begin, uint64_t* n_groups) {
  if (!tag || !keep || !group_begin || !n_groups || (n_records && (!records || !rec_off))) return FGB_ERR_INVALID_ARG;
  std::string cur, key;
  bool have = false;
  uint64_t kept = 0, groups = 0;
  for (uint64_t i = 0; i < n_records; ++i) {
    if (rec_off[i + 1] < rec_off[i] || rec_off[i + 1] - rec_off[i] < 32) return FGB_ERR_LAYOUT;
    const View v(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
    if (!v.cigar_in_bounds() || v.aux_off() > v.n) return FGB_ERR_LAYOUT;
    const uint8_t* val; size_t len;
    if (!bam::find_string_tag(v, tag, &val, &len)) { keep[i] = 0; continue; }
    keep[i] = 1;
    key.assign(reinterpret_cast<const char*>(val), len);
    if (strip_strand_suffix && key.size() >= 2 && key[key.size() - 2] == '/' && (key.back() == 'A' || key.back() == 'B'))
      key.resize(key.size() - 2);
    if (cell_tag) {
      key.push_back('\t');
      if (bam::find_string_tag(v, cell_tag, &val, &len)) key.append(reinterpret_cast<const char*>(val), len);
    }
    if (!have || key != cur) { group_begin[groups++] = kept; cur = key; have = true; }
    ++kept;
  }
  group_begin[groups] = kept;
  *n_groups = groups;
  return FGB_OK;
}

fgb_status fgb_host_source_reads(const uint8_t* records, const uint64_t* rec_off, uint32_t n_records,
                                 uint8_t min_input_base_quality, int trim, uint8_t* out_bases,
                                 uint8_t* out_quals, uint64_t* row_off, uint32_t* orig_idx,
                                 uint32_t* n_rows, uint32_t* n_minority) {
  if (!n_rows || !row_off || (n_records && (!records || !rec_off || !out_bases || !out_quals || !orig_idx)))
    return FGB_ERR_INVALID_ARG;
  prep::PrepOptions po;
  po.min_input_base_quality = min_input_base_quality;
  po.trim = trim != 0;
  std::vector<prep::SourceRead> srs;
  std::vector<uint32_t> ops;
  for (uint32_t i = 0; i < n_records; ++i) {
    if (rec_off[i + 1] < rec_off[i] || rec_off[i + 1] - rec_off[i] < 32) return FGB_ERR_LAYOUT;
    const View v(records + rec_off[i], rec_off[i + 1] - rec_off[i]);
    if (!v.cigar_in_bounds() || v.aux_off() > v.n) return FGB_ERR_LAYOUT;
    bam::cigar_ops(v, &ops);
    const size_t clip = bam::num_bases_extending_past_mate(v, ops);
    prep::SourceRead sr;
    if (prep::make_source_read(po, v, i, clip, &ops, &sr)) srs.push_back(std::move(sr));
  }
  const size_t minority = prep::filter_by_alignment(&srs);
  uint64_t off = 0;
  for (size_t r = 0; r < srs.size(); ++r) {
    row_off[r] = off;
    std::memcpy(out_bases + off, srs[r].bases.data(), srs[r].bases.size());
    std::memcpy(out_quals + off, srs[r].quals.data(), srs[r].quals.size());
    orig_idx[r] = srs[r].original_idx;
    off += srs[r].bases.size();
  }
  row_off[srs.size()] = off;
  *n_rows = static_cast<uint32_t>(srs.size());
  if (n_minority) *n_minority = static_cast<uint32_t>(minority);
  return FGB_OK;
}

fgb_status fgb_host_simplex_record(const char* read_name_prefix, const char* read_group_id, const char* umi,
                                   uint8_t read_type, int produce_per_base_tags, const uint8_t* bases,
                                   const uint8_t* quals, const uint16_t* depths, const uint16_t* errors,
                                   uint32_t len, const char cell_tag[2], const char* cell,
                                   const char* const* rx, uint32_t n_rx, uint8_t* out, size_t cap,
                                   size_t* out_len) {
  if (!read_name_prefix || !read_group_id || !umi || read_type > 2 || !out || !out_len ||
      (len && (!bases || !quals || !depths || !errors)) || (n_rx && !rx))
    return FGB_ERR_INVALID_ARG;
  fgb_caller c;
  c.prefix = read_name_prefix;
  c.rg = read_group_id;
  c.opt.produce_per_base_tags = produce_per_base_tags ? 1 : 0;
  // the UMI, cell and RX strings in one buffer, referenced the way the flush references the staged records
  std::string strs = umi;
  DUnit u;
  u.cons_len = len;
  u.read_type = read_type;
  u.umi = StrRef{0, static_cast<uint32_t>(strs.size())};
  if (cell_tag && cell) {
    c.opt.cell_tag[0] = cell_tag[0]; c.opt.cell_tag[1] = cell_tag[1];
    u.has_cell = 1;
    u.cell = StrRef{strs.size(), static_cast<uint32_t>(std::strlen(cell))};
    strs += cell;
  }
  std::vector<StrRef> rx_refs;
  for (uint32_t i = 0; i < n_rx; ++i) {
    if (!rx[i]) return FGB_ERR_INVALID_ARG;
    rx_refs.push_back(StrRef{strs.size(), static_cast<uint32_t>(std::strlen(rx[i]))});
    strs += rx[i];
  }
  u.rx_n = n_rx;
  uint32_t max_d = 0, min_d = len ? 0xFFFFFFFFu : 0u;
  for (uint32_t k = 0; k < len; ++k) { max_d = std::max<uint32_t>(max_d, depths[k]); min_d = std::min<uint32_t>(min_d, depths[k]); }
  const uint32_t size = simplex_record_size(&c, len, u.umi.len, u.has_cell, u.cell.len, n_rx > 0, n_rx ? rx_refs[0].len : 0u,
                                            int_tag_width(max_d), int_tag_width(min_d));
  if (size > cap) return FGB_ERR_INVALID_ARG;
  std::string scratch, err;
  const size_t n = write_simplex_record_at<uint16_t>(&c, out, u, rx_refs.data(), reinterpret_cast<const uint8_t*>(strs.data()),
                                                     bases, quals, depths, errors, &scratch, &err);
  if (n == 0) return FGB_ERR_INVALID_ARG;      // read name too long, or RX values the reference rejects
  if (n != size) return FGB_ERR_INVALID_ARG;   // simplex_record_size disagrees with the writer
  *out_len = n;
  return FGB_OK;
}

fgb_status fgb_host_duplex_record(const char* read_name_prefix, const char* read_group_id, const char* base_mi,
                                  int first_of_pair, int produce_per_base_tags, const uint8_t* bases,
                                  const uint8_t* quals, const uint16_t* errors, uint32_t len,
                                  const fgb_strand_columns* ab, const fgb_strand_columns* ba,
                                  const char cell_tag[2], const char* cell, const char* const* rx,
                                  const uint8_t* rx_first, uint32_t n_rx, uint8_t* out, size_t cap, size_t* out_len) {
  if (!read_name_prefix || !read_group_id || !base_mi || !ab || !out || !out_len ||
      (len && (!bases || !quals || !errors)) || (n_rx && (!rx || !rx_first)))
    return FGB_ERR_INVALID_ARG;
  fgb_caller c;
  c.prefix = read_name_prefix;
  c.rg = read_group_id;
  c.opt.produce_per_base_tags = produce_per_base_tags ? 1 : 0;
  Molecule m;
  m.base_mi = base_mi;
  if (cell_tag && cell) { c.opt.cell_tag[0] = cell_tag[0]; c.opt.cell_tag[1] = cell_tag[1]; m.has_cell = true; m.cell = cell; }
  auto strand = [](const fgb_strand_columns* s) {
    Strand r;
    if (s && s->present) { r.bases = s->bases; r.quals = s->quals; r.depths = s->depths; r.errors = s->errors; r.len = s->len; r.present = true; }
    return r;
  };
  DuplexRead d;
  d.bases = bases; d.quals = quals; d.errors = errors; d.len = len;
  d.ab = strand(ab); d.ba = strand(ba);
  if (!d.ab.present) return FGB_ERR_INVALID_ARG;
  std::vector<RxSource> src;
  for (uint32_t i = 0; i < n_rx; ++i) { if (!rx[i]) return FGB_ERR_INVALID_ARG; src.push_back(RxSource{rx[i], rx_first[i] != 0}); }
  static const std::vector<RxSource> kNone;
  bam::Writer w(&c.out);
  fgb_status st = write_duplex_record(&c, &w, d, first_of_pair != 0, m, src, kNone);
  if (st != FGB_OK) return st;
  if (c.out.size() > cap) return FGB_ERR_INVALID_ARG;
  std::memcpy(out, c.out.data(), c.out.size());
  *out_len = c.out.size();
  return FGB_OK;
}

fgb_status fgb_host_consensus_umis(const char* const* umis, uint32_t n, char* out, size_t cap) {
  if ((n && !umis) || !out || !cap) return FGB_ERR_INVALID_ARG;
  static const prep::UmiBuilder builder;
  std::vector<std::string> v;
  for (uint32_t i = 0; i < n; ++i) { if (!umis[i]) return FGB_ERR_INVALID_ARG; v.emplace_back(umis[i]); }
  std::string res;
  if (!prep::consensus_umis(builder, v, &res) || res.size() + 1 > cap) return FGB_ERR_INVALID_ARG;
  std::memcpy(out, res.c_str(), res.size() + 1);
  return FGB_OK;
}

int fgb_host_is_fr_pair(const uint8_t* record, size_t len) {
  if (!record || len < 32) return 0;
  const bam::View v(record, len);
  if (!v.cigar_in_bounds()) return 0;
  std::vector<uint32_t> ops;
  bam::cigar_ops(v, &ops);
  return bam::is_fr_pair(v, ops) ? 1 : 0;
}

uint32_t fgb_host_num_bases_extending_past_mate(const uint8_t* record, size_t len) {
  if (!record || len < 32) return 0;
  const bam::View v(record, len);
  if (!v.cigar_in_bounds() || v.aux_off() > len) return 0;
  std::vector<uint32_t> ops;
  bam::cigar_ops(v, &ops);
  return static_cast<uint32_t>(bam::num_bases_extending_past_mate(v, ops));
}

fgb_status fgb_host_clip_cigar_ops(const uint32_t* ops, uint32_t n_ops, uint32_t clip_amount, int from_start,
                                   uint32_t* out_ops, uint32_t* out_n, uint32_t* ref_consumed) {
  if ((n_ops && !ops) || !out_ops || !out_n) return FGB_ERR_INVALID_ARG;
  const std::vector<uint32_t> in(ops, ops + n_ops);
  size_t rc = 0;
  const std::vector<uint32_t> res = bam::clip_cigar_ops(in, clip_amount, from_start != 0, &rc);
  if (res.size() > static_cast<size_t>(n_ops) + 2) return FGB_ERR_LAYOUT;
  std::copy(res.begin(), res.end(), out_ops);
  *out_n = static_cast<uint32_t>(res.size());
  if (ref_consumed) *ref_consumed = static_cast<uint32_t>(rc);
  return FGB_OK;
}

int fgb_host_read_pos_at_ref_pos(const uint32_t* ops, uint32_t n_ops, uint64_t alignment_start,
                                 uint64_t ref_pos, int return_last_base_if_deleted, uint64_t* read_pos) {
  if ((n_ops && !ops) || !read_pos) return 0;
  const std::vector<uint32_t> in(ops, ops + n_ops);
  size_t out = 0;
  if (!bam::read_pos_at_ref_pos(in, alignment_start, ref_pos, return_last_base_if_deleted != 0, &out)) return 0;
  *read_pos = out;
  return 1;
}

fgb_status fgb_host_simplify_cigar(const uint32_t* ops, uint32_t n_ops, uint8_t* out_kinds, uint32_t* out_lens,
                                   uint32_t* out_n) {
  if ((n_ops && (!ops || !out_kinds || !out_lens)) || !out_n) return FGB_ERR_INVALID_ARG;
  const std::vector<uint32_t> in(ops, ops + n_ops);
  bam::SimpleCigar sc;
  bam::simplify_cigar(in, &sc);
  for (size_t i = 0; i < sc.size(); ++i) { out_kinds[i] = sc[i].first; out_lens[i] = sc[i].second; }
  *out_n = static_cast<uint32_t>(sc.size());
  return FGB_OK;
}

fgb_status fgb_filter_record(uint8_t* record, size_t len, const fgb_duplex_filter_params* p,
                             uint32_t* masked, uint8_t* status) {
  if (!record || !p || !status || len < 32) return FGB_ERR_INVALID_ARG;
  const bam::View v(record, len);
  if (!v.cigar_in_bounds() || v.aux_off() > len) return FGB_ERR_LAYOUT;
  uint32_t m = 0;
  *status = static_cast<uint8_t>(rfilter::filter_record(record, len, *p, &m));
  if (masked) *masked = m;
  return FGB_OK;
}

uint32_t fgb_struct_size(uint32_t id) {
  switch (id) {
    case 0: return sizeof(fgb_caller_options);
    case 1: return sizeof(fgb_filter_params);
    case 2: return sizeof(fgb_submit_options);
    case 3: return sizeof(fgb_raw_columns);
    case 4: return sizeof(fgb_raw_read);
    case 5: return sizeof(fgb_batch);
    case 6: return sizeof(fgb_codec_params);
    case 7: return sizeof(fgb_params);
    case 8: return sizeof(fgb_duplex_filter_params);
    case 9: return sizeof(fgb_record_columns);
    case 10: return sizeof(fgb_umi_options);
    case 11: return sizeof(fgb_group_options);
    case 12: return sizeof(fgb_sort_options);
    case 13: return sizeof(fgb_dedup_options);
    case 14: return sizeof(fgb_record_filter_options);
    case 15: return sizeof(fgb_metrics_options);
    case 16: return sizeof(fgb_metrics_template);
    case 17: return sizeof(fgb_zipper_options);
    default: return 0;
  }
}

fgb_status fgb_caller_stats(const fgb_caller* c, uint64_t stats[FGB_NSTATS]) {
  if (!c || !stats) return FGB_ERR_INVALID_ARG;
  std::memcpy(stats, c->stats, sizeof(c->stats));
  stats[FGB_STAT_OVERLAP_BASES] = c->overlap.stats.overlapping_bases;
  stats[FGB_STAT_OVERLAP_AGREEING] = c->overlap.stats.bases_agreeing;
  stats[FGB_STAT_OVERLAP_DISAGREEING] = c->overlap.stats.bases_disagreeing;
  stats[FGB_STAT_OVERLAP_CORRECTED] = c->overlap.stats.bases_corrected;
  return FGB_OK;
}

// No exception crosses the C ABI: an allocation failure anywhere below (on any of the caller's threads, see
// WorkerPool::run) becomes FGB_ERR_NOMEM; a failed add leaves nothing of the call queued on the direct path.
#define FGB_GUARD(c, call)                                                      \
  try { return (call); }                                                        \
  catch (const std::bad_alloc&) { if (c) (c)->last_error = "out of memory"; return FGB_ERR_NOMEM; } \
  catch (...) { if (c) (c)->last_error = "internal error"; return FGB_ERR_INVALID_ARG; }

fgb_status fgb_caller_create(int device, const fgb_caller_options* opt, fgb_caller** out) {
  fgb_caller* none = nullptr;
  FGB_GUARD(none, caller_create_impl(device, opt, out))
}
fgb_status fgb_caller_add_group(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off, uint32_t n_records) {
  FGB_GUARD(c, caller_add_group_impl(c, records, rec_off, n_records))
}
fgb_status fgb_caller_add_groups(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off,
                                 const uint64_t* group_rec, uint64_t n_groups) {
  FGB_GUARD(c, caller_add_groups_impl(c, records, rec_off, group_rec, n_groups))
}
fgb_status fgb_caller_flush(fgb_caller* c, const uint8_t** out_data, uint64_t* out_len, uint64_t* out_count) {
  FGB_GUARD(c, caller_flush_impl(c, out_data, out_len, out_count))
}
fgb_status fgb_caller_pending(const fgb_caller* c, fgb_batch* batch, const fgb_duplex_job** duplex_jobs,
                              uint64_t* n_duplex_jobs, const fgb_codec_job** codec_jobs, uint64_t* n_codec_jobs) {
  FGB_GUARD(c, caller_pending_impl(c, batch, duplex_jobs, n_duplex_jobs, codec_jobs, n_codec_jobs))
}

}  // extern "C"
