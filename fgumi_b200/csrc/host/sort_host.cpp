// `fgumi sort` (coordinate, template-coordinate and queryname) from raw BAM records: the header's library table, the
// host key and verify entry points, and the driver of the device sort (fgb_sort_records): runs that fit a device
// budget, each uploaded through page-locked staging, keyed, sorted by stable radix passes over the key words that vary
// and gathered into a [u32 block_size][record] stream on the device; several runs are merged on the host.  The key
// functions are ../sort_keys.h; the kernels and CUB calls sit behind sort_device.h in capi.cu.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <string_view>
#include <vector>

#include "../../../include/fgumi_b200.h"
#include "../sort_keys.h"
#include "bam.h"
#include "record_link.h"
#include "sort_device.h"
#include "umi_host.h"

namespace {

namespace sk = fgb::sortk;
namespace dev = fgb::sortdev;
namespace link = fgb::link;
using link::ms_since;

static_assert(FGB_SORT_COORDINATE == sk::kCoordinate && FGB_SORT_TEMPLATE_COORDINATE == sk::kTemplateCoordinate &&
                  FGB_SORT_QUERYNAME == sk::kQueryname && FGB_SORT_QUERYNAME_NATURAL == sk::kQuerynameNatural,
              "sort orders");
constexpr uint64_t kNone = UINT64_MAX;

// LibraryLookup::from_header (raw.rs:237-283): the distinct LB values sorted bytewise and numbered from 1; each RG ID
// maps to its LB's ordinal, an RG without LB to that of "" (0 unless some LB is empty).  IDs are kept sorted bytewise
// (std::string compares as unsigned bytes) so that the key functions look them up by binary search.
struct Lookup {
  std::vector<uint8_t> bytes;
  std::vector<uint32_t> off{0};
  std::vector<uint32_t> lib;
};

Lookup library_lookup(std::string_view text) {
  std::map<std::string, std::string> lb_of_rg;   // an RG without LB maps to ""
  std::vector<std::string> libs;
  fgb::bam::for_each_read_group(text, [&](std::string_view id, std::string_view lb, bool has_lb) {
    lb_of_rg[std::string(id)] = std::string(lb);
    if (has_lb) libs.emplace_back(lb);
  });
  std::sort(libs.begin(), libs.end());
  libs.erase(std::unique(libs.begin(), libs.end()), libs.end());
  Lookup l;
  for (const auto& [id, lb] : lb_of_rg) {
    l.bytes.insert(l.bytes.end(), id.begin(), id.end());
    l.off.push_back(static_cast<uint32_t>(l.bytes.size()));
    const auto it = std::lower_bound(libs.begin(), libs.end(), lb);
    l.lib.push_back(it != libs.end() && *it == lb ? static_cast<uint32_t>(it - libs.begin()) + 1 : 0);
  }
  return l;
}

bool options_ok(const fgb_sort_options* o) {
  if (!o || o->order > FGB_SORT_QUERYNAME_NATURAL) return false;
  return (o->cell_tag[0] == 0) == (o->cell_tag[1] == 0);
}

sk::Ctx make_ctx(const fgb_sort_options& o, const uint8_t* bytes, const uint32_t* off, const uint32_t* lib, uint32_t n_rg) {
  sk::Ctx c{};
  c.rg_bytes = bytes; c.rg_off = off; c.rg_lib = lib; c.n_rg = n_rg;
  c.order = o.order;
  c.has_cell = o.order == FGB_SORT_TEMPLATE_COORDINATE && o.cell_tag[0] != 0;
  c.cell[0] = static_cast<uint8_t>(o.cell_tag[0]);
  c.cell[1] = static_cast<uint8_t>(o.cell_tag[1]);
  return c;
}

bool queryname(const fgb_sort_options& o) {
  return o.order == FGB_SORT_QUERYNAME || o.order == FGB_SORT_QUERYNAME_NATURAL;
}

// Key words per record: 1 (coordinate), 5 (template-coordinate), or for queryname the name words of the longest
// l_read_name `lrn` among the run's records plus the last word.
int key_words(const fgb_sort_options& o, uint32_t lrn) {
  if (queryname(o))
    return static_cast<int>(sk::name_words(static_cast<uint8_t>(lrn), o.order == FGB_SORT_QUERYNAME_NATURAL)) + 1;
  return o.order == FGB_SORT_COORDINATE ? 1 : sk::kWords;
}

// Each record holds its 32-byte fixed part and rec_off ascends; else *bad = the first offending record.
bool records_ok(const uint64_t* rec_off, uint64_t n, uint64_t* bad) {
  for (uint64_t i = 0; i < n; ++i)
    if (rec_off[i + 1] < rec_off[i] || rec_off[i + 1] - rec_off[i] < 32) { if (bad) *bad = i; return false; }
  return true;
}

bool args_ok(const fgb_sort_options* opt, const char* header_text, size_t header_len, const uint8_t* records,
             const uint64_t* rec_off, uint64_t n) {
  return options_ok(opt) && (!header_len || header_text) && rec_off && (!n || records);
}

// Keys of every record, row-major (5 words per record), on n_threads host threads.
void host_keys(const fgb_sort_options& o, std::string_view header, const uint8_t* records, const uint64_t* rec_off,
               uint64_t n, uint64_t* keys) {
  const Lookup l = library_lookup(header);
  const sk::Ctx c = make_ctx(o, l.bytes.data(), l.off.data(), l.lib.data(), static_cast<uint32_t>(l.lib.size()));
  const uint64_t t = std::max<uint32_t>(o.n_threads, 1);
  fgb_umi::parallel_for(t, o.n_threads, [&](uint64_t w) {
    for (uint64_t i = n * w / t, e = n * (w + 1) / t; i < e; ++i)
      sk::record_key(records + rec_off[i], rec_off[i + 1] - rec_off[i], c, keys + sk::kWords * i);
  });
}

fgb_status sort_impl(const link::HandleInfo& hi, const fgb_sort_options& o, std::string_view header,
                     const uint8_t* records, const uint64_t* rec_off, uint64_t n, uint8_t* out) {
  auto fail = [&](cudaError_t e, const char* what) { return link::fail(hi.last_error, "fgb_sort_records", e, what); };
  link::Resources r(hi.stream, o.n_threads);
  const cudaStream_t s = hi.stream;
  double* tm = hi.timing;
  const bool qn = queryname(o), natural = o.order == FGB_SORT_QUERYNAME_NATURAL;
  cudaError_t e = cudaSetDevice(hi.device);
  if (e != cudaSuccess) return fail(e, "cudaSetDevice");
  // runs: as many records as fit the budget (input and output bytes, keys, permutations and scan / sort scratch: 68 +
  // 8 W bytes per record, W the run's key words)
  uint64_t budget;
  if ((e = link::device_budget(o.device_bytes, &budget)) != cudaSuccess) return fail(e, "cudaMemGetInfo");
  auto lrn = [&](uint64_t i) -> uint32_t { return qn ? records[rec_off[i] + 8] : 0; };   // l_read_name
  std::vector<uint64_t> run_begin{0};
  std::vector<int> run_words;
  uint64_t max_n = 0, max_bytes = 0, max_cells = 0;
  int max_words = 0;
  for (uint64_t b = 0; b < n;) {
    uint64_t i = b + 1;   // at least one record per run
    uint32_t l = lrn(b);
    while (i < n && i - b < INT32_MAX) {
      const uint32_t li = std::max(l, lrn(i));
      if (2 * (rec_off[i + 1] - rec_off[b]) + (i + 1 - b) * (68 + 8ull * key_words(o, li) + 4) > budget) break;
      l = li;
      ++i;
    }
    const int words = key_words(o, l);
    max_n = std::max(max_n, i - b);
    max_bytes = std::max(max_bytes, rec_off[i] - rec_off[b]);
    max_cells = std::max(max_cells, static_cast<uint64_t>(words) * (i - b));
    max_words = std::max(max_words, words);
    run_begin.push_back(i);
    run_words.push_back(words);
    b = i;
  }
  const uint64_t n_runs = run_begin.size() - 1;
  const bool merge_keys = n_runs > 1 && !qn;   // the queryname merge compares the records themselves
  // buffers for the largest run
  const Lookup l = library_lookup(header);
  uint8_t *d_rec, *d_out, *d_rg, *d_temp;
  uint64_t *d_off, *d_keys, *d_rows = nullptr, *d_ktmp[2], *d_osize, *d_ooff;
  uint32_t *d_size, *d_perm[2], *d_rgoff, *d_rglib;
  unsigned long long* d_andor;
  const uint32_t mn = static_cast<uint32_t>(max_n);
  size_t t_sort = 0, t_scan = 0;
  if ((e = dev::radix_pass(nullptr, &t_sort, nullptr, nullptr, nullptr, nullptr, mn, 0, 64, s)) != cudaSuccess ||
      (e = dev::out_offsets(nullptr, &t_scan, nullptr, nullptr, mn, nullptr, nullptr, s)) != cudaSuccess)
    return fail(e, "CUB temp storage");
  if ((e = r.alloc(&d_rec, max_bytes + 16)) != cudaSuccess || (e = r.alloc(&d_out, max_bytes + 4 * max_n)) ||
      (e = r.alloc(&d_off, max_n + 1)) || (e = r.alloc(&d_keys, max_cells)) ||
      (e = r.alloc(&d_ktmp[0], max_n)) || (e = r.alloc(&d_ktmp[1], max_n)) ||
      (e = r.alloc(&d_osize, max_n + 1)) || (e = r.alloc(&d_ooff, max_n + 1)) || (e = r.alloc(&d_size, max_n)) ||
      (e = r.alloc(&d_perm[0], max_n)) || (e = r.alloc(&d_perm[1], max_n)) ||
      (e = r.alloc(&d_rg, l.bytes.size())) || (e = r.alloc(&d_rgoff, l.off.size())) ||
      (e = r.alloc(&d_rglib, l.lib.size())) || (e = r.alloc(&d_andor, 2 * max_words)) ||
      (e = r.alloc(&d_temp, std::max(t_sort, t_scan) + 16)) || (merge_keys && (e = r.alloc(&d_rows, max_cells))))
    return fail(e, "cudaMalloc");
  const char* what;
  if ((e = r.open(std::min<uint64_t>(link::kStageBytes, std::max(max_bytes + 4 * max_n, (max_n + 1) * 8)), &what)))
    return fail(e, what);
  if ((!l.bytes.empty() && (e = cudaMemcpy(d_rg, l.bytes.data(), l.bytes.size(), cudaMemcpyHostToDevice))) ||
      (e = cudaMemcpy(d_rgoff, l.off.data(), l.off.size() * 4, cudaMemcpyHostToDevice)) ||
      (!l.lib.empty() && (e = cudaMemcpy(d_rglib, l.lib.data(), l.lib.size() * 4, cudaMemcpyHostToDevice))))
    return fail(e, "cudaMemcpy");
  const sk::Ctx ctx = make_ctx(o, d_rg, d_rgoff, d_rglib, static_cast<uint32_t>(l.lib.size()));
  // several runs: each run's sorted stream and its keys in sorted order (row-major) come back for the merge
  std::vector<uint8_t> run_stream;
  std::vector<std::vector<uint64_t>> run_keys(merge_keys ? n_runs : 0);
  if (n_runs > 1) run_stream.resize(rec_off[n] - rec_off[0] + 4 * n);
  std::vector<unsigned long long> init(2 * max_words), and_or(2 * max_words);
  for (int w = 0; w < max_words; ++w) { init[2 * w] = ~0ull; init[2 * w + 1] = 0; }
  for (uint64_t x = 0; x < n_runs; ++x) {
    const uint64_t b = run_begin[x], nr64 = run_begin[x + 1] - b;
    const uint32_t nr = static_cast<uint32_t>(nr64);
    const int W = run_words[x];
    const uint64_t base = rec_off[b], bytes = rec_off[b + nr64] - base, out_at = base - rec_off[0] + 4 * b;
    auto t0 = std::chrono::steady_clock::now();
    if ((e = r.upload(d_rec, records + base, bytes)) || (e = r.upload(d_off, rec_off + b, (nr64 + 1) * 8)) ||
        (e = cudaStreamSynchronize(s)))
      return fail(e, "upload");
    tm[0] += ms_since(t0);
    if ((e = cudaMemcpyAsync(d_andor, init.data(), 16 * W, cudaMemcpyHostToDevice, s)) ||
        (e = cudaEventRecord(r.ev[0], s)) ||
        (e = qn ? dev::name_keys(d_rec, d_off, base, nr, natural, W - 1, d_keys, d_size, d_andor, s)
                : dev::keys(d_rec, d_off, base, nr, ctx, W, d_keys, d_size, d_andor, s)) ||
        (e = cudaEventRecord(r.ev[1], s)) ||
        (e = cudaMemcpyAsync(and_or.data(), d_andor, 16 * W, cudaMemcpyDeviceToHost, s)) ||
        (e = cudaStreamSynchronize(s)))
      return fail(e, "key kernel");
    // LSD over the words, last first, skipping constant ones and sorting only the bits that vary
    uint32_t* perm = d_perm[0];
    uint32_t* spare = d_perm[1];
    bool first = true;
    if ((e = cudaEventRecord(r.ev[2], s)) != cudaSuccess) return fail(e, "cudaEventRecord");
    for (int w = W - 1; w >= 0; --w) {
      const uint64_t diff = and_or[2 * w] ^ and_or[2 * w + 1];
      if (!diff) continue;
      const int begin = __builtin_ctzll(diff), end = 64 - __builtin_clzll(diff);
      const uint64_t* src = d_keys + static_cast<uint64_t>(w) * nr;
      if (first) e = dev::iota(perm, nr, s);
      else { e = dev::word_gather(src, perm, nr, d_ktmp[0], s); src = d_ktmp[0]; }
      size_t tb = std::max(t_sort, t_scan) + 16;
      if (e || (e = dev::radix_pass(d_temp, &tb, src, d_ktmp[1], perm, spare, nr, begin, end, s)))
        return fail(e, "radix pass");
      std::swap(perm, spare);
      first = false;
    }
    if (first && (e = dev::iota(perm, nr, s))) return fail(e, "iota");
    size_t tb = std::max(t_sort, t_scan) + 16;
    if ((e = cudaEventRecord(r.ev[3], s)) ||
        (e = dev::out_offsets(d_temp, &tb, d_size, perm, nr, d_osize, d_ooff, s)) ||
        (e = dev::gather(d_rec, d_off, base, perm, d_ooff, nr, d_out, hi.sm_count, s)) ||
        (merge_keys && (e = dev::key_rows(d_keys, perm, nr, W, d_rows, s))) ||
        (e = cudaEventRecord(r.ev[4], s)) || (e = cudaStreamSynchronize(s)))
      return fail(e, "gather");
    float k_ms = 0, s_ms = 0, g_ms = 0;
    cudaEventElapsedTime(&k_ms, r.ev[0], r.ev[1]);
    cudaEventElapsedTime(&s_ms, r.ev[2], r.ev[3]);
    cudaEventElapsedTime(&g_ms, r.ev[3], r.ev[4]);
    tm[1] += k_ms; tm[2] += s_ms; tm[3] += g_ms;
    t0 = std::chrono::steady_clock::now();
    const uint64_t out_bytes = bytes + 4 * nr64;
    if ((e = r.download((n_runs > 1 ? run_stream.data() : out) + out_at, d_out, out_bytes)))
      return fail(e, "download");
    if (merge_keys) {
      run_keys[x].resize(W * nr64);
      if ((e = cudaMemcpy(run_keys[x].data(), d_rows, W * nr64 * 8, cudaMemcpyDeviceToHost)))
        return fail(e, "download");
    }
    tm[4] += ms_since(t0);
  }
  if (n_runs <= 1) return FGB_OK;
  // k-way merge by the key words, ties by run index: a binary heap of run heads.  Queryname runs are merged with the
  // reference comparator on the head records themselves, not with the encoded keys, so that the tests comparing many
  // runs with one run also check the encoding against the comparator.
  const auto t0 = std::chrono::steady_clock::now();
  const int W = run_words[0];
  std::vector<uint64_t> pos(n_runs, 0), cur(n_runs);
  for (uint64_t x = 0; x < n_runs; ++x) cur[x] = rec_off[run_begin[x]] - rec_off[0] + 4 * run_begin[x];
  auto after = [&](uint64_t a, uint64_t b) {   // heap order: true when run a's head goes after run b's
    if (qn) {
      uint32_t la, lb;
      std::memcpy(&la, run_stream.data() + cur[a], 4);
      std::memcpy(&lb, run_stream.data() + cur[b], 4);
      const int c = sk::queryname_cmp(run_stream.data() + cur[a] + 4, la, run_stream.data() + cur[b] + 4, lb, natural);
      return c ? c > 0 : a > b;
    }
    const uint64_t* ka = run_keys[a].data() + W * pos[a];
    const uint64_t* kb = run_keys[b].data() + W * pos[b];
    for (int w = 0; w < W; ++w)
      if (ka[w] != kb[w]) return ka[w] > kb[w];
    return a > b;
  };
  std::vector<uint64_t> heap;
  for (uint64_t x = 0; x < n_runs; ++x) heap.push_back(x);
  std::make_heap(heap.begin(), heap.end(), after);
  uint8_t* o_at = out;
  while (!heap.empty()) {
    std::pop_heap(heap.begin(), heap.end(), after);
    const uint64_t x = heap.back();
    uint32_t bs;
    std::memcpy(&bs, run_stream.data() + cur[x], 4);
    std::memcpy(o_at, run_stream.data() + cur[x], 4ull + bs);
    o_at += 4ull + bs;
    cur[x] += 4ull + bs;
    if (++pos[x] < run_begin[x + 1] - run_begin[x]) std::push_heap(heap.begin(), heap.end(), after);
    else heap.pop_back();
  }
  tm[5] = ms_since(t0);
  return FGB_OK;
}

}  // namespace

extern "C" {

fgb_status fgb_host_sort_keys(const fgb_sort_options* opt, const char* header_text, size_t header_len,
                              const uint8_t* records, const uint64_t* rec_off, uint64_t n_records, uint64_t* keys,
                              uint64_t* bad_record) {
  if (!args_ok(opt, header_text, header_len, records, rec_off, n_records) || queryname(*opt) || (n_records && !keys))
    return FGB_ERR_INVALID_ARG;
  if (bad_record) *bad_record = kNone;
  if (!records_ok(rec_off, n_records, bad_record)) return FGB_ERR_LAYOUT;
  try {
    host_keys(*opt, std::string_view(header_text ? header_text : "", header_len), records, rec_off, n_records, keys);
  } catch (const std::exception&) {
    return FGB_ERR_NOMEM;
  }
  return FGB_OK;
}

fgb_status fgb_host_sort_verify(const fgb_sort_options* opt, const char* header_text, size_t header_len,
                                const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                uint64_t* violations, uint64_t* first_violation, uint64_t* bad_record) {
  if (!args_ok(opt, header_text, header_len, records, rec_off, n_records) || !violations || !first_violation)
    return FGB_ERR_INVALID_ARG;
  if (bad_record) *bad_record = kNone;
  if (!records_ok(rec_off, n_records, bad_record)) return FGB_ERR_LAYOUT;
  if (queryname(*opt)) {   // the full key: the name comparator, then the flag order
    const bool natural = opt->order == FGB_SORT_QUERYNAME_NATURAL;
    const uint64_t t = std::max<uint32_t>(opt->n_threads, 1);
    std::vector<uint64_t> v(t, 0), first(t, kNone);
    try {
      fgb_umi::parallel_for(t, opt->n_threads, [&](uint64_t w) {
        for (uint64_t i = std::max<uint64_t>(n_records * w / t, 1), e = n_records * (w + 1) / t; i < e; ++i)
          if (sk::queryname_cmp(records + rec_off[i], rec_off[i + 1] - rec_off[i], records + rec_off[i - 1],
                                rec_off[i] - rec_off[i - 1], natural) < 0) {
            ++v[w];
            if (first[w] == kNone) first[w] = i;
          }
      });
    } catch (const std::exception&) {
      return FGB_ERR_NOMEM;
    }
    *violations = 0;
    *first_violation = kNone;
    for (uint64_t w = 0; w < t; ++w) {
      *violations += v[w];
      *first_violation = std::min(*first_violation, first[w]);
    }
    return FGB_OK;
  }
  try {
    std::vector<uint64_t> k(sk::kWords * n_records);
    host_keys(*opt, std::string_view(header_text ? header_text : "", header_len), records, rec_off, n_records, k.data());
    const int core = opt->order == FGB_SORT_COORDINATE ? 1 : 4;   // core_cmp leaves out name_hash_upper
    uint64_t v = 0, first = kNone;
    for (uint64_t i = 1; i < n_records; ++i) {
      const uint64_t* a = k.data() + sk::kWords * i;
      const uint64_t* p = a - sk::kWords;
      if (std::lexicographical_compare(a, a + core, p, p + core)) {
        ++v;
        if (first == kNone) first = i;
      }
    }
    *violations = v;
    *first_violation = first;
  } catch (const std::exception&) {
    return FGB_ERR_NOMEM;
  }
  return FGB_OK;
}

fgb_status fgb_host_sort_name_key(const fgb_sort_options* opt, const uint8_t* record, uint64_t len, uint64_t* words,
                                  uint32_t cap, uint32_t* n_words) {
  if (!options_ok(opt) || !queryname(*opt) || !record || !n_words) return FGB_ERR_INVALID_ARG;
  if (len < 32) return FGB_ERR_LAYOUT;
  const int W = key_words(*opt, record[8]);
  *n_words = static_cast<uint32_t>(W);
  if (cap < static_cast<uint32_t>(W) || !words) return FGB_ERR_INVALID_ARG;
  sk::NameEncoder enc;
  enc.init(record, len, opt->order == FGB_SORT_QUERYNAME_NATURAL);
  for (int w = 0; w + 1 < W; ++w) words[w] = enc.word();
  words[W - 1] = sk::name_last_word(enc, record);
  return FGB_OK;
}

fgb_status fgb_sort_records(fgb_handle* h, const fgb_sort_options* opt, const char* header_text, size_t header_len,
                            const uint8_t* records, const uint64_t* rec_off, uint64_t n_records, uint8_t* out,
                            uint64_t cap, uint64_t* out_len, uint64_t* bad_record) {
  if (!h || !out_len || !args_ok(opt, header_text, header_len, records, rec_off, n_records)) return FGB_ERR_INVALID_ARG;
  const link::HandleInfo hi = link::info(h, link::Command::kSort);
  if (bad_record) *bad_record = kNone;
  std::fill(hi.timing, hi.timing + 6, 0.0);
  if (!records_ok(rec_off, n_records, bad_record)) {
    *hi.last_error = "fgb_sort_records: record " + std::to_string(*bad_record) + " is shorter than 32 bytes";
    return FGB_ERR_LAYOUT;
  }
  const uint64_t need = rec_off[n_records] - rec_off[0] + 4 * n_records;
  if (cap < need || (need && !out)) {
    *hi.last_error = "fgb_sort_records: the output needs " + std::to_string(need) + " bytes";
    return FGB_ERR_INVALID_ARG;
  }
  if (hi.busy) { *hi.last_error = "fgb_sort_records: a submit has not been waited on"; return FGB_ERR_BUSY; }
  *out_len = need;
  if (!n_records) return FGB_OK;
  return link::guarded(hi.last_error, "fgb_sort_records", [&] {
    return sort_impl(hi, *opt, std::string_view(header_text ? header_text : "", header_len), records, rec_off,
                     n_records, out);
  });
}

fgb_status fgb_sort_last_timing(const fgb_handle* h, double ms[6]) {
  if (!h || !ms) return FGB_ERR_INVALID_ARG;
  std::memcpy(ms, link::info(const_cast<fgb_handle*>(h), link::Command::kSort).timing, 6 * sizeof(double));
  return FGB_OK;
}

}  // extern "C"
