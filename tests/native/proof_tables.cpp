// Checks the proof tables of host_tables.cpp that the C-ABI does not expose (qt3, sumt, pair_q) -- and qt again, at
// every depth -- against the oracle's ConsensusBaseBuilder add / call sequence, over a grid of error-rate settings.
// Every check builds the worst pileup a table entry admits and asks the oracle for its call: whatever the kernels take
// from a table without looking must be what the reference's literal f64 algorithm returns.
//
// usage: proof_tables            prints one "table <name> checks <n> active <settings>" line per table, then "ok"
// A failing check prints "FAIL ..." and exits 1.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "../../oracle/fgumi_oracle.hpp"
#include "host_tables.h"

namespace {

const unsigned kGrid[] = {0, 1, 2, 3, 10, 20, 30, 45, 60, 70, 75, 80, 85, 90, 93};
const uint8_t kBases[4] = {'A', 'C', 'G', 'T'};

struct Tally {
  const char* name;
  uint64_t checks = 0;
  unsigned active = 0;
};

[[noreturn]] void fail(unsigned pre, unsigned post, const char* what, unsigned n, unsigned extra, uint8_t got_b,
                       uint8_t got_q, uint8_t want_b, unsigned want_q) {
  std::printf("FAIL pre=%u post=%u %s n=%u extra=%u got=(%c,%u) want=(%c,%u)\n", pre, post, what, n, extra, got_b,
              got_q, want_b, want_q);
  std::exit(1);
}

// One pileup through the oracle; `obs` holds (base, quality) in the order they are added.
void call_oracle(fgoracle::ConsensusBaseBuilder& bb, const std::vector<std::pair<uint8_t, uint8_t>>& obs, uint8_t* b,
                 uint8_t* q) {
  bb.reset();
  for (const auto& o : obs) bb.add(o.first, o.second);
  bb.call(b, q);
}

double dval(const fgb::HostTables& t, unsigned q) { return t.correct[q] - t.err_alt[q]; }

// the quality in [lo, 93] whose D is smallest (the worst a threshold admits) or largest (the strongest dissenter)
unsigned arg_d(const fgb::HostTables& t, unsigned lo, bool largest) {
  unsigned best = lo;
  for (unsigned q = lo; q <= 93; ++q) {
    const double d = dval(t, q), b = dval(t, best);
    if (largest ? d > b : d < b) best = q;
  }
  return best;
}

// Dissenters at row indices of an n-row pileup: first rows, last rows, or spread evenly.
std::vector<unsigned> placement(unsigned n, unsigned k, int where) {
  std::vector<unsigned> at;
  for (unsigned i = 0; i < k; ++i) {
    if (where == 0) at.push_back(i);
    else if (where == 1) at.push_back(n - k + i);
    else at.push_back((i * 2 + 1) * n / (2 * k));
  }
  return at;
}

}  // namespace

int main() {
  Tally t_qt{"qt"}, t_qt3{"qt3"}, t_pair{"pair_q"}, t_sumt3{"sumt3"}, t_sumt4{"sumt4"}, t_degen{"degenerate"};
  std::mt19937 rng(12345);
  unsigned sumt_full = 0;
  std::vector<std::pair<uint8_t, uint8_t>> obs;
  obs.reserve(512);
  for (unsigned pre : kGrid) {
    for (unsigned post : kGrid) {
      static fgb::HostTables t;
      fgb::build_host_tables(pre, post, &t);
      fgoracle::ConsensusBaseBuilder bb(static_cast<uint8_t>(pre), static_cast<uint8_t>(post));
      const unsigned fq = t.fast_qual;
      uint8_t gb, gq;

      // ---- degenerate settings: no proof may fire where the tables give none ----
      if (t.nmax2 == 0) {
        for (unsigned n = 0; n < 256; ++n) {
          if (t.qt[n] != 255 || t.qt3[n] != 255) fail(pre, post, "nmax2=0 leaves qt/qt3 on", n, t.qt[n], 0, t.qt3[n], 0, 255);
          ++t_degen.checks;
        }
        for (unsigned n = 0; n < 8; ++n) {
          if (t.sumt[n] != 0xFFFF) fail(pre, post, "nmax2=0 leaves sumt on", n, t.sumt[n], 0, 0, 0, 0xFFFF);
          ++t_degen.checks;
        }
        ++t_degen.active;
      }
      if (post == 1) {
        for (unsigned n = 0; n < 256; ++n) {
          if (t.qt[n] != 255 || t.qt3[n] != 255) fail(pre, post, "post=1 leaves qt/qt3 on", n, t.qt[n], 0, t.qt3[n], 0, 255);
          ++t_degen.checks;
        }
        ++t_degen.active;
      }

      // ---- qt[n]: n identical observations at the weakest quality >= qt[n] (n >= 255 reads qt[255]) ----
      bool any = false;
      for (unsigned n = 1; n <= 300; ++n) {
        const unsigned thr = t.qt[n < 255 ? n : 255];
        if (thr > 93) continue;
        any = true;
        const unsigned qw = arg_d(t, thr, false);
        for (unsigned q : {qw, thr}) {
          const uint8_t b = kBases[(n + q) & 3];
          obs.assign(n, {b, static_cast<uint8_t>(q)});
          call_oracle(bb, obs, &gb, &gq);
          if (gb != b || gq != fq) fail(pre, post, "qt", n, q, gb, gq, b, fq);
          ++t_qt.checks;
        }
      }
      t_qt.active += any;

      // ---- qt3[n]: a majority at the weakest quality >= qt3[n] with up to kNearK dissenters ----
      any = false;
      for (unsigned n = 7; n <= 254; ++n) {
        const unsigned thr = t.qt3[n];
        if (thr > 93) continue;
        any = true;
        if (t.qt3[n] < t.qt[n]) fail(pre, post, "qt3 below qt", n, t.qt[n], 0, t.qt3[n], 0, t.qt[n]);
        const unsigned qw = arg_d(t, thr, false), qs = arg_d(t, 1, true);
        std::uniform_int_distribution<unsigned> qdist(thr, 93);
        for (unsigned k = 0; k <= fgb::kNearK; ++k) {
          for (int where = 0; where < 3; ++where) {
            const std::vector<unsigned> at = placement(n, k, where);
            for (int kind = 0; kind < 3; ++kind) {
              const uint8_t maj = kBases[(n + k + where + kind) & 3];
              obs.assign(n, {maj, static_cast<uint8_t>(qw)});
              for (unsigned i = 0; i < k; ++i) {
                // kind 0: one dissenting base at the strongest quality; 1: split over the other bases; 2: random
                // qualities >= qt3[n] for every row
                uint8_t db = kBases[(maj == 'A' ? 1 : 0)];
                if (kind >= 1) db = kBases[(std::find(kBases, kBases + 4, maj) - kBases + 1 + i) & 3];
                obs[at[i]] = {db, static_cast<uint8_t>(kind == 2 ? qdist(rng) : qs)};
              }
              if (kind == 2)
                for (unsigned r = 0; r < n; ++r)
                  if (obs[r].first == maj) obs[r].second = static_cast<uint8_t>(qdist(rng));
              call_oracle(bb, obs, &gb, &gq);
              if (gb != maj || gq != fq) fail(pre, post, "qt3", n, k * 100 + where * 10 + kind, gb, gq, maj, fq);
              ++t_qt3.checks;
            }
          }
        }
      }
      t_qt3.active += any;

      // ---- pair_q: every ordered pair of qualities 1..93 ----
      any = false;
      for (unsigned q1 = 1; q1 <= 93; ++q1)
        for (unsigned q2 = 1; q2 <= 93; ++q2) {
          const unsigned want = t.pair_q[q1 * 94 + q2];
          if (want == 255) continue;
          any = true;
          const uint8_t b = kBases[(q1 + q2) & 3];
          obs.assign({{b, static_cast<uint8_t>(q1)}, {b, static_cast<uint8_t>(q2)}});
          call_oracle(bb, obs, &gb, &gq);
          if (gb != b || gq != want) fail(pre, post, "pair_q", 2, q1 * 100 + q2, gb, gq, b, want);
          ++t_pair.checks;
        }
      t_pair.active += any;

      // ---- sumt[3], sumt[4]: unanimous multisets of qualities in 1..63 whose sum reaches the threshold.  Settings
      // with the table on are enumerated in full for the first eight of them, otherwise over sums in
      // [sumt, sumt + 8]; each multiset is added in ascending and in descending order. ----
      const bool full = (t.sumt[3] != 0xFFFF || t.sumt[4] != 0xFFFF) && sumt_full < 8;
      sumt_full += full;
      for (unsigned n = 3; n <= 4; ++n) {
        const unsigned lo = t.sumt[n];
        if (lo == 0xFFFF) continue;
        Tally& tl = n == 3 ? t_sumt3 : t_sumt4;
        ++tl.active;
        const unsigned hi = full ? 63 * n : lo + 8;
        unsigned q[4];
        for (q[0] = 1; q[0] <= 63; ++q[0])
          for (q[1] = q[0]; q[1] <= 63; ++q[1])
            for (q[2] = q[1]; q[2] <= 63; ++q[2])
              for (q[3] = (n == 4 ? q[2] : 0); q[3] <= (n == 4 ? 63u : 0u); ++q[3]) {
                const unsigned s = q[0] + q[1] + q[2] + q[3];
                if (s < lo || s > hi) continue;
                const uint8_t b = kBases[s & 3];
                for (int dir = 0; dir < 2; ++dir) {
                  obs.clear();
                  for (unsigned i = 0; i < n; ++i) obs.push_back({b, static_cast<uint8_t>(q[dir ? n - 1 - i : i])});
                  call_oracle(bb, obs, &gb, &gq);
                  if (gb != b || gq != fq) fail(pre, post, n == 3 ? "sumt3" : "sumt4", n, s, gb, gq, b, fq);
                  ++tl.checks;
                }
              }
      }
    }
  }
  for (const Tally* tl : {&t_qt, &t_qt3, &t_pair, &t_sumt3, &t_sumt4, &t_degen})
    std::printf("table %s checks %llu active %u\n", tl->name, static_cast<unsigned long long>(tl->checks), tl->active);
  std::printf("ok\n");
  return 0;
}
