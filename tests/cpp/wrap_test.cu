// CPU checks of the 32-bit counters of the barriers and of the LL Allreduce: flag_reached and
// ll_seq_next (kernels.cuh), a simulation of the host's launch schedule (next_comm and
// resync_after_error in b200mpi.cu) across the epoch wrap, and the parser of the counter settings
// (hostutil.h).  Host code only: no GPU is touched.
//
//   wrap_test            every check, with the scrub period clamped as the library does
//   wrap_test --period P the schedule simulation alone with an UNCLAMPED scrub period P; prints
//                        "ahead" lines for every row or counter that looks ahead of the value waited for
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../mpi_b200/csrc/hostutil.h"
#include "../../mpi_b200/csrc/kernels.cuh"

using namespace b200;

static int failures = 0;
#define CHECK(cond, ...)                            \
  do {                                              \
    if (!(cond)) {                                  \
      if (++failures <= 20) {                       \
        printf("FAIL %s:%d: ", __FILE__, __LINE__); \
        printf(__VA_ARGS__);                        \
        printf("\n");                               \
      }                                             \
    }                                               \
  } while (0)

static uint64_t rng_state = 0x6a09e667f3bcc909ull;
static uint64_t next_rand() {
  rng_state += 0x9e3779b97f4a7c15ull;
  return mix64(rng_state);
}

static void test_flag_reached() {
  const uint32_t wants[] = {0u, 1u, 4096u, 0x7fffffffu, 0x80000000u, 0x80000001u, 0xfffff001u, 0xffffffffu};
  for (uint32_t w : wants) {
    CHECK(flag_reached(w, w), "lag 0 at %u", w);
    CHECK(!flag_reached(w - 1u, w), "lag 1 at %u", w);
    CHECK(!flag_reached(w - 2u, w), "lag 2 at %u", w);
    CHECK(!flag_reached(w - 0x7fffffffu, w), "lag 2^31-1 at %u", w);
    CHECK(!flag_reached(w - 0x80000000u, w), "lag 2^31 at %u", w);
    CHECK(flag_reached(w - 0x80000001u, w), "lag 2^31+1 must look ahead (2^31-1) at %u", w);
    CHECK(flag_reached(w + 1u, w), "lead 1 at %u", w);
    CHECK(flag_reached(w + 0x7fffffffu, w), "lead 2^31-1 at %u", w);
  }
  // pairs that straddle 0
  CHECK(flag_reached(0u, 0xffffffffu) && !flag_reached(0xffffffffu, 0u), "0 vs 2^32-1");
  CHECK(flag_reached(4095u, 0xfffff001u) && !flag_reached(0xfffff001u, 4095u), "end of the wrap launch vs its start");
  CHECK(flag_reached(1u, 0xfffff001u) && !flag_reached(0xfffff001u, 1u), "first launch after the wrap vs the wrap launch");
  CHECK(flag_reached(8u, 0xffff8008u) && !flag_reached(0xffff8008u, 8u), "ring counters across their wrap");
  // flags_reached (the start barrier's six-word test) == six flag_reached, on edges and random words
  const uint32_t lags[] = {0u, 1u, 2u, 0x7fffffffu, 0x80000000u, 0x80000001u, 0xfffffffeu, 0xffffffffu};
  for (int i = 0; i < 200000; ++i) {
    const uint64_t r = next_rand();
    const uint32_t want = i < 1000 ? wants[i % 8] : (uint32_t)r;
    uint32_t v[6];
    for (int k = 0; k < 6; ++k) {
      const uint64_t q = next_rand();
      v[k] = want - (i & 1 ? lags[q % 8] : (uint32_t)q);
    }
    bool all = true;
    for (int k = 0; k < 6; ++k) all = all && flag_reached(v[k], want);
    CHECK(flags_reached(v[0], v[1], v[2], v[3], v[4], v[5], want) == all, "flags_reached differs from six flag_reached at want %u", want);
  }
}

// ---------------------------------------------------------------------------------------------
// The host schedule: next_comm (a scrub with the largest grid before every launch whose epoch index
// is scrub_every - 1 mod scrub_every, then the collective) and resync_after_error (one stride, no
// launch).  Values are kept unwrapped in 64 bits, offset by 2^40 so that the preset below stays
// positive; the device sees the low 32 bits.
// ---------------------------------------------------------------------------------------------
struct Schedule {
  uint32_t every;
  uint64_t epoch;
  std::vector<uint64_t> cell, flag, ring; // per slot row: last start value, last end value, last ring counter
  uint64_t launches = 0, ahead = 0, end0_launches = 0, end0_scrubs = 0, end0_skips = 0;
  uint64_t last_scrub_index = UINT64_MAX, scrubs = 0;
  bool verbose = false;

  Schedule(uint32_t e0, uint32_t every_) : every(every_), epoch((1ull << 40) + e0) {
    // the preset of B200MPI_EPOCH_START (b200mpi.cu: preset_control_region)
    cell.assign(kMaxBlocks, epoch - (uint64_t)kScrubEvery * kEpochStride);
    flag.assign(kMaxBlocks, epoch - 1);
    ring.assign(kMaxBlocks, (epoch - kEpochStride) * 8);
  }
  uint64_t index() const { return (epoch - 1) / kEpochStride; }
  // next_comm's rule, on the 32-bit epoch the library holds (its index has 20 bits)
  bool scrub_due_at(uint64_t e) const { return (((uint32_t)e / kEpochStride) & (every - 1)) == every - 1; }
  bool scrub_due() const { return scrub_due_at(epoch); }
  // `have` was last written, the launch waits for every value in [lo, hi]: have must be behind lo as the
  // device compares, and lag hi by less than 2^31 in truth.
  void expect_behind(const char* what, int row, uint64_t have, uint64_t lo, uint64_t hi) {
    const bool looks_ahead = flag_reached((uint32_t)have, (uint32_t)lo);
    const bool too_far = hi - have >= (1ull << 31);
    if (looks_ahead || too_far) {
      if (++ahead <= 5 && verbose) printf("ahead: %s row %d: value %u against %u..%u (true lag %llu) at launch %llu\n", what, row, (uint32_t)have,
                                          (uint32_t)lo, (uint32_t)hi, (unsigned long long)(hi - have), (unsigned long long)launches);
    }
  }
  void one(int grid, bool scrub, int ring_steps) {
    const uint64_t e = epoch, end = e + kEpochStride - 1;
    if ((uint32_t)end == 0) {
      ++end0_launches;
      if (scrub) ++end0_scrubs;
    }
    for (int b = 0; b < grid; ++b) {
      expect_behind("slot cell", b, cell[b], e, e);
      expect_behind("slot flag", b, flag[b], e + 1, end);
      if (ring_steps > 0) expect_behind("ring counter", b, ring[b], e * 8 + 1, e * 8 + ring_steps);
      cell[b] = e;
      flag[b] = end;
      if (scrub) ring[b] = e * 8;
      else if (ring_steps > 0) ring[b] = e * 8 + ring_steps;
    }
    ++launches;
    epoch += kEpochStride;
  }
  void launch(int grid, int ring_steps) {
    if (scrub_due()) {
      const uint64_t k = index();
      if (last_scrub_index != UINT64_MAX) {
        // every scrub-due index between two scrubs was consumed by a resync
        CHECK(k - last_scrub_index == every || skipped_scrub, "scrub at index %llu after %llu (period %u)", (unsigned long long)k,
              (unsigned long long)last_scrub_index, every);
      }
      last_scrub_index = k;
      skipped_scrub = false;
      ++scrubs;
      one(kMaxBlocks, true, 0);
    }
    one(grid, false, ring_steps);
  }
  void resync() {
    if ((uint32_t)(epoch + kEpochStride - 1) == 0) ++end0_skips;
    if (scrub_due()) skipped_scrub = true;
    epoch += kEpochStride;
  }
  bool skipped_scrub = false;
};

// More than 3 * 2^20 launches from `e0`, shaped like a job of small messages: random grids of 1..16
// CTAs, and about once per 2^19 launches a full grid of 132 (the SM count: block_cap).  A quarter of
// the launches are ring kernels (1..14 steps); about one in 4096 fails and is followed by a resync.
// Once in the run the worst case is played: a failed call lands just before a scrub is due, so that
// its resync skips that scrub, and the last launch before the next scrub is a full-grid ring kernel.
static Schedule simulate(uint32_t e0, uint32_t every, bool verbose) {
  Schedule s(e0, every);
  s.verbose = verbose;
  const uint64_t total = 3ull * (1u << 20) + 4096;
  constexpr int kFullGrid = 132;
  bool skipped_one = false, big_ring_due = false;
  const uint64_t first = s.epoch;
  while (s.launches < total) {
    const uint64_t r = next_rand();
    // the next index is the last before a scrub
    const bool before_scrub = s.scrub_due_at(s.epoch + kEpochStride) && !s.scrub_due();
    int grid = ((r >> 40) & ((1u << 19) - 1)) == 0 ? kFullGrid : 1 + (int)(r % 16);
    int steps = ((r >> 20) & 3) == 0 ? 1 + (int)((r >> 24) % 14) : 0;
    if (big_ring_due && before_scrub) {
      grid = kFullGrid;
      steps = 14;
      big_ring_due = false;
    }
    s.launch(grid, steps); // when it fails, every rank resyncs
    const bool scrub_due = s.scrub_due();
    if (((r >> 32) & 4095) == 0 || (!skipped_one && scrub_due && s.launches > (1u << 20))) {
      if (scrub_due && !skipped_one) skipped_one = big_ring_due = true;
      s.resync();
    }
  }
  const uint64_t wraps = ((s.epoch - 1) >> 32) - ((first - 1) >> 32);
  if (!verbose) {
    CHECK(s.ahead == 0, "start %u period %u: %llu rows or counters looked ahead", e0, every, (unsigned long long)s.ahead);
    CHECK(wraps >= 3, "start %u: only %llu wraps", e0, (unsigned long long)wraps);
    CHECK(s.end0_launches + s.end0_skips == wraps, "start %u: %llu launches and %llu resyncs with end value 0 over %llu wraps", e0,
          (unsigned long long)s.end0_launches, (unsigned long long)s.end0_skips, (unsigned long long)wraps);
    // 2^20 - 1 is scrub_every - 1 mod every period: the launch that ends on 0 is always the scrub
    CHECK(s.end0_scrubs == s.end0_launches, "start %u: a launch other than the scrub ended on 0", e0);
    CHECK(skipped_one, "start %u: the run never skipped a scrub", e0);
  }
  return s;
}

static const uint32_t kStarts[] = {1u, (1u << 29) - 40 * kEpochStride + 1, (1u << 31) - 40 * kEpochStride + 1, (uint32_t)((1ull << 32) - 40 * kEpochStride + 1)};

static void test_schedule() {
  for (uint32_t e0 : kStarts) {
    simulate(e0, kScrubEvery, false);
    simulate(e0, 4, false); // the period the GPU tests use
  }
}

static void test_ll_seq() {
  // +1 (a call) never yields 0 and reports exactly the crossing
  for (uint32_t last : {0u, 1u, 2u, 0x7fffffffu, 0x80000000u, 0xfffffffcu, 0xfffffffdu, 0xfffffffeu}) {
    const LLSeqNext x = ll_seq_next(last, 1);
    CHECK(!x.wrapped && x.seq == last + 1, "+1 from %u", last);
  }
  LLSeqNext w = ll_seq_next(0xffffffffu, 1);
  CHECK(w.wrapped && w.seq == 1, "+1 from 2^32-1: %u %d", w.seq, w.wrapped);
  // +2 (resync) landing on 2^32-2, 2^32-1 (no crossing), 0 and 1 (crossing)
  w = ll_seq_next(0xfffffffcu, 2);
  CHECK(!w.wrapped && w.seq == 0xfffffffeu, "resync onto 2^32-2");
  w = ll_seq_next(0xfffffffdu, 2);
  CHECK(!w.wrapped && w.seq == 0xffffffffu, "resync onto 2^32-1");
  w = ll_seq_next(0xfffffffeu, 2);
  CHECK(w.wrapped && w.seq != 0, "resync onto 0: %u %d", w.seq, w.wrapped);
  w = ll_seq_next(0xffffffffu, 2);
  CHECK(w.wrapped && w.seq != 0, "resync onto 1: %u %d", w.seq, w.wrapped);
  // walks over two wraps with random resyncs: one report per crossing, never 0
  for (uint32_t start : {0xffff0000u, 0xfffffff0u, 0u}) {
    uint32_t seq = start;
    uint64_t reports = 0;
    for (uint64_t i = 0; i < 3u * 65536u + 7; ++i) {
      const uint32_t step = (next_rand() & 15) == 0 ? 2 : 1;
      const LLSeqNext x = ll_seq_next(seq, step);
      const bool crosses = (uint64_t)seq + step >= (1ull << 32);
      CHECK(x.seq != 0, "yielded 0 from %u", seq);
      CHECK(x.wrapped == crosses, "%u + %u: wrapped %d", seq, step, x.wrapped);
      reports += x.wrapped;
      seq = x.seq;
      if (i == 65536) seq = 0xfffffff8u; // close to the wrap again
    }
    CHECK(reports == (start == 0 ? 1u : 2u), "start %u: %llu wraps reported", start, (unsigned long long)reports);
  }
}

static void test_env_parser() {
  CounterEnv e;
  CHECK(parse_counter_env(nullptr, nullptr, nullptr, kScrubEvery, kEpochStride, e).empty() && e.scrub_every == kScrubEvery && e.epoch_start == 1 &&
            e.ll_seq_start == 0 && !e.preset,
        "defaults");
  const struct { const char* in; uint32_t want; } scrub[] = {{"4", 4}, {"5", 4}, {"0", 2}, {"1", 2}, {"2", 2}, {"16384", kScrubEvery}, {"16385", kScrubEvery},
                                                             {"65536", kScrubEvery}, {"2097152", kScrubEvery}, {"4294967295", kScrubEvery}, {"010", 8}, {"0256", 256}};
  for (auto& s : scrub) {
    const std::string err = parse_counter_env(s.in, nullptr, nullptr, kScrubEvery, kEpochStride, e);
    CHECK(err.empty() && e.scrub_every == s.want, "B200MPI_SCRUB_EVERY=%s -> %u (%s)", s.in, e.scrub_every, err.c_str());
  }
  for (const char* bad : {"", "x", "4k", "-4", "+4", " 4", "4 ", " ", "1e3", "0x100", "4294967296", "99999999999999999999"}) {
    CHECK(!parse_counter_env(bad, nullptr, nullptr, kScrubEvery, kEpochStride, e).empty(), "B200MPI_SCRUB_EVERY='%s' accepted", bad);
    CHECK(!parse_counter_env(nullptr, bad, nullptr, kScrubEvery, kEpochStride, e).empty(), "B200MPI_EPOCH_START='%s' accepted", bad);
    CHECK(!parse_counter_env(nullptr, nullptr, bad, kScrubEvery, kEpochStride, e).empty(), "B200MPI_LL_SEQ_START='%s' accepted", bad);
  }
  for (const char* bad : {"0", "2", "4096", "4098", "4294963200", "4294967295", "010", "0xfffff001"})
    CHECK(!parse_counter_env(nullptr, bad, nullptr, kScrubEvery, kEpochStride, e).empty(), "epoch start %s is not 1 mod 4096 but was accepted", bad);
  for (const char* good : {"1", "4097", "04097", "4294963201", "2147479553"}) {
    const std::string err = parse_counter_env(nullptr, good, nullptr, kScrubEvery, kEpochStride, e);
    CHECK(err.empty() && e.preset && e.epoch_start == (uint32_t)strtoull(good, nullptr, 10), "epoch start %s rejected: %s", good, err.c_str());
  }
  CHECK(parse_counter_env(nullptr, nullptr, "4294967291", kScrubEvery, kEpochStride, e).empty() && e.ll_seq_start == 4294967291u && !e.preset, "ll seq start");
}

int main(int argc, char** argv) {
  if (argc == 3 && strcmp(argv[1], "--period") == 0) {
    const uint32_t every = (uint32_t)strtoul(argv[2], nullptr, 0);
    uint64_t ahead = 0, scrubs = 0;
    for (uint32_t e0 : kStarts) {
      const Schedule s = simulate(e0, every, true);
      ahead += s.ahead;
      scrubs += s.scrubs;
    }
    printf("period %u: %llu rows or counters looked ahead, %llu scrubs ran\n", every, (unsigned long long)ahead, (unsigned long long)scrubs);
    return 0;
  }
  test_flag_reached();
  test_ll_seq();
  test_env_parser();
  test_schedule();
  if (failures) {
    printf("%d failures\n", failures);
    return 1;
  }
  printf("wrap ok\n");
  return 0;
}
