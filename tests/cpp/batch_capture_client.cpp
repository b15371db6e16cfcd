// C++ client of the batch driver that publishes what loopTimerFunc publishes (fast_lio_sam_qn.cpp:245-248) from driver jobs,
// through the C ABI alone (include/b200reg.h): every tick collects the job the previous tick submitted -- its results, its
// source, target, coarse-aligned and final-aligned clouds and its LM trace (setDebugPrint's table) -- releases it, then
// submits this tick's queries with the candidate search left to the job.
//   batch_capture_client <dir> <n_keyframes> <points_per_keyframe> <n_queries> <queries_per_tick> <depth>
// <dir> holds clouds.bin (n_keyframes x points x 4 float32: x y z intensity, LiDAR frame), poses.bin (n_keyframes x 16
// float64, row-major), stamps.bin (n_keyframes float64) and queries.bin (n_queries int32).  For tick k it writes what it
// would publish to <dir>/tick<k>_<kind>.bin (kind 1, 2, 4, 8: the clouds of the tick's queries, x y z intensity) and
// <dir>/tick<k>_trace.bin (b200reg_lm_trial records), and prints one JSON line with each tick's CSR offsets, validity
// flags and the result records as hex.
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <string>
#include <vector>

#include "../../include/b200reg.h"

template <class T>
static std::vector<T> read_bin(const std::string& path, size_t n) {
  std::vector<T> v(n);
  FILE* f = fopen(path.c_str(), "rb");
  if (!f || fread(v.data(), sizeof(T), n, f) != n) {
    fprintf(stderr, "cannot read %s\n", path.c_str());
    exit(2);
  }
  fclose(f);
  return v;
}

template <class T>
static void write_bin(const std::string& path, const std::vector<T>& v) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f || fwrite(v.data(), sizeof(T), v.size(), f) != v.size()) {
    fprintf(stderr, "cannot write %s\n", path.c_str());
    exit(2);
  }
  fclose(f);
}

static void print_offsets(const std::vector<int64_t>& o) {
  printf("[");
  for (size_t i = 0; i < o.size(); i++) printf("%s%lld", i ? ", " : "", (long long)o[i]);
  printf("]");
}

static void hex(const void* p, size_t bytes) {
  const unsigned char* b = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < bytes; i++) printf("%02x", b[i]);
}

struct Pending {
  int tick;
  int64_t ticket;
  std::vector<int32_t> query;
  std::vector<b200reg_result> res;
  std::vector<b200reg_quatro_info> qi;
};

// One tick's collection: wait, read every kind and the trace by ticket (the getters' CSR: count, offsets, then the
// records), publish them, release the ticket.  Returns the first error.
static int collect(b200reg_batch* batch, Pending& p, const std::string& dir, bool first) {
  int rc = b200reg_batch_wait(batch, p.ticket, nullptr);
  printf("%s{\"tick\": %d, \"status\": %d", first ? "" : ", ", p.tick, rc);
  if (!rc) {
    const int kinds[4] = {B200REG_CLOUD_SOURCE, B200REG_CLOUD_TARGET, B200REG_CLOUD_COARSE, B200REG_CLOUD_FINAL};
    printf(", \"offsets\": {");
    for (int k = 0; k < 4 && !rc; k++) {
      const int pairs = b200reg_batch_loop_clouds(batch, p.ticket, kinds[k], nullptr, 0, nullptr);
      if (pairs < 0) {
        rc = pairs;
        break;
      }
      std::vector<int64_t> offsets(pairs + 1);
      int r = b200reg_batch_loop_clouds(batch, p.ticket, kinds[k], offsets.data(), 0, nullptr);  // offsets only
      if (r != B200REG_OK && r != B200REG_ESTATE) rc = r;
      std::vector<float> xyzi(4 * (size_t)offsets[pairs]);
      if (!rc) rc = b200reg_batch_loop_clouds(batch, p.ticket, kinds[k], offsets.data(), (size_t)offsets[pairs], xyzi.data());
      write_bin(dir + "/tick" + std::to_string(p.tick) + "_" + std::to_string(kinds[k]) + ".bin", xyzi);  // the publish
      printf("%s\"%d\": ", k ? ", " : "", kinds[k]);
      print_offsets(offsets);
    }
    printf("}");
    const int pairs = rc ? rc : b200reg_batch_lm_trace(batch, p.ticket, nullptr, 0, nullptr);
    if (pairs < 0) {
      if (!rc) rc = pairs;
    } else {
      std::vector<int64_t> offsets(pairs + 1);
      const int r = b200reg_batch_lm_trace(batch, p.ticket, offsets.data(), 0, nullptr);
      if (r != B200REG_OK && r != B200REG_ESTATE) rc = r;
      std::vector<b200reg_lm_trial> trials((size_t)offsets[pairs]);
      if (!rc) rc = b200reg_batch_lm_trace(batch, p.ticket, offsets.data(), trials.size(), trials.data());
      write_bin(dir + "/tick" + std::to_string(p.tick) + "_trace.bin", trials);
      printf(", \"trace_offsets\": ");
      print_offsets(offsets);
    }
    printf(", \"results\": \"");
    hex(p.res.data(), sizeof(b200reg_result) * p.res.size());
    printf("\", \"quatro\": \"");
    hex(p.qi.data(), sizeof(b200reg_quatro_info) * p.qi.size());
    printf("\"");
  }
  const int released = b200reg_batch_release(batch, p.ticket);
  printf(", \"released\": %d, \"after_release\": %d}", released, b200reg_batch_loop_clouds(batch, p.ticket, B200REG_CLOUD_FINAL, nullptr, 0, nullptr));
  if (rc) fprintf(stderr, "tick %d: error %d: %s\n", p.tick, rc, b200reg_last_error());
  return rc;
}

int main(int argc, char** argv) {
  if (argc < 7) return 2;
  const std::string dir = argv[1];
  const int nk = atoi(argv[2]), nq = atoi(argv[4]), per_tick = atoi(argv[5]), depth = atoi(argv[6]);
  const size_t pts = strtoul(argv[3], nullptr, 10);
  if (per_tick < 1) return 2;
  const std::vector<float> clouds = read_bin<float>(dir + "/clouds.bin", (size_t)nk * pts * 4);
  const std::vector<double> poses = read_bin<double>(dir + "/poses.bin", (size_t)nk * 16);
  const std::vector<double> stamps = read_bin<double>(dir + "/stamps.bin", (size_t)nk);
  const std::vector<int32_t> queries = read_bin<int32_t>(dir + "/queries.bin", (size_t)nq);

  b200reg_ctx* ctx = nullptr;
  b200reg_keyframes* kf = nullptr;
  b200reg_batch* batch = nullptr;
  int rc = b200reg_ctx_create(0, &ctx);
  if (!rc) rc = b200reg_keyframes_create(ctx, &kf);
  if (!rc) rc = b200reg_batch_create(0, depth, &batch);
  for (int i = 0; i < nk && !rc; i++) {
    const int idx = b200reg_keyframes_add(ctx, kf, &clouds[(size_t)i * pts * 4], pts, 16, &poses[16 * (size_t)i], stamps[i]);
    if (idx != i) rc = idx < 0 ? idx : -1;
  }
  // the debug topics: all four clouds and setDebugPrint's trace, for every job submitted from here on
  if (!rc) rc = b200reg_batch_set_loop_clouds(batch, B200REG_CLOUD_SOURCE | B200REG_CLOUD_TARGET | B200REG_CLOUD_COARSE | B200REG_CLOUD_FINAL);
  if (!rc) rc = b200reg_batch_set_lm_trace(batch, 1);
  b200reg_loop_config cfg;
  b200reg_default_loop_config(&cfg);
  std::deque<Pending> pending;  // a deque never moves its elements on push_back: the jobs' output arrays stay put
  bool first = true;
  printf("{\"ticks\": [");
  for (int i = 0, tick = 0; i < nq && !rc; i += per_tick, tick++) {  // one loopTimerFunc tick
    while (!pending.empty() && !rc) {
      rc = collect(batch, pending.front(), dir, first);
      first = false;
      pending.pop_front();
    }
    const int n = nq - i < per_tick ? nq - i : per_tick;
    pending.push_back({tick, -1, std::vector<int32_t>(&queries[i], &queries[i] + n), std::vector<b200reg_result>(n),
                       std::vector<b200reg_quatro_info>(n)});
    Pending& p = pending.back();
    p.ticket = b200reg_batch_submit_perform_loop_closure(batch, kf, n, p.query.data(), nullptr, &cfg, p.res.data(), p.qi.data());
    if (p.ticket < 0) rc = (int)p.ticket;
  }
  while (!pending.empty() && !rc) {  // shutdown: the last tick's job
    rc = collect(batch, pending.front(), dir, first);
    first = false;
    pending.pop_front();
  }
  if (rc) {
    fprintf(stderr, "error %d: %s\n", rc, b200reg_last_error());
    b200reg_batch_wait_all(batch);
  }
  printf("], \"status\": %d}\n", rc);
  b200reg_batch_destroy(batch);
  b200reg_keyframes_destroy(ctx, kf);
  b200reg_ctx_destroy(ctx);
  return rc != 0;
}
