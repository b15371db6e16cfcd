// C++ client of the batch driver over the device keyframe store (include/b200reg.h,
// b200reg_batch_submit_perform_loop_closure): ingests a keyframe sequence, submits the query keyframes in batches of 16
// with the candidate search left to the jobs, and waits, through the C ABI alone.
//   keyframe_batch_client <dir> <n_keyframes> <points_per_keyframe> <n_queries> <depth>
// <dir> holds clouds.bin (n_keyframes x points x 4 float32: x y z intensity, LiDAR frame), poses.bin (n_keyframes x 16
// float64, row-major), stamps.bin (n_keyframes float64) and queries.bin (n_queries int32).  Prints one JSON line with the
// result and Quatro records as hex, and what b200reg_keyframes_destroy returned with jobs in flight and after them.
#include <cstdio>
#include <cstdlib>
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

static void hex(const void* p, size_t bytes) {
  const unsigned char* b = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < bytes; i++) printf("%02x", b[i]);
}

int main(int argc, char** argv) {
  if (argc < 6) return 2;
  const std::string dir = argv[1];
  const int nk = atoi(argv[2]), nq = atoi(argv[4]), depth = atoi(argv[5]);
  const size_t pts = strtoul(argv[3], nullptr, 10);
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
  b200reg_loop_config cfg;
  b200reg_default_loop_config(&cfg);
  std::vector<b200reg_result> res(nq);
  std::vector<b200reg_quatro_info> qi(nq);
  std::vector<int64_t> tickets;
  for (int i = 0; i < nq && !rc; i += 16) {  // closest_idx NULL: each job runs fetchClosestKeyframeIdx itself
    const int n = nq - i < 16 ? nq - i : 16;
    const int64_t t = b200reg_batch_submit_perform_loop_closure(batch, kf, n, &queries[i], nullptr, &cfg, &res[i], &qi[i]);
    if (t < 0) rc = (int)t;
    else tickets.push_back(t);
  }
  const int destroy_in_flight = rc ? 0 : b200reg_keyframes_destroy(ctx, kf);  // refused: the jobs read the store
  for (int64_t t : tickets) {
    const int r = b200reg_batch_wait(batch, t, nullptr);
    if (r && !rc) rc = r;
  }
  if (rc) fprintf(stderr, "error %d: %s\n", rc, b200reg_last_error());
  const int size = b200reg_keyframes_size(kf);
  const int destroy_after = b200reg_keyframes_destroy(ctx, kf);
  int valid = 0;
  for (int i = 0; i < nq; i++) valid += res[i].valid;
  printf("{\"status\": %d, \"keyframes\": %d, \"valid\": %d, \"destroy_in_flight\": %d, \"destroy_after\": %d, \"results\": \"", rc,
         size, valid, destroy_in_flight, destroy_after);
  hex(res.data(), sizeof(b200reg_result) * res.size());
  printf("\", \"quatro\": \"");
  hex(qi.data(), sizeof(b200reg_quatro_info) * qi.size());
  printf("\"}\n");
  b200reg_batch_destroy(batch);
  b200reg_ctx_destroy(ctx);
  return rc != 0;
}
