// A client of the C ABI alone (include/b200reg.h) that feeds loopTimerFunc's four publishes (fast_lio_sam_qn.cpp:245-248)
// from one batched call: add keyframes -> fetch the closest keyframes -> perform the loop closures -> the source, target,
// coarse-aligned and final-aligned clouds of every pair.
// usage: loop_clouds_client keyframes.bin out_prefix query...
//   keyframes.bin: int32 count, then per keyframe int64 n, 16 doubles pose (row-major), double stamp, n x 4 float32 (x y z i)
// Prints one JSON line (candidates, validity, per-kind CSR offsets) and writes each kind's points to out_prefix_<kind>.bin.
#include <b200reg.h>

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>
#include <vector>

#define CHECK(call)                                                                         \
  do {                                                                                      \
    const int rc_ = (call);                                                                 \
    if (rc_ < 0) {                                                                          \
      std::fprintf(stderr, "%s failed: %d %s\n", #call, rc_, b200reg_last_error());         \
      std::exit(1);                                                                         \
    }                                                                                       \
  } while (0)

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  int32_t nkf = 0;
  f.read(reinterpret_cast<char*>(&nkf), sizeof(nkf));
  b200reg_ctx* ctx = nullptr;
  CHECK(b200reg_ctx_create(0, &ctx));
  b200reg_keyframes* kf = nullptr;
  CHECK(b200reg_keyframes_create(ctx, &kf));
  for (int k = 0; k < nkf; k++) {
    int64_t n = 0;
    double pose[16], stamp = 0;
    f.read(reinterpret_cast<char*>(&n), sizeof(n));
    f.read(reinterpret_cast<char*>(pose), sizeof(pose));
    f.read(reinterpret_cast<char*>(&stamp), sizeof(stamp));
    std::vector<float> xyzi(4 * (size_t)n);
    f.read(reinterpret_cast<char*>(xyzi.data()), (std::streamsize)(xyzi.size() * sizeof(float)));
    CHECK(b200reg_keyframes_add(ctx, kf, xyzi.data(), (size_t)n, 16, pose, stamp));
  }
  if (!f) return 3;
  std::vector<int32_t> queries;
  for (int a = 3; a < argc; a++) queries.push_back(std::atoi(argv[a]));
  const int count = (int)queries.size();
  b200reg_loop_config cfg;
  b200reg_default_loop_config(&cfg);
  std::vector<int32_t> closest(count);
  CHECK(b200reg_fetch_closest_keyframes(ctx, kf, count, queries.data(), cfg.loop_detection_radius,
                                        cfg.loop_detection_timediff_threshold, closest.data()));
  CHECK(b200reg_ctx_set_loop_clouds(ctx, B200REG_CLOUD_SOURCE | B200REG_CLOUD_TARGET | B200REG_CLOUD_COARSE | B200REG_CLOUD_FINAL));
  std::vector<b200reg_result> res(count);
  std::vector<b200reg_quatro_info> qi(count);
  CHECK(b200reg_perform_loop_closure(ctx, kf, count, queries.data(), closest.data(), &cfg, res.data(), qi.data()));
  std::printf("{\"closest\": [");
  for (int i = 0; i < count; i++) std::printf("%s%d", i ? ", " : "", closest[i]);
  std::printf("], \"quatro_valid\": [");
  for (int i = 0; i < count; i++) std::printf("%s%d", i ? ", " : "", qi[i].valid);
  std::printf("], \"valid\": [");
  for (int i = 0; i < count; i++) std::printf("%s%d", i ? ", " : "", res[i].valid);
  std::printf("], \"offsets\": {");
  const int kinds[4] = {B200REG_CLOUD_SOURCE, B200REG_CLOUD_TARGET, B200REG_CLOUD_COARSE, B200REG_CLOUD_FINAL};
  for (int k = 0; k < 4; k++) {
    const int pairs = b200reg_loop_clouds(ctx, kinds[k], nullptr, 0, nullptr);
    CHECK(pairs);
    std::vector<int64_t> offsets(pairs + 1);
    const int rc = b200reg_loop_clouds(ctx, kinds[k], offsets.data(), 0, nullptr);  // offsets only
    if (rc != B200REG_ESTATE) CHECK(rc);
    std::vector<float> xyzi(4 * (size_t)offsets[pairs]);
    CHECK(b200reg_loop_clouds(ctx, kinds[k], offsets.data(), (size_t)offsets[pairs], xyzi.data()));
    std::ofstream o(std::string(argv[2]) + "_" + std::to_string(kinds[k]) + ".bin", std::ios::binary);
    o.write(reinterpret_cast<const char*>(xyzi.data()), (std::streamsize)(xyzi.size() * sizeof(float)));
    std::printf("%s\"%d\": [", k ? ", " : "", kinds[k]);
    for (int i = 0; i <= pairs; i++) std::printf("%s%lld", i ? ", " : "", (long long)offsets[i]);
    std::printf("]");
  }
  std::printf("}}\n");
  CHECK(b200reg_keyframes_destroy(ctx, kf));
  CHECK(b200reg_ctx_destroy(ctx));
  return 0;
}
