// A client of the C ABI alone (include/b200reg.h) that reads the Quatro correspondences and max-clique inliers of loop
// attempts, as a node would to draw them: add keyframes -> fetch the closest keyframes -> perform the loop closures on a
// context with recording on, then the same attempt as a batch-driver job.
// usage: quatro_matches_client keyframes.bin out_prefix query...
//   keyframes.bin: int32 count, then per keyframe int64 n, 16 doubles pose (row-major), double stamp, n x 4 float32 (x y z i)
// Prints one JSON line (candidates, clique sizes, CSR offsets of the context's and the job's matches, the job's release
// status) and writes each set of matches to out_prefix_<ctx|job>.bin: corr (2 x int32), inlier (int32), src xyz and dst xyz
// (3 x float32 each), one block per array over all rows.
#include <b200reg.h>

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <functional>
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

typedef std::function<int(int64_t*, size_t, int32_t*, int32_t*, float*, float*)> Getter;

// reads one set of matches through `get` (b200reg_quatro_matches' rules), writes it to `path`, prints its offsets
static void dump(const Getter& get, const std::string& path) {
  const int pairs = get(nullptr, 0, nullptr, nullptr, nullptr, nullptr);
  CHECK(pairs);
  std::vector<int64_t> offsets(pairs + 1);
  const int rc = get(offsets.data(), 0, nullptr, nullptr, nullptr, nullptr);  // offsets only
  if (rc != B200REG_ESTATE) CHECK(rc);
  const size_t m = (size_t)offsets[pairs];
  std::vector<int32_t> corr(2 * m), inlier(m);
  std::vector<float> sxyz(3 * m), dxyz(3 * m);
  CHECK(get(offsets.data(), m, corr.data(), inlier.data(), sxyz.data(), dxyz.data()));
  std::ofstream o(path, std::ios::binary);
  o.write(reinterpret_cast<const char*>(corr.data()), (std::streamsize)(corr.size() * 4));
  o.write(reinterpret_cast<const char*>(inlier.data()), (std::streamsize)(inlier.size() * 4));
  o.write(reinterpret_cast<const char*>(sxyz.data()), (std::streamsize)(sxyz.size() * 4));
  o.write(reinterpret_cast<const char*>(dxyz.data()), (std::streamsize)(dxyz.size() * 4));
  std::printf("[");
  for (int i = 0; i <= pairs; i++) std::printf("%s%lld", i ? ", " : "", (long long)offsets[i]);
  std::printf("]");
}

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
  // the synchronous call
  CHECK(b200reg_ctx_set_quatro_matches(ctx, 1));
  std::vector<b200reg_result> res(count);
  std::vector<b200reg_quatro_info> qi(count);
  CHECK(b200reg_perform_loop_closure(ctx, kf, count, queries.data(), closest.data(), &cfg, res.data(), qi.data()));
  std::printf("{\"closest\": [");
  for (int i = 0; i < count; i++) std::printf("%s%d", i ? ", " : "", closest[i]);
  std::printf("], \"clique_size\": [");
  for (int i = 0; i < count; i++) std::printf("%s%d", i ? ", " : "", qi[i].clique_size);
  std::printf("], \"ctx\": ");
  dump([&](int64_t* o, size_t cap, int32_t* c, int32_t* in, float* s, float* d) { return b200reg_quatro_matches(ctx, o, cap, c, in, s, d); },
       std::string(argv[2]) + "_ctx.bin");
  // the same attempt as a driver job; the candidate search runs inside it
  b200reg_batch* batch = nullptr;
  CHECK(b200reg_batch_create(0, 2, &batch));
  CHECK(b200reg_batch_set_quatro_matches(batch, 1));
  std::vector<b200reg_result> jres(count);
  std::vector<b200reg_quatro_info> jqi(count);
  const int64_t t = b200reg_batch_submit_perform_loop_closure(batch, kf, count, queries.data(), nullptr, &cfg, jres.data(), jqi.data());
  CHECK((int)(t < 0 ? t : 0));
  CHECK(b200reg_batch_wait(batch, t, nullptr));
  std::printf(", \"job\": ");
  dump([&](int64_t* o, size_t cap, int32_t* c, int32_t* in, float* s, float* d) {
         return b200reg_batch_quatro_matches(batch, t, o, cap, c, in, s, d);
       },
       std::string(argv[2]) + "_job.bin");
  const int released = b200reg_batch_release(batch, t);
  const int after = b200reg_batch_quatro_matches(batch, t, nullptr, 0, nullptr, nullptr, nullptr, nullptr);
  std::printf(", \"released\": %d, \"after_release\": %d}\n", released, after);
  CHECK(b200reg_batch_destroy(batch));
  CHECK(b200reg_keyframes_destroy(ctx, kf));
  CHECK(b200reg_ctx_destroy(ctx));
  return 0;
}
