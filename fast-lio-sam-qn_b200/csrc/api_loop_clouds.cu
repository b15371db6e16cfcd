// api_loop_clouds.cu -- the clouds loopTimerFunc publishes after each loop attempt (fast_lio_sam_qn.cpp:245-248), returned by
// the batched loop-closure calls: b200reg_ctx_set_loop_clouds, b200reg_loop_clouds and the capture those calls run.
#include <algorithm>
#include <cstring>

#include "api.cuh"

namespace {
constexpr int KIND_SOURCE = 0, KIND_TARGET = 1, KIND_COARSE = 2, KIND_FINAL = 3;  // slot = log2 of the B200REG_CLOUD_* bit
}  // namespace

namespace b200 {

LoopCapture::LoopCapture(b200reg_ctx* c, int count) : c_(c), count_(count), mask_(c->loop_clouds.mask), scratch_(c) {
  c->loop_clouds.stored = 0;
}

int LoopCapture::clouds(const std::vector<int>& where, b200reg_cloud* const* src, b200reg_cloud* const* dst, bool src_tgt_rows,
                        bool coarse_rows) {
  if (!mask_) return B200REG_OK;
  const int m = where.empty() ? count_ : (int)where.size();
  where_.resize(m);
  for (int k = 0; k < m; k++) where_[k] = where.empty() ? k : where[k];
  src_.assign(src, src + m);
  dst_.assign(dst, dst + m);
  src_tgt_rows_ = src_tgt_rows;
  // room for every row that can be present: COARSE and FINAL of a pair exist only if its stages run, unknown until they have
  size_t points[4] = {0, 0, 0, 0};
  for (int k = 0; k < m; k++) {
    if (src_tgt_rows) points[KIND_SOURCE] += src[k]->dev.n;
    if (src_tgt_rows) points[KIND_TARGET] += dst[k]->dev.n;
    if (coarse_rows) points[KIND_COARSE] += src[k]->dev.n;
    points[KIND_FINAL] += src[k]->dev.n;
  }
  Layout l;
  size_t off[4];
  for (int s = 0; s < 4; s++) off[s] = l.take((mask_ >> s & 1) ? points[s] * sizeof(float4) : 0);
  char* slab = nullptr;
  const cudaError_t e = scratch_.alloc((void**)&slab, l.size);
  if (e != cudaSuccess)
    return fail(B200REG_ECUDA, "loop clouds: cannot allocate " + std::to_string(l.size) + " bytes: " + cudaGetErrorString(e));
  for (int s = 0; s < 4; s++) slab_[s] = (float4*)(slab + off[s]);
  return B200REG_OK;
}

int LoopCapture::finish(const b200reg_quatro_info* qi, const float* fine_tf16) {
  if (!mask_) return B200REG_OK;
  auto& lc = c_->loop_clouds;
  std::vector<int64_t> offsets[4];
  std::vector<int> solved(count_, -1);  // caller pair -> stage pair
  for (size_t k = 0; k < where_.size(); k++) solved[where_[k]] = (int)k;
  std::vector<CaptureRow> rows;
  int max_n = 0;
  for (int s = 0; s < 4; s++) {
    offsets[s].assign(count_ + 1, 0);
    if (!(mask_ >> s & 1)) continue;
    for (int i = 0; i < count_; i++) {
      const int k = solved[i];
      bool present = false;
      if (k >= 0) {
        const bool coarse_valid = qi && qi[k].valid;
        const bool fine_ran = !qi || qi[k].valid;  // icpAlignment runs after a valid coarse stage only (loop_closure.cpp:145-156)
        present = s == KIND_SOURCE || s == KIND_TARGET ? src_tgt_rows_ : s == KIND_COARSE ? coarse_valid : fine_ran;
      }
      offsets[s][i + 1] = offsets[s][i];
      if (!present) continue;
      const b200reg_cloud* cl = s == KIND_TARGET ? dst_[k] : src_[k];
      CaptureRow r;
      memset(&r, 0, sizeof(r));
      r.pts = cl->dev.pts;
      r.inten = cl->inten;
      r.out = slab_[s] + offsets[s][i];
      r.n = cl->dev.n;
      // COARSE = transformPcd(src, T_quatro); FINAL = align()'s output cloud of the fine source: COARSE in Quatro mode
      r.coarse = s == KIND_COARSE || (s == KIND_FINAL && qi);
      r.fine = s == KIND_FINAL;
      if (r.coarse) memcpy(r.Tq, qi[k].T, sizeof(r.Tq));
      if (r.fine) memcpy(r.Tf, fine_tf16 + 16 * (size_t)k, sizeof(r.Tf));
      rows.push_back(r);
      offsets[s][i + 1] += r.n;
      max_n = std::max(max_n, r.n);
    }
  }
  cudaStream_t st = c_->stream;
  if (!rows.empty()) {
    CaptureRow* d_rows = nullptr;
    CU(scratch_.upload(&d_rows, rows.data(), sizeof(CaptureRow) * rows.size()));
    {
      ProfScope ps(c_, CLS_MISC);
      launch_capture_rows(d_rows, (int)rows.size(), max_n, st);
      c_->launches++;
      for (const CaptureRow& r : rows) c_->prof_bytes[CLS_MISC] += 36.0 * r.n;  // 16 in + 4 intensity + 16 out
    }
    CU(cudaGetLastError());
  }
  for (int s = 0; s < 4; s++) {
    lc.pts[s].resize((size_t)offsets[s][count_]);
    if (!lc.pts[s].empty())
      CU(cudaMemcpyAsync(lc.pts[s].data(), slab_[s], lc.pts[s].size() * sizeof(float4), cudaMemcpyDeviceToHost, st));
    lc.offsets[s].swap(offsets[s]);
  }
  CU(cudaStreamSynchronize(st));
  lc.stored = mask_;
  return B200REG_OK;
}

int loop_clouds_copy(const b200reg_ctx::LoopClouds* lc, int kind, int64_t* offsets_out, size_t capacity, float* xyzi_out,
                     const std::string& none) {
  int s = -1;
  for (int b = 0; b < 4; b++)
    if (kind == 1 << b) s = b;
  if (s < 0) return fail(B200REG_EINVAL, "kind: one of B200REG_CLOUD_SOURCE, _TARGET, _COARSE, _FINAL");
  if (!lc || !(lc->stored & kind)) return fail(B200REG_ESTATE, none);
  const int pairs = (int)lc->offsets[s].size() - 1;
  if (!offsets_out) return pairs;
  memcpy(offsets_out, lc->offsets[s].data(), sizeof(int64_t) * lc->offsets[s].size());
  if (lc->pts[s].size() > capacity)
    return fail(B200REG_ESTATE, "loop clouds hold " + std::to_string(lc->pts[s].size()) + " points, capacity " + std::to_string(capacity));
  if (xyzi_out && !lc->pts[s].empty()) memcpy(xyzi_out, lc->pts[s].data(), sizeof(float4) * lc->pts[s].size());
  return B200REG_OK;
}

}  // namespace b200

extern "C" {

int b200reg_ctx_set_loop_clouds(b200reg_ctx* c, int mask) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  if (mask & ~(B200REG_CLOUD_SOURCE | B200REG_CLOUD_TARGET | B200REG_CLOUD_COARSE | B200REG_CLOUD_FINAL))
    return fail(B200REG_EINVAL, "mask: an OR of B200REG_CLOUD_SOURCE, _TARGET, _COARSE, _FINAL");
  c->loop_clouds.mask = mask;
  return B200REG_OK;
}

int b200reg_loop_clouds(b200reg_ctx* c, int kind, int64_t* offsets_out, size_t capacity, float* xyzi_out) {
  if (!c) return fail(B200REG_EINVAL, "ctx is NULL");
  return loop_clouds_copy(&c->loop_clouds, kind, offsets_out, capacity, xyzi_out,
                          "no such loop clouds: the context's last loop-closure call did not capture this kind (b200reg_ctx_set_loop_clouds)");
}

}  // extern "C"
