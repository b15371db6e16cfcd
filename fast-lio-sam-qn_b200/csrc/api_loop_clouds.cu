// api_loop_clouds.cu -- the clouds loopTimerFunc publishes after each loop attempt (fast_lio_sam_qn.cpp:245-248), returned by
// the batched loop-closure calls (b200reg_loop_clouds): the capture those calls run.
#include <algorithm>
#include <cstring>

#include "api.cuh"

namespace {
constexpr int KIND_SOURCE = 0, KIND_TARGET = 1, KIND_COARSE = 2, KIND_FINAL = 3;  // slot = log2 of the B200REG_CLOUD_* bit
}  // namespace

namespace b200 {

int LoopCapture::clouds(int count, b200reg_cloud* const* src, b200reg_cloud* const* dst, bool src_tgt_rows, bool coarse_rows) {
  if (!mask_) return B200REG_OK;
  src_.assign(src, src + count);
  dst_.assign(dst, dst + count);
  src_tgt_rows_ = src_tgt_rows;
  // room for every row that can be present: COARSE and FINAL of a pair exist only if its stages run, unknown until they have
  size_t points[4] = {0, 0, 0, 0};
  for (int k = 0; k < count; k++) {
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
  const int count = (int)src_.size();
  CsrRecord* lc = &c_->records.rec[Records::CLOUD];  // one record per kind
  std::vector<CaptureRow> rows;
  int max_n = 0;
  for (int s = 0; s < 4; s++) {
    if (!(mask_ >> s & 1)) continue;
    std::vector<int64_t>& offsets = lc[s].offsets;
    offsets.assign(count + 1, 0);
    for (int k = 0; k < count; k++) {
      const bool coarse_valid = qi && qi[k].valid;
      const bool fine_ran = !qi || qi[k].valid;  // icpAlignment runs after a valid coarse stage only (loop_closure.cpp:145-156)
      const bool present = s == KIND_SOURCE || s == KIND_TARGET ? src_tgt_rows_ : s == KIND_COARSE ? coarse_valid : fine_ran;
      offsets[k + 1] = offsets[k];
      if (!present) continue;
      const b200reg_cloud* cl = s == KIND_TARGET ? dst_[k] : src_[k];
      CaptureRow r;
      memset(&r, 0, sizeof(r));
      r.pts = cl->dev.pts;
      r.inten = cl->inten;
      r.out = slab_[s] + offsets[k];
      r.n = cl->dev.n;
      // COARSE = transformPcd(src, T_quatro); FINAL = align()'s output cloud of the fine source: COARSE in Quatro mode
      r.coarse = s == KIND_COARSE || (s == KIND_FINAL && qi);
      r.fine = s == KIND_FINAL;
      if (r.coarse) memcpy(r.Tq, qi[k].T, sizeof(r.Tq));
      if (r.fine) memcpy(r.Tf, fine_tf16 + 16 * (size_t)k, sizeof(r.Tf));
      rows.push_back(r);
      offsets[k + 1] += r.n;
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
    if (!(mask_ >> s & 1)) continue;
    lc[s].rows.resize(sizeof(float4) * lc[s].offsets[count]);
    if (!lc[s].rows.empty()) CU(cudaMemcpyAsync(lc[s].rows.data(), slab_[s], lc[s].rows.size(), cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  return B200REG_OK;
}

}  // namespace b200
