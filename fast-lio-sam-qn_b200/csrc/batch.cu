// batch.cu -- the batch driver of the C ABI (include/b200reg.h, "b200reg_batch_*"): `depth` engine contexts, each on its
// own host thread with its own CUDA streams and memory pool, take alternate jobs.  While one context waits for a PCIe
// upload or polls its LM loop, the kernels of the others keep the SMs busy -- the batch-level concurrency SURVEY.md §8(d)
// names as the lever for the HBM fraction.  Host code only; everything it calls is the public C ABI, except the jobs over
// the keyframe store, which go through the job interface of api_keyframes.cu (api.cuh), and the records of a capturing
// job (loop clouds, LM trace, Quatro matches, residuals), which it moves out of the worker's context and reads with the
// context getters' copy-out (api.cuh).
//
// Reference context: the reference registers ONE pair per 2 Hz timer tick, serially, on one thread
// (fast_lio_sam_qn/src/fast_lio_sam_qn.cpp:203-219, LoopClosure is not re-entrant, :81).
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <iterator>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "api.cuh"

namespace {

struct Job {
  int kind = 0;  // 0 icpAlignment, 1 coarseToFineAlignment, 2 performLoopClosure over a keyframe store
  int count = 0;
  std::vector<const float*> src, tgt;
  std::vector<size_t> src_n, tgt_n;
  size_t stride = 0;
  int on_device = 0;
  b200reg_gicp_params gp;
  b200reg_quatro_params qp;
  std::shared_ptr<KfJob> kfjob;  // kind 2: its arguments and the store's state at submit
  b200reg_result* out = nullptr;
  b200reg_quatro_info* qout = nullptr;
  // the driver's capture settings at submit (b200reg_batch_set_loop_clouds / _set_lm_trace / _set_quatro_matches /
  // _set_residuals), and the records the job left, moved out of its worker's context when it ended: they outlive the wait,
  // until b200reg_batch_release or b200reg_batch_destroy
  Capture capture;
  std::shared_ptr<Records> captured;
  // completion
  int status = 0;
  std::string error;
  bool done = false;
  std::chrono::steady_clock::time_point t_submit, t_done;
};

struct Worker {
  b200reg_ctx* ctx = nullptr;
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<std::shared_ptr<Job>> q;
  bool stop = false;
};

}  // namespace

struct b200reg_batch {
  int device = 0;
  std::vector<std::unique_ptr<Worker>> workers;
  std::mutex mu;  // tickets / completion
  std::condition_variable cv_done;
  std::map<int64_t, std::shared_ptr<Job>> jobs;  // submitted, not waited for yet
  int64_t next_ticket = 0;
  size_t rr = 0;
  // capture: the settings the next submit copies; the settings of every ticket (an entry where they changed, so a driver
  // that never captures keeps none); the outputs of the waited-for jobs that captured (null: the job failed), until released
  Capture capture;
  std::map<int64_t, Capture> capture_from;
  std::map<int64_t, std::shared_ptr<Records>> kept;
};

static thread_local std::string g_batch_err;

static void run_worker(b200reg_batch* b, Worker* w) {
  for (;;) {
    std::shared_ptr<Job> j;
    {
      std::unique_lock<std::mutex> lk(w->mu);
      w->cv.wait(lk, [&] { return w->stop || !w->q.empty(); });
      if (w->q.empty()) return;  // stop requested and nothing left
      j = w->q.front();
      w->q.pop_front();
    }
    b200reg_ctx* c = w->ctx;
    c->capture = j->capture;  // for this job only
    int rc;
    if (j->kind == 0)
      rc = b200reg_icp_alignment(c, j->count, j->src.data(), j->src_n.data(), j->tgt.data(), j->tgt_n.data(), j->stride, j->on_device,
                                 &j->gp, j->out);
    else if (j->kind == 1)
      rc = b200reg_loop_closure(c, j->count, j->src.data(), j->src_n.data(), j->tgt.data(), j->tgt_n.data(), j->stride, j->on_device,
                                &j->qp, &j->gp, j->out, j->qout);
    else
      rc = kf_job_run(c, j->kfjob.get(), j->out, j->qout);
    j->kfjob.reset();  // the store no longer counts the job as in flight: a wait that returns sees it finished
    if (j->capture.on()) {  // the job takes the stored records without a copy; nothing carries over to the worker's next job
      auto rec = std::make_shared<Records>();
      std::swap(*rec, c->records);
      if (!rc) j->captured = std::move(rec);
    }
    {
      std::lock_guard<std::mutex> lk(b->mu);
      j->status = rc;
      if (rc) j->error = b200reg_last_error();  // this thread's message
      j->t_done = std::chrono::steady_clock::now();
      j->done = true;
    }
    b->cv_done.notify_all();
  }
}

extern "C" {

int b200reg_batch_create(int device, int depth, b200reg_batch** out) {
  if (!out || depth < 1 || depth > 16) return B200REG_EINVAL;
  std::unique_ptr<b200reg_batch> b(new b200reg_batch);
  b->device = device;
  for (int i = 0; i < depth; i++) {
    std::unique_ptr<Worker> w(new Worker);
    const int rc = b200reg_ctx_create(device, &w->ctx);
    if (rc) {  // no GPU: fail loudly, nothing to fall back to
      for (auto& x : b->workers) b200reg_ctx_destroy(x->ctx);
      return rc;
    }
    b->workers.push_back(std::move(w));
  }
  for (auto& w : b->workers) w->th = std::thread(run_worker, b.get(), w.get());
  *out = b.release();
  return B200REG_OK;
}

int b200reg_batch_destroy(b200reg_batch* b) {
  if (!b) return B200REG_OK;
  for (auto& w : b->workers) {
    {
      std::lock_guard<std::mutex> lk(w->mu);
      w->stop = true;
    }
    w->cv.notify_all();
  }
  for (auto& w : b->workers)
    if (w->th.joinable()) w->th.join();
  for (auto& w : b->workers) b200reg_ctx_destroy(w->ctx);
  delete b;
  return B200REG_OK;
}

static int64_t submit(b200reg_batch* b, std::shared_ptr<Job> j) {
  j->t_submit = std::chrono::steady_clock::now();
  int64_t ticket;
  Worker* w;
  j->capture = b->capture;
  {
    std::lock_guard<std::mutex> lk(b->mu);
    ticket = b->next_ticket++;
    const Capture prev = b->capture_from.empty() ? Capture() : b->capture_from.rbegin()->second;
    if (b->capture != prev) b->capture_from[ticket] = b->capture;
    b->jobs[ticket] = j;
    w = b->workers[b->rr].get();
    b->rr = (b->rr + 1) % b->workers.size();
  }
  {
    std::lock_guard<std::mutex> lk(w->mu);
    w->q.push_back(j);
  }
  w->cv.notify_one();
  return ticket;
}

static std::shared_ptr<Job> make_job(int kind, int count, const float* const* src_xyz, const size_t* src_n, const float* const* tgt_xyz,
                                     const size_t* tgt_n, size_t stride_bytes, int on_device) {
  std::shared_ptr<Job> j(new Job);
  j->kind = kind;
  j->count = count;
  j->src.assign(src_xyz, src_xyz + count);
  j->tgt.assign(tgt_xyz, tgt_xyz + count);
  j->src_n.assign(src_n, src_n + count);
  j->tgt_n.assign(tgt_n, tgt_n + count);
  j->stride = stride_bytes;
  j->on_device = on_device;
  return j;
}

int64_t b200reg_batch_submit_icp(b200reg_batch* b, int count, const float* const* src_xyz, const size_t* src_n, const float* const* tgt_xyz,
                                 const size_t* tgt_n, size_t stride_bytes, int on_device, const b200reg_gicp_params* params,
                                 b200reg_result* out) {
  if (!b || count <= 0 || !src_xyz || !src_n || !tgt_xyz || !tgt_n || !params || !out) return B200REG_EINVAL;
  auto j = make_job(0, count, src_xyz, src_n, tgt_xyz, tgt_n, stride_bytes, on_device);
  j->gp = *params;
  j->out = out;
  return submit(b, j);
}

int64_t b200reg_batch_submit_loop_closure(b200reg_batch* b, int count, const float* const* src_xyz, const size_t* src_n,
                                          const float* const* tgt_xyz, const size_t* tgt_n, size_t stride_bytes, int on_device,
                                          const b200reg_quatro_params* qparams, const b200reg_gicp_params* gparams, b200reg_result* out,
                                          b200reg_quatro_info* quatro_out) {
  if (!b || count <= 0 || !src_xyz || !src_n || !tgt_xyz || !tgt_n || !qparams || !gparams || !out) return B200REG_EINVAL;
  auto j = make_job(1, count, src_xyz, src_n, tgt_xyz, tgt_n, stride_bytes, on_device);
  j->gp = *gparams;
  j->qp = *qparams;
  j->out = out;
  j->qout = quatro_out;
  return submit(b, j);
}

int64_t b200reg_batch_submit_perform_loop_closure(b200reg_batch* b, b200reg_keyframes* kf, int count, const int32_t* query_idx,
                                                  const int32_t* closest_idx, const b200reg_loop_config* cfg, b200reg_result* out,
                                                  b200reg_quatro_info* quatro_out) {
  if (!b || !out) return fail(B200REG_EINVAL, "bad argument");
  std::shared_ptr<Job> j(new Job);
  j->kind = 2;
  j->count = count;
  j->out = out;
  j->qout = quatro_out;
  const int rc = kf_job_create(kf, b->device, count, query_idx, closest_idx, cfg, &j->kfjob);
  if (rc) return rc;
  return submit(b, j);
}

int b200reg_batch_wait(b200reg_batch* b, int64_t ticket, double* latency_ms) {
  if (!b) return B200REG_EINVAL;
  std::shared_ptr<Job> j;
  {
    std::unique_lock<std::mutex> lk(b->mu);
    auto it = b->jobs.find(ticket);
    if (it == b->jobs.end()) return B200REG_EINVAL;  // unknown or already waited for
    j = it->second;
    b->cv_done.wait(lk, [&] { return j->done; });
    b->jobs.erase(it);
    if (j->capture.on()) b->kept[ticket] = std::move(j->captured);
  }
  if (latency_ms) *latency_ms = std::chrono::duration<double, std::milli>(j->t_done - j->t_submit).count();
  if (j->status) b200reg_set_last_error(j->error.c_str());
  return j->status;
}

int b200reg_batch_wait_all(b200reg_batch* b) {
  if (!b) return B200REG_EINVAL;
  int first = B200REG_OK;
  for (;;) {
    int64_t t;
    {
      std::lock_guard<std::mutex> lk(b->mu);
      if (b->jobs.empty()) break;
      t = b->jobs.begin()->first;
    }
    const int rc = b200reg_batch_wait(b, t, nullptr);
    if (rc && !first) first = rc;
  }
  return first;
}

int b200reg_batch_set_loop_clouds(b200reg_batch* b, int mask) {
  if (!b) return fail(B200REG_EINVAL, "batch is NULL");
  if (mask & ~(B200REG_CLOUD_SOURCE | B200REG_CLOUD_TARGET | B200REG_CLOUD_COARSE | B200REG_CLOUD_FINAL))
    return fail(B200REG_EINVAL, "mask: an OR of B200REG_CLOUD_SOURCE, _TARGET, _COARSE, _FINAL");
  b->capture.cloud_mask = mask;
  return B200REG_OK;
}

int b200reg_batch_set_lm_trace(b200reg_batch* b, int enable) {
  if (!b) return fail(B200REG_EINVAL, "batch is NULL");
  b->capture.lm_trace = enable != 0;
  return B200REG_OK;
}

int b200reg_batch_set_quatro_matches(b200reg_batch* b, int enable) {
  if (!b) return fail(B200REG_EINVAL, "batch is NULL");
  b->capture.quatro_matches = enable != 0;
  return B200REG_OK;
}

int b200reg_batch_set_residuals(b200reg_batch* b, int enable) {
  if (!b) return fail(B200REG_EINVAL, "batch is NULL");
  b->capture.residuals = enable != 0;
  return B200REG_OK;
}

}  // extern "C"

// What the getters say of a job without record r: the start of the message, and the end for a job that did not record it
// because of its settings at submit
struct RecordText {
  const char* missing;
  const char* off;
};
static const RecordText kRecordText[Records::N] = {
    {"no LM trace: ", " was not traced (b200reg_batch_set_lm_trace at its submit)"},
    {"no residuals: ", " did not record them (b200reg_batch_set_residuals at its submit)"},
    {"no Quatro matches: ", " did not record them (b200reg_batch_set_quatro_matches at its submit, or a job without a Quatro stage)"},
    {"no such loop clouds: ", " did not capture this kind (b200reg_batch_set_loop_clouds at its submit)"},
    {"no such loop clouds: ", " did not capture this kind (b200reg_batch_set_loop_clouds at its submit)"},
    {"no such loop clouds: ", " did not capture this kind (b200reg_batch_set_loop_clouds at its submit)"},
    {"no such loop clouds: ", " did not capture this kind (b200reg_batch_set_loop_clouds at its submit)"},
};

// The getters of a job's record r: the ticket rules, then record_copy over the records the job left (the pointer keeps them
// alive while they are copied out, outside the lock), with the message that says why record r is missing.  r < 0 (a bad
// loop-cloud kind) is refused by record_copy, after the ticket.
static int batch_record(b200reg_batch* b, int64_t ticket, int r, int64_t* offsets_out, size_t capacity,
                        std::initializer_list<void*> cols) {
  if (!b) return fail(B200REG_EINVAL, "batch is NULL");
  std::shared_ptr<Records> rec;
  std::string none;
  {
    std::lock_guard<std::mutex> lk(b->mu);
    if (ticket < 0 || ticket >= b->next_ticket) return fail(B200REG_EINVAL, "ticket " + std::to_string(ticket) + " was never handed out");
    if (r >= 0) {
      const std::string missing = kRecordText[r].missing + std::string("batch job ") + std::to_string(ticket);
      const auto k = b->kept.find(ticket);
      if (b->jobs.count(ticket)) {
        none = missing + " has not been waited for yet (b200reg_batch_wait)";
      } else if (k != b->kept.end()) {
        rec = k->second;
        none = missing + (rec ? kRecordText[r].off : " failed");
      } else {
        const auto s = b->capture_from.upper_bound(ticket);  // the settings the job copied at its submit
        const Capture cap = s == b->capture_from.begin() ? Capture() : std::prev(s)->second;
        none = missing + (cap.wants(r) ? " was released (b200reg_batch_release)" : kRecordText[r].off);
      }
    }
  }
  return record_copy(rec.get(), r, none, offsets_out, capacity, cols);
}

extern "C" {

int b200reg_batch_loop_clouds(b200reg_batch* b, int64_t ticket, int kind, int64_t* offsets_out, size_t capacity, float* xyzi_out) {
  return batch_record(b, ticket, cloud_record(kind), offsets_out, capacity, {xyzi_out});
}

int b200reg_batch_lm_trace(b200reg_batch* b, int64_t ticket, int64_t* offsets_out, size_t capacity, b200reg_lm_trial* trials_out) {
  return batch_record(b, ticket, Records::TRACE, offsets_out, capacity, {trials_out});
}

int b200reg_batch_quatro_matches(b200reg_batch* b, int64_t ticket, int64_t* offsets_out, size_t capacity, int32_t* corr_out,
                                 int32_t* inlier_out, float* src_xyz_out, float* dst_xyz_out) {
  return batch_record(b, ticket, Records::MATCHES, offsets_out, capacity, {corr_out, inlier_out, src_xyz_out, dst_xyz_out});
}

int b200reg_batch_residuals(b200reg_batch* b, int64_t ticket, int64_t* offsets_out, size_t capacity, int32_t* nn_out, float* d2_out) {
  return batch_record(b, ticket, Records::RESIDUALS, offsets_out, capacity, {nn_out, d2_out});
}

int b200reg_batch_release(b200reg_batch* b, int64_t ticket) {
  if (!b) return fail(B200REG_EINVAL, "batch is NULL");
  std::shared_ptr<Records> drop;  // freed after the lock is released
  std::lock_guard<std::mutex> lk(b->mu);
  if (ticket < 0 || ticket >= b->next_ticket) return fail(B200REG_EINVAL, "ticket " + std::to_string(ticket) + " was never handed out");
  if (b->jobs.count(ticket)) return fail(B200REG_ESTATE, "batch job " + std::to_string(ticket) + " has not been waited for yet (b200reg_batch_wait)");
  const auto k = b->kept.find(ticket);
  if (k != b->kept.end()) {
    drop = std::move(k->second);
    b->kept.erase(k);
  }
  return B200REG_OK;
}

int64_t b200reg_batch_launch_count(const b200reg_batch* b) {
  if (!b) return 0;
  int64_t n = 0;
  for (auto& w : b->workers) n += b200reg_ctx_launch_count(w->ctx);
  return n;
}

int b200reg_batch_depth(const b200reg_batch* b) { return b ? (int)b->workers.size() : 0; }

}  // extern "C"
