// api_quatro.cu -- the C ABI of the Quatro path: FPFH descriptors, b200reg_quatro_align, coarse-to-fine and
// b200reg_loop_closure.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "api.cuh"

namespace b200 {
int coarse_to_fine_on_clouds(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                             const b200reg_quatro_params* qp, const b200reg_gicp_params* gp, b200reg_result* out,
                             b200reg_quatro_info* quatro_out, float* fine_tf16) {
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<b200reg_quatro_info> qi(count);
  CloudBag coarse_bag(c);  // the transformed source clouds are released on every exit path
  std::vector<b200reg_cloud*>& coarse = coarse_bag.cl;
  int rc = b200reg_quatro_align(c, count, src, dst, qp, qi.data(), nullptr);
  if (rc) return rc;
  if (quatro_out) memcpy(quatro_out, qi.data(), sizeof(b200reg_quatro_info) * count);
  // pairs whose coarse stage is valid go on to icpAlignment(coarse_aligned_, dst) (loop_closure.cpp:145-156)
  std::vector<int> vidx;
  for (int i = 0; i < count; i++) {
    out[i] = default_result();
    for (int k = 0; k < 16; k++) {
      out[i].T[k] = qi[i].T[k];
      out[i].Tf[k] = (float)qi[i].T[k];
      out[i].pose_between[k] = qi[i].T[k];  // an invalid coarse stage returns what quatro::align returned (loop_closure.cpp:144-148)
    }
    if (qi[i].valid) vidx.push_back(i);
  }
  if (!vidx.empty()) {
    const int nv = (int)vidx.size();
    std::vector<CloudDev> sdesc(nv);
    std::vector<double> Ts(16 * (size_t)nv);
    std::vector<float4*> outs(nv);
    std::vector<const float*> cptr(nv);
    std::vector<size_t> cn(nv);
    int max_n = 0;
    for (int k = 0; k < nv; k++) {
      const int i = vidx[k];
      sdesc[k] = src[i]->dev;
      memcpy(&Ts[16 * (size_t)k], qi[i].T, 128);
      float4* raw = nullptr;
      CU(scratch.alloc((void**)&raw, (size_t)sdesc[k].n * 16));
      outs[k] = raw;
      cptr[k] = (const float*)raw;
      cn[k] = sdesc[k].n;
      max_n = std::max(max_n, sdesc[k].n);
    }
    CloudDev* d_desc = nullptr;
    double* d_T = nullptr;
    float4** d_outs = nullptr;
    CU(scratch.upload(&d_desc, sdesc.data(), sizeof(CloudDev) * nv));
    CU(scratch.upload(&d_T, Ts.data(), 128 * (size_t)nv));
    CU(scratch.upload(&d_outs, outs.data(), sizeof(float4*) * nv));
    launch_transform_raw(d_desc, d_T, nv, max_n, d_outs, s);
    c->launches++;
    coarse.assign(nv, nullptr);
    rc = b200reg_clouds_create(c, nv, cptr.data(), cn.data(), 16, 1, coarse.data());
    std::vector<b200reg_cloud*> tg(nv);
    for (int k = 0; k < nv; k++) tg[k] = dst[vidx[k]];
    std::vector<b200reg_result> gres(nv);
    if (!rc) rc = b200reg_gicp_align(c, nv, coarse.data(), tg.data(), nullptr, gp, gres.data());
    if (rc) return rc;
    for (int k = 0; k < nv; k++) {
      const int i = vidx[k];
      if (fine_tf16) memcpy(&fine_tf16[16 * (size_t)i], gres[k].Tf, sizeof(gres[k].Tf));
      b200reg_result r = gres[k];
      // reg_output.pose_between_eig_ = fine (float -> double) * quatro_tf_  (loop_closure.cpp:156)
      double F[16], Q[16];
      for (int a = 0; a < 16; a++) {
        F[a] = (double)gres[k].Tf[a];
        Q[a] = qi[i].T[a];
      }
      for (int a = 0; a < 4; a++)
        for (int b = 0; b < 4; b++) {
          double v = 0, pb = 0;
          for (int m = 0; m < 4; m++) {
            v += F[4 * a + m] * Q[4 * m + b];
            pb += gres[k].pose_between[4 * a + m] * Q[4 * m + b];  // fine_output.pose_between_eig_ is Identity when the fine
          }                                                        // stage is not valid: the reference then keeps I * Q
          r.T[4 * a + b] = v;           // telemetry: the solver's own final transform composed with the coarse stage
          r.Tf[4 * a + b] = (float)v;
          r.pose_between[4 * a + b] = pb;
        }
      out[i] = r;
    }
  }
  lm_trace_remap(c, count, vidx);
  return B200REG_OK;
}

static int pow2_at_least(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// The one sizing of the global-memory solver workspace (BigSolveWs) for up to `cap` correspondences, cap a multiple of
// 1024.  nsrc > 0 adds k_adv_select_wide's scatter array for a source cloud of nsrc points.
struct BigWsLayout {
  int cap, words, p2;
  size_t o_S = 0, o_D = 0, o_adj = 0, o_radj = 0, o_int = 0, o_skey = 0, o_w = 0, o_res = 0, o_hval = 0, o_hidx = 0, o_best = 0,
         o_slot = 0;
  BigWsLayout(Layout& l, int cap_, int nsrc) : cap(cap_), words(cap_ / 32), p2(pow2_at_least(cap_)) {
    if (cap == 0) return;  // no workspace (optimizedMatching)
    o_S = l.take((size_t)cap * 24);
    o_D = l.take((size_t)cap * 24);
    o_adj = l.take((size_t)cap * words * 4);
    o_radj = l.take((size_t)cap * words * 4);
    o_int = l.take((size_t)cap * 4 * 9);
    o_skey = l.take((size_t)p2 * 8);
    o_w = l.take((size_t)cap * 8);
    o_res = l.take((size_t)cap * 8);
    o_hval = l.take((size_t)p2 * 16);
    o_hidx = l.take((size_t)p2 * 8);
    o_best = l.take(8);
    o_slot = nsrc > 0 ? l.take((size_t)nsrc * 4) : 0;
  }
  BigSolveWs bind(char* slab) const {
    BigSolveWs w;
    w.cap = cap;
    w.words = words;
    w.p2 = p2;
    w.S = (double*)(slab + o_S);
    w.D = (double*)(slab + o_D);
    w.adj = (unsigned*)(slab + o_adj);
    w.radj = (unsigned*)(slab + o_radj);
    int* ip = (int*)(slab + o_int);
    w.deg = ip; w.pdeg = ip + cap; w.core = ip + 2 * (size_t)cap; w.alive = ip + 3 * (size_t)cap; w.rank = ip + 4 * (size_t)cap;
    w.order = ip + 5 * (size_t)cap; w.csize = ip + 6 * (size_t)cap; w.clique = ip + 7 * (size_t)cap; w.list = ip + 8 * (size_t)cap;
    w.skey = (unsigned long long*)(slab + o_skey);
    w.w = (double*)(slab + o_w);
    w.res = (double*)(slab + o_res);
    w.hval = (double*)(slab + o_hval);
    w.hidx = (int*)(slab + o_hidx);
    w.best = (unsigned long long*)(slab + o_best);
    w.slot = o_slot ? (int*)(slab + o_slot) : nullptr;
    return w;
  }
};

// squared feature distance gate of the matcher (dis > thr2 is dropped, matcher.cc:422,444).  advancedMatching searches
// without a gate: FLT_MAX makes every finite distance qualify.  A square that overflows, or a NaN threshold, drops nothing
// in the reference either: +inf.
static float match_thr2(double distance_threshold, bool advanced) {
  if (advanced) return 3.402823466e38f;
  const float t2 = (float)distance_threshold * (float)distance_threshold;
  return t2 <= 3.402823466e38f ? t2 : INFINITY;
}

static QuatroParamsDev quatro_params_dev(const b200reg_quatro_params* prm, bool advanced) {
  QuatroParamsDev q;
  q.normal_r2 = (float)(prm->fpfh_normal_radius * prm->fpfh_normal_radius);
  q.fpfh_r2 = (float)(prm->fpfh_radius * prm->fpfh_radius);
  q.thr2 = match_thr2(prm->distance_threshold, advanced);
  q.advanced = advanced ? 1 : 0;
  q.tuple_scale = (float)prm->tuple_scale;
  q.max_corres = prm->max_corres;
  q.noise_bound = prm->noise_bound;
  q.gnc_factor = prm->rot_gnc_factor;
  q.cost_thr = prm->rot_cost_thr;
  q.max_iter = prm->rot_max_iter;
  q.seed = prm->seed;
  return q;
}

// b200reg_quatro_align (corr_fixed: count x 2 x CAP ints, or NULL) and b200reg_quatro_align_ex (offsets_out non-NULL;
// corr_csr: `capacity` pairs, or NULL).  Every pair is matched and, if its set holds at most BIGC correspondences,
// solved in one batched pass.  A larger advancedMatching set is then solved on its own in one workspace shared by all
// such pairs of the call (sized for the largest), one pair after another, so device memory stays bounded by the largest.
// optimizedMatching keeps at most max_corres + 3 <= BIGC: k_teaser_solve solves the sets of at most MAXC in that pass,
// and the larger ones are solved afterwards in one batched pass of the global-memory chain.
static int quatro_align_impl(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst, const b200reg_quatro_params* prm,
                      b200reg_quatro_info* out, int32_t* corr_fixed, int64_t* offsets_out, size_t capacity, int32_t* corr_csr) {
  if (!c || count <= 0 || !src || !dst || !prm || !out) return fail(B200REG_EINVAL, "bad argument");
  if (prm->estimate_scale) return fail(B200REG_EINVAL, "estimate_scale is not supported (the deployment sets it false)");
  const bool advanced = !prm->use_optimized_matching;  // Matcher::advancedMatching (matcher.cc:118-356)
  if (!advanced && (prm->max_corres < 1 || prm->max_corres > OPT_MAX_CORRES)) return fail(B200REG_EINVAL, "max_corres must be in 1..8189");
  // optimizedMatching's out_corr: MAXC pairs, or max_corres + 3 when that is more
  const int opt_cap = advanced ? 0 : std::max(MAXC, prm->max_corres + 3);
  const int corr_stride = advanced ? BIGC : MAXC;  // B200REG_ADV_CORR_CAPACITY / B200REG_CORR_CAPACITY
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  int rc;
  {
    std::vector<b200reg_cloud*> all;
    for (int i = 0; i < count; i++) {
      if (!src[i] || !dst[i]) return fail(B200REG_EINVAL, "NULL cloud");
      all.push_back(src[i]);
      all.push_back(dst[i]);
    }
    if ((rc = b200reg_clouds_fpfh(c, (int)all.size(), all.data(), prm->fpfh_normal_radius, prm->fpfh_radius))) return rc;
  }
  std::vector<MatchDev> pairs(count);
  std::vector<BigSolveWs> big_host;
  big_host.reserve(count);  // addresses stay valid for the async copies below
  int max_ni = 0, max_nj = 0;
  for (int i = 0; i < count; i++) {
    MatchDev& m = pairs[i];
    const bool swapped = dst[i]->dev.n > src[i]->dev.n;  // fi = larger cloud (matcher.cc:364-369)
    m.fi = swapped ? dst[i]->dev : src[i]->dev;
    m.fj = swapped ? src[i]->dev : dst[i]->dev;
    m.swapped = swapped ? 1 : 0;
    const size_t ni = m.fi.n, nj = m.fj.n;
    Layout l;
    const size_t o_nn = l.take(nj * 4), o_dis = l.take(nj * 4), o_fj = l.take(ni * 4), o_rnn = l.take(ni * 4);
    // advancedMatching: the cross-checked set has at most nj members; the solver workspace is sized for the next
    // power of two (>= 1024, <= BIGC)
    int cap = 1024;
    while (advanced && cap < (int)nj && cap < BIGC) cap <<= 1;
    const size_t o_cor = l.take(2 * nj * 4), o_tk = l.take(nj * 4), o_cnt = l.take(8 * 4), o_st = l.take(8 * 8),
                 o_oc = l.take(2 * (size_t)(advanced ? cap : opt_cap) * 4), o_T = l.take(16 * 8);
    const size_t o_big = advanced ? l.take(sizeof(BigSolveWs)) : 0;
    const BigWsLayout wl(l, advanced ? cap : 0, 0);  // empty when !advanced
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    m.nn = (int*)(slab + o_nn);
    m.dis = (float*)(slab + o_dis);
    m.first_j = (int*)(slab + o_fj);
    m.rnn = (int*)(slab + o_rnn);
    m.corres = (int*)(slab + o_cor);
    m.tkey = (unsigned*)(slab + o_tk);
    m.counters = (int*)(slab + o_cnt);
    m.stats = (double*)(slab + o_st);
    m.out_corr = (int*)(slab + o_oc);
    m.T = (double*)(slab + o_T);
    m.big = nullptr;
    if (advanced) {
      m.big = (BigSolveWs*)(slab + o_big);
      big_host.push_back(wl.bind(slab));
      CU(cudaMemcpyAsync(m.big, &big_host.back(), sizeof(BigSolveWs), cudaMemcpyHostToDevice, s));
    }
    max_ni = std::max(max_ni, (int)ni);
    max_nj = std::max(max_nj, (int)nj);
  }
  MatchDev* d_pairs = nullptr;
  CU(scratch.upload(&d_pairs, pairs.data(), sizeof(MatchDev) * count));
  const QuatroParamsDev q = quatro_params_dev(prm, advanced);
  {
    ProfScope ps(c, CLS_MATCH);
    c->launches += launch_quatro_match_solve(d_pairs, count, max_ni, max_nj, q, s);
    for (int i = 0; i < count; i++) c->prof_bytes[CLS_MATCH] += 132.0 * (pairs[i].fi.n + pairs[i].fj.n) + 8.0 * pairs[i].fj.n;  // SURVEY §8(d) Q4
  }
  CU(cudaGetLastError());
  std::vector<int> counters(8 * (size_t)count);
  for (int i = 0; i < count; i++) {
    CU(cudaMemcpyAsync(&counters[8 * i], pairs[i].counters, 32, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(out[i].T, pairs[i].T, 128, cudaMemcpyDeviceToHost, s));
    if (corr_fixed) {
      const size_t have = advanced ? (size_t)big_host[i].cap : (size_t)MAXC;  // what this pair's buffer holds
      CU(cudaMemcpyAsync(&corr_fixed[2 * (size_t)corr_stride * i], pairs[i].out_corr, 2 * have * 4, cudaMemcpyDeviceToHost, s));
    }
  }
  CU(cudaStreamSynchronize(s));
  // counters[6] > 0: k_adv_select found more than BIGC correspondences and left the pair unsolved
  std::vector<int> wide;
  int max_wide = 0, max_src = 0;
  for (int i = 0; i < count; i++)
    if (counters[8 * i + 6] > 0) {
      const int n = counters[8 * i + 6];
      if (corr_fixed) {
        char msg[200];
        snprintf(msg, sizeof msg, "advancedMatching kept %d correspondences for pair %d; corr_out holds %d per pair "
                 "(b200reg_quatro_align_ex returns any number)", n, i, BIGC);
        return fail(B200REG_ESTATE, msg);
      }
      if (n >= BIG_NMAX) {
        char msg[160];
        snprintf(msg, sizeof msg, "advancedMatching kept %d correspondences for pair %d; the solver takes fewer than %d", n, i, BIG_NMAX);
        return fail(B200REG_ESTATE, msg);
      }
      wide.push_back(i);
      max_wide = std::max(max_wide, n);
      max_src = std::max(max_src, pairs[i].swapped ? pairs[i].fj.n : pairs[i].fi.n);
    }
  // optimizedMatching sets beyond MAXC: k_teaser_solve left them unsolved
  std::vector<int> big;
  int max_big = 0;
  for (int i = 0; i < count && !advanced; i++)
    if (counters[8 * i + 2] > MAXC) {
      const int n = counters[8 * i + 2];
      if (corr_fixed) {
        char msg[200];
        snprintf(msg, sizeof msg, "optimizedMatching kept %d correspondences for pair %d; corr_out holds %d per pair "
                 "(b200reg_quatro_align_ex returns any number)", n, i, MAXC);
        return fail(B200REG_ESTATE, msg);
      }
      big.push_back(i);
      max_big = std::max(max_big, n);
    }
  std::vector<int64_t> offsets;
  if (offsets_out) {
    offsets.assign(count + 1, 0);
    for (int i = 0; i < count; i++) offsets[i + 1] = offsets[i] + (counters[8 * i + 6] > 0 ? counters[8 * i + 6] : counters[8 * i + 2]);
    memcpy(offsets_out, offsets.data(), sizeof(int64_t) * (count + 1));
    if (corr_csr && (uint64_t)offsets[count] > capacity) {
      char msg[160];
      snprintf(msg, sizeof msg, "the final correspondences number %lld; corr_out holds %zu", (long long)offsets[count], capacity);
      return fail(B200REG_ESTATE, msg);
    }
    if (corr_csr)
      for (int i = 0; i < count; i++)
        if (counters[8 * i + 6] == 0 && counters[8 * i + 2] > 0)
          CU(cudaMemcpyAsync(corr_csr + 2 * offsets[i], pairs[i].out_corr, (size_t)counters[8 * i + 2] * 8, cudaMemcpyDeviceToHost, s));
  }
  // each optimizedMatching set beyond MAXC gets a workspace for its own size, and all of them are solved in one batched
  // pass; each pair's view reads its own out_corr and writes its own counters and T
  std::vector<MatchDev> big_views(big.size());
  std::vector<BigSolveWs> big_ws(big.size());
  if (!big.empty()) {
    const int nb = (int)big.size();
    Layout l;
    const size_t o_views = l.take(sizeof(MatchDev) * nb), o_ws = l.take(sizeof(BigSolveWs) * nb);
    std::vector<BigWsLayout> wls;
    wls.reserve(nb);
    for (int i : big) wls.emplace_back(l, std::max(1024, pow2_at_least(counters[8 * i + 2])), 0);
    char* slab = nullptr;
    if (scratch.alloc((void**)&slab, l.size) != cudaSuccess) {
      cudaGetLastError();
      char msg[200];
      snprintf(msg, sizeof msg, "optimizedMatching kept up to %d correspondences; solving them needs a workspace of %zu bytes, "
               "which could not be allocated", max_big, l.size);
      return fail(B200REG_ECUDA, msg);
    }
    for (int k = 0; k < nb; k++) {
      big_ws[k] = wls[k].bind(slab);
      big_views[k] = pairs[big[k]];
      big_views[k].big = (BigSolveWs*)(slab + o_ws) + k;
    }
    CU(cudaMemcpyAsync(slab + o_ws, big_ws.data(), sizeof(BigSolveWs) * nb, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(slab + o_views, big_views.data(), sizeof(MatchDev) * nb, cudaMemcpyHostToDevice, s));
    {
      ProfScope ps(c, CLS_MATCH);
      c->launches += launch_big_solve((const MatchDev*)(slab + o_views), nb, max_big, q, s);
    }
    CU(cudaGetLastError());
    for (int i : big) {
      CU(cudaMemcpyAsync(&counters[8 * i], pairs[i].counters, 32, cudaMemcpyDeviceToHost, s));
      CU(cudaMemcpyAsync(out[i].T, pairs[i].T, 128, cudaMemcpyDeviceToHost, s));
    }
  }
  if (!wide.empty()) {
    const int cap = (max_wide + 1023) / 1024 * 1024;
    Layout l;
    const size_t o_big = l.take(sizeof(BigSolveWs)), o_pair = l.take(sizeof(MatchDev)), o_oc = l.take((size_t)cap * 8);
    const BigWsLayout wl(l, cap, max_src);
    char* slab = nullptr;
    if (scratch.alloc((void**)&slab, l.size) != cudaSuccess) {
      cudaGetLastError();
      char msg[200];
      snprintf(msg, sizeof msg, "advancedMatching kept %d correspondences; solving them needs a workspace of %zu bytes, which "
               "could not be allocated", max_wide, l.size);
      return fail(B200REG_ECUDA, msg);
    }
    const BigSolveWs w = wl.bind(slab);
    CU(cudaMemcpyAsync(slab + o_big, &w, sizeof w, cudaMemcpyHostToDevice, s));
    std::vector<MatchDev> views(wide.size());  // each pair with its selection and solve redirected to the shared workspace;
                                               // stream order keeps one pair's use of it from overlapping the next
    ProfScope ps(c, CLS_MATCH);
    for (size_t k = 0; k < wide.size(); k++) {
      const int i = wide[k], n = counters[8 * i + 6];
      views[k] = pairs[i];
      views[k].out_corr = (int*)(slab + o_oc);
      views[k].big = (BigSolveWs*)(slab + o_big);
      CU(cudaMemcpyAsync(slab + o_pair, &views[k], sizeof(MatchDev), cudaMemcpyHostToDevice, s));
      c->launches += launch_adv_wide((const MatchDev*)(slab + o_pair), n, q, s);
      CU(cudaGetLastError());
      CU(cudaMemcpyAsync(&counters[8 * i], pairs[i].counters, 32, cudaMemcpyDeviceToHost, s));
      CU(cudaMemcpyAsync(out[i].T, pairs[i].T, 128, cudaMemcpyDeviceToHost, s));
      if (corr_csr) CU(cudaMemcpyAsync(corr_csr + 2 * offsets[i], views[k].out_corr, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    }
  }
  CU(cudaStreamSynchronize(s));
  for (int i = 0; i < count; i++) {
    out[i].valid = counters[8 * i + 3];
    out[i].n_mutual = counters[8 * i + 1];
    out[i].n_corr = counters[8 * i + 2];
    out[i].clique_size = counters[8 * i + 4];
    out[i].gnc_iterations = counters[8 * i + 5];
    out[i].reserved = 0;
  }
  return B200REG_OK;
}
}  // namespace b200

extern "C" {

void b200reg_default_quatro_params(b200reg_quatro_params* p) {
  if (!p) return;
  p->fpfh_normal_radius = 0.9;
  p->fpfh_radius = 1.5;
  p->noise_bound = 0.3;
  p->rot_gnc_factor = 1.4;
  p->rot_cost_thr = 1e-4;
  p->rot_max_iter = 50;
  p->max_corres = 200;
  p->distance_threshold = 35.0;
  p->tuple_scale = 0.95;
  p->seed = 1;
  p->estimate_scale = 0;
  p->use_optimized_matching = 1;
}

int b200reg_clouds_fpfh(b200reg_ctx* c, int count, b200reg_cloud* const* clouds, double normal_radius, double fpfh_radius) {
  if (!c || count <= 0 || !clouds || !(normal_radius > 0) || !(fpfh_radius > 0)) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  std::vector<CloudDev> descs;
  std::vector<b200reg_cloud*> todo;
  int max_n = 0;
  for (int i = 0; i < count; i++) {
    b200reg_cloud* cl = clouds[i];
    if (!cl) return fail(B200REG_EINVAL, "NULL cloud");
    if (cl->has_fpfh && cl->normal_r == normal_radius && cl->fpfh_r == fpfh_radius) continue;
    if (std::find(todo.begin(), todo.end(), cl) != todo.end()) continue;
    if (!cl->fslab) {
      const size_t n = cl->dev.n;
      Layout l;
      const size_t o_n = l.take(n * sizeof(float4)), o_s = l.take(n * FPAD * sizeof(float)), o_f = l.take(n * FPAD * sizeof(float)),
                   o_fn = l.take(n * sizeof(float4)), o_fns = l.take(n * sizeof(float4)),
                   o_ft = l.take(2 * ((n + 63) / 64) * sizeof(float4)), o_fc = l.take(n * sizeof(uint32_t));
      char* fs = nullptr;
      CU(cudaMallocFromPoolAsync((void**)&fs, l.size, c->pool, s));
      cl->fslab = fs;
      cl->dev.nrm = (float4*)(fs + o_n);
      cl->dev.spfh = (float*)(fs + o_s);
      cl->dev.fpfh = (float*)(fs + o_f);
      cl->dev.fproj = (float4*)(fs + o_fn);
      cl->dev.fpfh_s = cl->dev.spfh;  // the SPFH table is dead once k_fpfh has consumed it
      cl->dev.fproj_s = (float4*)(fs + o_fns);
      cl->dev.ftile = (float4*)(fs + o_ft);
      cl->dev.fcode_s = (uint32_t*)(fs + o_fc);
    }
    todo.push_back(cl);
    descs.push_back(cl->dev);
    max_n = std::max(max_n, cl->dev.n);
  }
  if (todo.empty()) return B200REG_OK;
  // sort buffers of the filter-code ordering (scratch: only this call uses them); the work memory of all clouds is one
  // region, zeroed by one memset
  std::vector<SortLayout> sl;
  Layout bl, zl;
  for (auto& d : descs) sl.emplace_back(bl, zl, d.n, 32);
  char *sb = nullptr, *sz = nullptr;
  CU(scratch.alloc((void**)&sb, bl.size));
  CU(scratch.alloc((void**)&sz, zl.size));
  CU(cudaMemsetAsync(sz, 0, zl.size, s));
  std::vector<SortDev> sorts;
  for (auto& x : sl) sorts.push_back(x.bind(sb, sz));
  CloudDev* d_descs = nullptr;
  SortDev* d_sorts = nullptr;
  CU(scratch.upload(&d_descs, descs.data(), sizeof(CloudDev) * descs.size()));
  CU(scratch.upload(&d_sorts, sorts.data(), sizeof(SortDev) * sorts.size()));
  {
    ProfScope ps(c, CLS_FPFH);
    const float nr2 = (float)(normal_radius * normal_radius), fr2 = (float)(fpfh_radius * fpfh_radius);
    c->launches += launch_fpfh(d_descs, d_sorts, (int)descs.size(), max_n, nr2, fr2, s);
    for (auto& d : descs) c->prof_bytes[CLS_FPFH] += (32.0 + 164.0 + 280.0) * d.n;  // SURVEY §8(d) Q1+Q2+Q3
  }
  CU(cudaGetLastError());
  for (b200reg_cloud* cl : todo) {
    cl->has_fpfh = true;
    cl->normal_r = normal_radius;
    cl->fpfh_r = fpfh_radius;
  }
  return B200REG_OK;
}

int b200reg_get_fpfh(b200reg_ctx* c, const b200reg_cloud* cl, float* normals_out, float* fpfh_out) {
  if (!c || !cl) return fail(B200REG_EINVAL, "bad argument");
  if (!cl->has_fpfh) return fail(B200REG_ESTATE, "FPFH not computed");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const int n = cl->dev.n;
  std::vector<float4> nrm(n);
  std::vector<float> f((size_t)n * FPAD);
  std::vector<int> orig;
  CU(cudaMemcpyAsync(nrm.data(), cl->dev.nrm, (size_t)n * 16, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(f.data(), cl->dev.fpfh, (size_t)n * FPAD * 4, cudaMemcpyDeviceToHost, s));
  if (const int rc = sorted_to_original(c, cl->dev, orig)) return rc;
  for (int p = 0; p < n; p++) {
    const size_t o = orig[p];
    if (normals_out) {
      const bool ok = nrm[p].w != 0.f;
      normals_out[3 * o + 0] = ok ? nrm[p].x : NAN;
      normals_out[3 * o + 1] = ok ? nrm[p].y : NAN;
      normals_out[3 * o + 2] = ok ? nrm[p].z : NAN;
    }
    if (fpfh_out) memcpy(&fpfh_out[o * FDIM], &f[(size_t)p * FPAD], FDIM * sizeof(float));
  }
  return B200REG_OK;
}

int b200reg_quatro_align(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                         const b200reg_quatro_params* prm, b200reg_quatro_info* out, int32_t* corr_out) {
  return quatro_align_impl(c, count, src, dst, prm, out, corr_out, nullptr, 0, nullptr);
}

int b200reg_quatro_align_ex(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                            const b200reg_quatro_params* prm, b200reg_quatro_info* out, int64_t* offsets_out, size_t capacity,
                            int32_t* corr_out) {
  if (!offsets_out) return fail(B200REG_EINVAL, "bad argument");
  return quatro_align_impl(c, count, src, dst, prm, out, nullptr, offsets_out, capacity, corr_out);
}

int b200reg_quatro_solve_tap(b200reg_ctx* c, int n, const float* src_xyz, const float* dst_xyz, int wide,
                             const b200reg_quatro_params* prm, b200reg_quatro_info* info, int32_t* clique_out) {
  if (!c || n < 1 || n >= BIG_NMAX || !src_xyz || !dst_xyz || !prm || !info) return fail(B200REG_EINVAL, "bad argument");
  if (!wide && n > BIGC) return fail(B200REG_EINVAL, "wide = 0 solves at most B200REG_ADV_CORR_CAPACITY correspondences");
  if (wide == 2 && n > MAXC) return fail(B200REG_EINVAL, "wide = 2 solves at most B200REG_CORR_CAPACITY correspondences");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  const int counters[8] = {0, n, n, 0, 0, 0, 0, 0};
  MatchDev m{};
  const MatchDev* d_pair = nullptr;
  const int* d_clique = nullptr;
  if (wide == 2) {
    // k_teaser_solve, the solver of optimizedMatching's sets, reads its pair as b200reg_quatro_align leaves it: fi = the
    // source points, fj = the destination points, both in original order (identity rank), correspondence i = (i, i)
    std::vector<float4> pts(2 * (size_t)n);
    std::vector<int> ident(n), corr(2 * (size_t)n);
    for (int i = 0; i < n; i++) {
      float w;
      memcpy(&w, &i, 4);  // the original index, as the index build stores it
      pts[i] = make_float4(src_xyz[3 * i], src_xyz[3 * i + 1], src_xyz[3 * i + 2], w);
      pts[n + i] = make_float4(dst_xyz[3 * i], dst_xyz[3 * i + 1], dst_xyz[3 * i + 2], w);
      ident[i] = i;
      corr[2 * i] = corr[2 * i + 1] = i;
    }
    Layout l;
    const size_t o_pts = l.take(pts.size() * 16), o_rank = l.take((size_t)n * 4), o_oc = l.take(corr.size() * 4),
                 o_cnt = l.take(8 * 4), o_T = l.take(16 * 8), o_clq = l.take((size_t)n * 4), o_pair = l.take(sizeof(MatchDev));
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    m.fi.n = m.fj.n = n;
    m.fi.pts = (float4*)(slab + o_pts);
    m.fj.pts = m.fi.pts + n;
    m.fi.rank = m.fj.rank = (int*)(slab + o_rank);
    m.swapped = 0;
    m.out_corr = (int*)(slab + o_oc);
    m.counters = (int*)(slab + o_cnt);
    m.T = (double*)(slab + o_T);
    m.clique = (int*)(slab + o_clq);
    d_clique = m.clique;
    d_pair = (const MatchDev*)(slab + o_pair);
    CU(cudaMemcpyAsync(m.fi.pts, pts.data(), pts.size() * 16, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.fi.rank, ident.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.out_corr, corr.data(), corr.size() * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.counters, counters, sizeof counters, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(slab + o_pair, &m, sizeof m, cudaMemcpyHostToDevice, s));
    c->launches += launch_teaser_solve(d_pair, 1, quatro_params_dev(prm, false), s);
  } else {
    std::vector<double> S(3 * (size_t)n), D(3 * (size_t)n);
    for (size_t k = 0; k < 3 * (size_t)n; k++) {
      S[k] = src_xyz[k];  // k_big_gather's float -> double
      D[k] = dst_xyz[k];
    }
    // the workspace b200reg_quatro_align gives a set of this size on each path
    const int cap = wide ? (n + 1023) / 1024 * 1024 : std::max(1024, pow2_at_least(n));
    Layout l;
    const size_t o_big = l.take(sizeof(BigSolveWs)), o_cnt = l.take(8 * 4), o_T = l.take(16 * 8), o_pair = l.take(sizeof(MatchDev));
    const BigWsLayout wl(l, cap, 0);
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    const BigSolveWs w = wl.bind(slab);
    m.counters = (int*)(slab + o_cnt);
    m.T = (double*)(slab + o_T);
    m.big = (BigSolveWs*)(slab + o_big);
    d_clique = w.clique;
    d_pair = (const MatchDev*)(slab + o_pair);
    double T[16];
    for (int k = 0; k < 16; k++) T[k] = (k % 5 == 0) ? 1.0 : 0.0;
    CU(cudaMemcpyAsync(w.S, S.data(), S.size() * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(w.D, D.data(), D.size() * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(w.deg, 0, (size_t)n * 4, s));
    CU(cudaMemcpyAsync(m.counters, counters, sizeof counters, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.T, T, sizeof T, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.big, &w, sizeof w, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(slab + o_pair, &m, sizeof m, cudaMemcpyHostToDevice, s));
    c->launches += launch_big_graph_solve(d_pair, 1, quatro_params_dev(prm, true), wide ? n : 0, s);
  }
  CU(cudaGetLastError());
  int got[8];
  CU(cudaMemcpyAsync(got, m.counters, sizeof got, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(info->T, m.T, 128, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (clique_out && got[4] > 0) CU(cudaMemcpyAsync(clique_out, d_clique, (size_t)got[4] * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  info->valid = got[3];
  info->n_mutual = n;
  info->n_corr = n;
  info->clique_size = got[4];
  info->gnc_iterations = got[5];
  info->reserved = 0;
  return B200REG_OK;
}

int b200reg_match_tap(b200reg_ctx* c, int count, const float* const* fi, const int32_t* ni, const float* const* fj, const int32_t* nj,
                      double distance_threshold, int advanced, int32_t* const* nn_out, float* const* dis_out, int32_t* const* rnn_out,
                      int32_t* const* mutual_out, int32_t* n_mutual_out) {
  if (!c || count <= 0 || !fi || !ni || !fj || !nj || !nn_out || !dis_out || !rnn_out || !mutual_out || !n_mutual_out)
    return fail(B200REG_EINVAL, "bad argument");
  for (int k = 0; k < count; k++) {
    if (!fi[k] || !fj[k] || !nn_out[k] || !dis_out[k] || !rnn_out[k] || !mutual_out[k] || ni[k] < 1 || nj[k] < 1)
      return fail(B200REG_EINVAL, "bad argument");
    if (nj[k] > ni[k]) return fail(B200REG_EINVAL, "nj > ni: fi is the base of the forward search and must be the larger set");
  }
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  // cloud 2k = fi of pair k, 2k + 1 = its fj: the record tables b200reg_clouds_fpfh keeps, and the sort's temporaries
  std::vector<CloudDev> cl(2 * (size_t)count);
  std::vector<SortDev> sorts(2 * (size_t)count);
  std::vector<MatchDev> pairs(count);
  Layout l;
  std::vector<size_t> o_c(2 * (size_t)count), o_p(count);
  auto cloud_bytes = [](size_t n) {
    Layout x;
    for (size_t b : {n * FPAD * 4, n * 16, n * FPAD * 4, n * 16, 2 * ((n + 63) / 64) * 16, n * 4}) x.take(b);
    SortLayout(x, x, (int)n, 32);
    return x.size;
  };
  int max_n = 0, max_ni = 0, max_nj = 0;
  for (int k = 0; k < count; k++) {
    o_c[2 * k] = l.take(cloud_bytes(ni[k]));
    o_c[2 * k + 1] = l.take(cloud_bytes(nj[k]));
    o_p[k] = l.take(((size_t)nj[k] * 5 + (size_t)ni[k] * 2) * 4 + 32 + 64 + 256);
    max_ni = std::max(max_ni, (int)ni[k]);
    max_nj = std::max(max_nj, (int)nj[k]);
  }
  max_n = max_ni;
  char* slab = nullptr;
  CU(scratch.alloc((void**)&slab, l.size));
  for (int q = 0; q < 2 * count; q++) {
    const size_t n = q & 1 ? nj[q / 2] : ni[q / 2];
    CloudDev& d = cl[q];
    char* b = slab + o_c[q];
    Layout x;
    d.n = (int)n;
    d.fpfh = (float*)(b + x.take(n * FPAD * 4));
    d.fproj = (float4*)(b + x.take(n * 16));
    d.fpfh_s = (float*)(b + x.take(n * FPAD * 4));
    d.fproj_s = (float4*)(b + x.take(n * 16));
    d.ftile = (float4*)(b + x.take(2 * ((n + 63) / 64) * 16));
    d.fcode_s = (uint32_t*)(b + x.take(n * 4));
    const SortLayout sl(x, x, (int)n, 32);
    sorts[q] = sl.bind(b, b);
    CU(cudaMemsetAsync(sorts[q].hist, 0, sl.ws, s));
    // the caller's rows into slots 0..32 of the record table; k_load_records completes the records in place
    CU(cudaMemcpy2DAsync(d.fpfh, FPAD * 4, q & 1 ? fj[q / 2] : fi[q / 2], FDIM * 4, FDIM * 4, n, cudaMemcpyHostToDevice, s));
  }
  for (int k = 0; k < count; k++) {
    MatchDev& m = pairs[k];
    m.fi = cl[2 * k];
    m.fj = cl[2 * k + 1];
    const size_t a = ni[k], b = nj[k];
    char* p = slab + o_p[k];
    m.nn = (int*)p;
    m.dis = (float*)(p + b * 4);
    m.corres = (int*)(p + b * 8);
    m.tkey = (unsigned*)(p + b * 16);
    m.first_j = (int*)(p + b * 20);
    m.rnn = (int*)(p + b * 20 + a * 4);
    m.counters = (int*)(p + b * 20 + a * 8);
    m.stats = (double*)(p + (b * 20 + a * 8 + 32 + 63) / 64 * 64);
  }
  CloudDev* d_cl = nullptr;
  SortDev* d_sorts = nullptr;
  MatchDev* d_pairs = nullptr;
  CU(scratch.upload(&d_cl, cl.data(), sizeof(CloudDev) * cl.size()));
  CU(scratch.upload(&d_sorts, sorts.data(), sizeof(SortDev) * sorts.size()));
  CU(scratch.upload(&d_pairs, pairs.data(), sizeof(MatchDev) * count));
  {
    ProfScope ps(c, CLS_MATCH);
    c->launches += launch_load_records(d_cl, 2 * count, max_n, s);
    c->launches += launch_feature_order(d_cl, d_sorts, 2 * count, max_n, s);
    c->launches += launch_feature_match(d_pairs, count, max_ni, max_nj, match_thr2(distance_threshold, !!advanced), advanced ? 1 : 0, s);
  }
  CU(cudaGetLastError());
  std::vector<int> counters(8 * (size_t)count);
  for (int k = 0; k < count; k++) {
    CU(cudaMemcpyAsync(nn_out[k], pairs[k].nn, (size_t)nj[k] * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(dis_out[k], pairs[k].dis, (size_t)nj[k] * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(rnn_out[k], pairs[k].rnn, (size_t)ni[k] * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&counters[8 * k], pairs[k].counters, 32, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  for (int k = 0; k < count; k++) {
    n_mutual_out[k] = counters[8 * k + 1];
    if (n_mutual_out[k] > 0)
      CU(cudaMemcpyAsync(mutual_out[k], pairs[k].corres, (size_t)n_mutual_out[k] * 8, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

int b200reg_loop_closure(b200reg_ctx* c, int count, const float* const* src_xyz, const size_t* src_n, const float* const* tgt_xyz,
                         const size_t* tgt_n, size_t stride_bytes, int on_device, const b200reg_quatro_params* qp,
                         const b200reg_gicp_params* gp, b200reg_result* out, b200reg_quatro_info* quatro_out) {
  if (!c || count <= 0 || !src_xyz || !src_n || !tgt_xyz || !tgt_n || !qp || !gp || !out) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  LoopCapture cap(c, count);
  CloudBag bag(c);
  std::vector<b200reg_cloud*> sc(count), tc(count);
  int rc = create_pair_clouds(c, count, src_xyz, src_n, tgt_xyz, tgt_n, stride_bytes, on_device, cap.on(), bag, sc.data(), tc.data());
  if (!rc) rc = cap.clouds({}, sc.data(), tc.data(), false, true);
  std::vector<b200reg_quatro_info> own(quatro_out ? 0 : count);  // the capture reads the coarse stage's infos
  b200reg_quatro_info* qi = quatro_out ? quatro_out : own.data();
  std::vector<float> fine_tf(cap.on() ? 16 * (size_t)count : 0);
  if (!rc) rc = coarse_to_fine_on_clouds(c, count, sc.data(), tc.data(), qp, gp, out, qi, cap.on() ? fine_tf.data() : nullptr);
  if (!rc) rc = cap.finish(qi, fine_tf.data());
  return rc;
}

}  // extern "C"
