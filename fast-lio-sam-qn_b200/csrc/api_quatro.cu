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
  // the fine stage ran on the pairs vidx: its records, renumbered to these pairs
  c->records.rec[Records::TRACE].remap(count, vidx);
  c->records.rec[Records::RESIDUALS].remap(count, vidx);
  return B200REG_OK;
}

// BigSolveWs::cap for a set of up to n correspondences on each solve tier, the one sizing rule b200reg_quatro_align and
// b200reg_quatro_solve_tap share.  first: the batched advancedMatching pass, n the bound nj on the cross-checked set;
// opt_big: the batched pass over optimizedMatching sets beyond MAXC; wide: the advancedMatching sets beyond BIGC, solved
// one pair at a time in one workspace, n the largest.
enum class SolveTier { first, opt_big, wide };
static int solve_ws_cap(SolveTier tier, int n) {
  if (tier == SolveTier::wide) return (n + 1023) / 1024 * 1024;
  int cap = 1024;  // the power of two >= n, at least 1024; at most BIGC on the first pass
  while (cap < n && (tier == SolveTier::opt_big || cap < BIGC)) cap <<= 1;
  return cap;
}

// The global-memory solver workspace (BigSolveWs) for up to `cap` correspondences, cap a multiple of 1024 from
// solve_ws_cap.  nsrc > 0 adds k_adv_select_wide's scatter array for a source cloud of nsrc points.
struct BigWsLayout {
  int cap, words, p2;
  size_t o_S = 0, o_D = 0, o_adj = 0, o_radj = 0, o_int = 0, o_skey = 0, o_w = 0, o_res = 0, o_hval = 0, o_hidx = 0, o_best = 0,
         o_slot = 0;
  BigWsLayout(Layout& l, int cap_, int nsrc) : cap(cap_), words(cap_ / 32), p2(cap_ > 1 ? 1 << (32 - __builtin_clz(cap_ - 1)) : 1) {
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

// A cloud's descriptor tables (CloudDev::fpfh ... fcode_s) for n points.  with_spfh adds the normals and the SPFH table
// b200reg_clouds_fpfh computes them from; the SPFH table is dead once k_fpfh has consumed it, so fpfh_s reuses it.
// Offsets first, pointers at bind().
struct FeatureLayout {
  bool spfh;
  size_t o_nrm, o_spfh, o_fpfh, o_fproj, o_fpfh_s, o_fproj_s, o_ftile, o_fcode_s;
  FeatureLayout(Layout& l, size_t n, bool with_spfh)
      : spfh(with_spfh), o_nrm(spfh ? l.take(n * 16) : 0), o_spfh(spfh ? l.take(n * FPAD * 4) : 0), o_fpfh(l.take(n * FPAD * 4)),
        o_fproj(l.take(n * 16)), o_fpfh_s(spfh ? o_spfh : l.take(n * FPAD * 4)), o_fproj_s(l.take(n * 16)),
        o_ftile(l.take(2 * ((n + 63) / 64) * 16)), o_fcode_s(l.take(n * 4)) {}
  void bind(char* slab, CloudDev& d) const {
    if (spfh) { d.nrm = (float4*)(slab + o_nrm); d.spfh = (float*)(slab + o_spfh); }
    d.fpfh = (float*)(slab + o_fpfh); d.fproj = (float4*)(slab + o_fproj); d.fpfh_s = (float*)(slab + o_fpfh_s);
    d.fproj_s = (float4*)(slab + o_fproj_s); d.ftile = (float4*)(slab + o_ftile); d.fcode_s = (uint32_t*)(slab + o_fcode_s);
  }
};

// The matcher's per-pair arrays (MatchDev::nn ... stats) for ni >= nj descriptors, and the solve's outputs: T, and
// out_corr of corr_cap pairs unless that is 0.  ni = nj = 0 leaves the matcher's arrays empty, for a solve of given
// correspondences.  Offsets first, pointers at bind().
struct MatchLayout {
  size_t o_nn, o_dis, o_fj, o_rnn, o_cor, o_tk, o_cnt, o_st, o_oc, o_T;
  MatchLayout(Layout& l, size_t ni, size_t nj, size_t corr_cap)
      : o_nn(l.take(nj * 4)), o_dis(l.take(nj * 4)), o_fj(l.take(ni * 4)), o_rnn(l.take(ni * 4)), o_cor(l.take(2 * nj * 4)),
        o_tk(l.take(nj * 4)), o_cnt(l.take(sizeof(MatchCounters))), o_st(l.take(8 * 8)), o_oc(corr_cap ? l.take(2 * corr_cap * 4) : 0),
        o_T(l.take(16 * 8)) {}
  void bind(char* slab, MatchDev& m) const {
    m.nn = (int*)(slab + o_nn); m.dis = (float*)(slab + o_dis); m.first_j = (int*)(slab + o_fj); m.rnn = (int*)(slab + o_rnn);
    m.corres = (int*)(slab + o_cor); m.tkey = (unsigned*)(slab + o_tk); m.counters = (MatchCounters*)(slab + o_cnt);
    m.stats = (double*)(slab + o_st); m.out_corr = o_oc ? (int*)(slab + o_oc) : nullptr; m.T = (double*)(slab + o_T);
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

// one b200reg_quatro_align call: every pair's device workspace and, after each pass, its counters and out[i].T.  A call
// that records its matches (b200reg_ctx_set_quatro_matches) also keeps where each pair's clique list lives, the CSR
// offsets of its matches and the slab the capture writes.
struct QuatroCall {
  b200reg_ctx* c;
  Scratch& scratch;
  QuatroParamsDev q;
  b200reg_quatro_info* out;
  std::vector<MatchDev> pairs;
  std::vector<MatchCounters> counters;
  bool record;
  std::vector<const int*> clique_at;  // pair i's clique list once it is solved
  std::vector<int64_t> rec_offsets;   // pairs + 1
  char* rec_slab = nullptr;
};

// the size of a pair's final correspondence set: n_wide while the wide tier has the pair pending
static int set_size(const MatchCounters& k) { return k.n_wide > 0 ? k.n_wide : k.n_corr; }

// queues the copy of pair i's counters and T to the host
static cudaError_t fetch_result(QuatroCall& qc, int i) {
  const cudaError_t e = cudaMemcpyAsync(&qc.counters[i], qc.pairs[i].counters, sizeof(MatchCounters), cudaMemcpyDeviceToHost, qc.c->stream);
  return e != cudaSuccess ? e : cudaMemcpyAsync(qc.out[i].T, qc.pairs[i].T, 128, cudaMemcpyDeviceToHost, qc.c->stream);
}

static void fill_info(const MatchCounters& k, b200reg_quatro_info& o) {
  o.valid = k.valid;
  o.n_mutual = k.n_mutual;
  o.n_corr = k.n_corr;
  o.clique_size = k.clique_size;
  o.gnc_iterations = k.gnc_iterations;
  o.reserved = 0;
}

// Matches every pair and solves, in one batched pass, each set of at most MAXC (optimizedMatching, k_teaser_solve) or
// BIGC (advancedMatching, the global-memory chain).  corr_fixed (count x 2 x corr_stride ints) receives each pair's
// out_corr as this pass leaves it.
static int match_and_solve_first(QuatroCall& qc, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst, int corr_stride,
                                 int32_t* corr_fixed) {
  b200reg_ctx* c = qc.c;
  cudaStream_t s = c->stream;
  const bool advanced = qc.q.advanced;
  // optimizedMatching's out_corr: MAXC pairs, or max_corres + 3 when that is more
  const int opt_cap = std::max(MAXC, qc.q.max_corres + 3);
  qc.pairs.resize(count);
  qc.counters.resize(count);
  qc.clique_at.assign(count, nullptr);
  std::vector<BigSolveWs> big_host;
  big_host.reserve(count);  // addresses stay valid for the async copies below
  int max_ni = 0, max_nj = 0;
  for (int i = 0; i < count; i++) {
    MatchDev& m = qc.pairs[i];
    const bool swapped = dst[i]->dev.n > src[i]->dev.n;  // fi = larger cloud (matcher.cc:364-369)
    m.fi = swapped ? dst[i]->dev : src[i]->dev;
    m.fj = swapped ? src[i]->dev : dst[i]->dev;
    m.swapped = swapped ? 1 : 0;
    const size_t ni = m.fi.n, nj = m.fj.n;
    const int cap = advanced ? solve_ws_cap(SolveTier::first, (int)nj) : 0;
    // a recording call gives each optimizedMatching pair a clique row as long as its out_corr: k_teaser_solve, or
    // k_big_finish for a set beyond MAXC, lists the clique there.  advancedMatching's stays in its workspace.
    const bool clique_row = qc.record && !advanced;
    Layout l;
    const MatchLayout ml(l, ni, nj, advanced ? cap : opt_cap);
    const size_t o_big = advanced ? l.take(sizeof(BigSolveWs)) : 0;
    const BigWsLayout wl(l, cap, 0);  // empty when !advanced
    const size_t o_clq = clique_row ? l.take((size_t)opt_cap * 4) : 0;
    char* slab = nullptr;
    CU(qc.scratch.alloc((void**)&slab, l.size));
    ml.bind(slab, m);
    if (clique_row) m.clique = (int*)(slab + o_clq);
    qc.clique_at[i] = m.clique;
    if (advanced) {
      m.big = (BigSolveWs*)(slab + o_big);
      big_host.push_back(wl.bind(slab));
      qc.clique_at[i] = big_host.back().clique;
      CU(cudaMemcpyAsync(m.big, &big_host.back(), sizeof(BigSolveWs), cudaMemcpyHostToDevice, s));
    }
    max_ni = std::max(max_ni, (int)ni);
    max_nj = std::max(max_nj, (int)nj);
  }
  MatchDev* d_pairs = nullptr;
  CU(qc.scratch.upload(&d_pairs, qc.pairs.data(), sizeof(MatchDev) * count));
  {
    ProfScope ps(c, CLS_MATCH);
    c->launches += launch_quatro_match_solve(d_pairs, count, max_ni, max_nj, qc.q, s);
    for (const MatchDev& m : qc.pairs) c->prof_bytes[CLS_MATCH] += 132.0 * (m.fi.n + m.fj.n) + 8.0 * m.fj.n;  // SURVEY §8(d) Q4
  }
  CU(cudaGetLastError());
  for (int i = 0; i < count; i++) {
    CU(fetch_result(qc, i));
    if (corr_fixed) {
      const size_t have = advanced ? (size_t)big_host[i].cap : (size_t)MAXC;  // what this pair's buffer holds
      CU(cudaMemcpyAsync(&corr_fixed[2 * (size_t)corr_stride * i], qc.pairs[i].out_corr, 2 * have * 4, cudaMemcpyDeviceToHost, s));
    }
  }
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

// The optimizedMatching sets beyond MAXC, which k_teaser_solve left unsolved: each gets a workspace for its own size, and
// all of them are solved in one batched pass; each pair's view reads its own out_corr and writes its own counters and T.
static int solve_opt_big(QuatroCall& qc, const std::vector<int>& big) {
  cudaStream_t s = qc.c->stream;
  const int nb = (int)big.size();
  int max_big = 0;
  Layout l;
  const size_t o_views = l.take(sizeof(MatchDev) * nb), o_ws = l.take(sizeof(BigSolveWs) * nb);
  std::vector<BigWsLayout> wls;
  for (int i : big) {
    max_big = std::max(max_big, qc.counters[i].n_corr);
    wls.emplace_back(l, solve_ws_cap(SolveTier::opt_big, qc.counters[i].n_corr), 0);
  }
  char* slab = nullptr;
  if (qc.scratch.alloc((void**)&slab, l.size) != cudaSuccess) {
    cudaGetLastError();
    char msg[200];
    snprintf(msg, sizeof msg, "optimizedMatching kept up to %d correspondences; solving them needs a workspace of %zu bytes, "
             "which could not be allocated", max_big, l.size);
    return fail(B200REG_ECUDA, msg);
  }
  std::vector<MatchDev> views(nb);
  std::vector<BigSolveWs> ws(nb);
  for (int k = 0; k < nb; k++) {
    ws[k] = wls[k].bind(slab);
    views[k] = qc.pairs[big[k]];
    views[k].big = (BigSolveWs*)(slab + o_ws) + k;
  }
  CU(cudaMemcpyAsync(slab + o_ws, ws.data(), sizeof(BigSolveWs) * nb, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(slab + o_views, views.data(), sizeof(MatchDev) * nb, cudaMemcpyHostToDevice, s));
  {
    ProfScope ps(qc.c, CLS_MATCH);
    qc.c->launches += launch_big_solve((const MatchDev*)(slab + o_views), nb, max_big, qc.q, s);
  }
  CU(cudaGetLastError());
  for (int i : big) CU(fetch_result(qc, i));
  CU(cudaStreamSynchronize(s));  // views and ws stay alive until their copies are done
  return B200REG_OK;
}

// The advancedMatching sets beyond BIGC, which k_adv_select left unsolved: solved one pair after another in one workspace
// sized for the largest, so device memory stays bounded by the largest.  corr_csr receives pair i's set at offsets[i].
static int solve_wide(QuatroCall& qc, const std::vector<int>& wide, int32_t* corr_csr, const std::vector<int64_t>& offsets) {
  cudaStream_t s = qc.c->stream;
  int max_wide = 0, max_src = 0;
  for (int i : wide) {
    max_wide = std::max(max_wide, qc.counters[i].n_wide);
    max_src = std::max(max_src, qc.pairs[i].swapped ? qc.pairs[i].fj.n : qc.pairs[i].fi.n);
  }
  const int cap = solve_ws_cap(SolveTier::wide, max_wide);
  Layout l;
  const size_t o_big = l.take(sizeof(BigSolveWs)), o_pair = l.take(sizeof(MatchDev)), o_oc = l.take((size_t)cap * 8);
  const BigWsLayout wl(l, cap, max_src);
  char* slab = nullptr;
  if (qc.scratch.alloc((void**)&slab, l.size) != cudaSuccess) {
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
  {
    ProfScope ps(qc.c, CLS_MATCH);
    for (size_t k = 0; k < wide.size(); k++) {
      const int i = wide[k], n = qc.counters[i].n_wide;
      views[k] = qc.pairs[i];
      if (!qc.record) views[k].out_corr = (int*)(slab + o_oc);  // a recording call gave each pair rows of its own (record_begin)
      views[k].big = (BigSolveWs*)(slab + o_big);
      CU(cudaMemcpyAsync(slab + o_pair, &views[k], sizeof(MatchDev), cudaMemcpyHostToDevice, s));
      qc.c->launches += launch_adv_wide((const MatchDev*)(slab + o_pair), n, qc.q, s);
      CU(cudaGetLastError());
      CU(fetch_result(qc, i));
      if (corr_csr) CU(cudaMemcpyAsync(corr_csr + 2 * offsets[i], views[k].out_corr, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    }
  }
  CU(cudaStreamSynchronize(s));  // w and views stay alive until their copies are done
  return B200REG_OK;
}

// A recording call, once every pair is matched: the CSR offsets of the final sets, and one slab for the capture's rows
// and, ahead of solve_wide, for each wide pair's set and clique list (its workspace is shared with the next wide pair).
static int record_begin(QuatroCall& qc, int count) {
  qc.rec_offsets.assign(count + 1, 0);
  for (int i = 0; i < count; i++) qc.rec_offsets[i + 1] = qc.rec_offsets[i] + set_size(qc.counters[i]);
  const size_t total = (size_t)qc.rec_offsets[count];
  Layout l;
  l.take(total * 9 * 4);  // corr, inlier, src xyz, dst xyz: MatchCaptureOut
  std::vector<size_t> o_wide(count, 0);
  for (int i = 0; i < count; i++)
    if (qc.counters[i].n_wide > 0) o_wide[i] = l.take((size_t)qc.counters[i].n_wide * 3 * 4);
  if (qc.scratch.alloc((void**)&qc.rec_slab, l.size) != cudaSuccess) {
    cudaGetLastError();
    return fail(B200REG_ECUDA, "Quatro matches: cannot allocate " + std::to_string(l.size) + " bytes");
  }
  for (int i = 0; i < count; i++)
    if (qc.counters[i].n_wide > 0) {
      qc.pairs[i].out_corr = (int*)(qc.rec_slab + o_wide[i]);
      qc.pairs[i].clique = qc.pairs[i].out_corr + 2 * (size_t)qc.counters[i].n_wide;
      qc.clique_at[i] = qc.pairs[i].clique;
    }
  return B200REG_OK;
}

// A recording call, once every pair is solved: every match row into the slab in one launch and one copy into the
// context's record
static int record_finish(QuatroCall& qc, int count) {
  b200reg_ctx* c = qc.c;
  const int64_t total = qc.rec_offsets[count];
  MatchCaptureOut o;
  o.corr = (int*)qc.rec_slab;
  o.inlier = o.corr + 2 * total;
  o.sxyz = (float*)(o.inlier + total);
  o.dxyz = o.sxyz + 3 * total;
  std::vector<MatchCaptureRow> rows;
  int max_n = 0;
  for (int i = 0; i < count; i++) {
    const int n = (int)(qc.rec_offsets[i + 1] - qc.rec_offsets[i]);
    if (n == 0) continue;
    const MatchDev& p = qc.pairs[i];
    const CloudDev& sd = p.swapped ? p.fj : p.fi;
    const CloudDev& dd = p.swapped ? p.fi : p.fj;
    MatchCaptureRow r;
    r.corr = p.out_corr;
    r.clique = qc.clique_at[i];
    r.spts = sd.pts;
    r.srank = sd.rank;
    r.dpts = dd.pts;
    r.drank = dd.rank;
    r.n = n;
    r.m = qc.counters[i].clique_size;
    r.off = qc.rec_offsets[i];
    rows.push_back(r);
    max_n = std::max(max_n, n);
  }
  CsrRecord& qm = c->records.rec[Records::MATCHES];
  qm.rows.resize((size_t)total * 36);
  if (!rows.empty()) {
    MatchCaptureRow* d_rows = nullptr;
    CU(qc.scratch.upload(&d_rows, rows.data(), sizeof(MatchCaptureRow) * rows.size()));
    {
      ProfScope ps(c, CLS_MISC);
      launch_match_capture(d_rows, (int)rows.size(), max_n, o, c->stream);
      c->launches++;
      c->prof_bytes[CLS_MISC] += 76.0 * total;  // 8 corr + 32 points + ~4 clique in, 36 out
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(qm.rows.data(), qc.rec_slab, qm.rows.size(), cudaMemcpyDeviceToHost, c->stream));
  }
  CU(cudaStreamSynchronize(c->stream));
  qm.offsets = qc.rec_offsets;
  return B200REG_OK;
}

// b200reg_quatro_align (corr_fixed: count x 2 x CAP ints, or NULL) and b200reg_quatro_align_ex (offsets_out non-NULL;
// corr_csr: `capacity` pairs, or NULL).  Every pair is matched and, if its set holds at most BIGC correspondences,
// solved in one batched pass.  A larger advancedMatching set is then solved by solve_wide.  optimizedMatching keeps at
// most max_corres + 3 <= BIGC: k_teaser_solve solves the sets of at most MAXC in that pass, and solve_opt_big the rest.
static int quatro_align_impl(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst, const b200reg_quatro_params* prm,
                      b200reg_quatro_info* out, int32_t* corr_fixed, int64_t* offsets_out, size_t capacity, int32_t* corr_csr) {
  if (!c || count <= 0 || !src || !dst || !prm || !out) return fail(B200REG_EINVAL, "bad argument");
  if (prm->estimate_scale) return fail(B200REG_EINVAL, "estimate_scale is not supported (the deployment sets it false)");
  const bool advanced = !prm->use_optimized_matching;  // Matcher::advancedMatching (matcher.cc:118-356)
  if (!advanced && (prm->max_corres < 1 || prm->max_corres > OPT_MAX_CORRES)) return fail(B200REG_EINVAL, "max_corres must be in 1..8189");
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
  QuatroCall qc{c, scratch, quatro_params_dev(prm, advanced), out, {}, {}, c->capture.quatro_matches, {}, {}};
  if ((rc = match_and_solve_first(qc, count, src, dst, corr_stride, corr_fixed))) return rc;
  std::vector<int> big, wide;
  for (int i = 0; i < count; i++) {
    const int n = set_size(qc.counters[i]);
    if (corr_fixed && n > corr_stride) {
      char msg[200];
      snprintf(msg, sizeof msg, "%s kept %d correspondences for pair %d; corr_out holds %d per pair "
               "(b200reg_quatro_align_ex returns any number)", advanced ? "advancedMatching" : "optimizedMatching", n, i, corr_stride);
      return fail(B200REG_ESTATE, msg);
    }
    if (qc.counters[i].n_wide > 0) {
      if (n >= BIG_NMAX) {
        char msg[160];
        snprintf(msg, sizeof msg, "advancedMatching kept %d correspondences for pair %d; the solver takes fewer than %d", n, i, BIG_NMAX);
        return fail(B200REG_ESTATE, msg);
      }
      wide.push_back(i);
    } else if (!advanced && n > MAXC) {
      big.push_back(i);
    }
  }
  std::vector<int64_t> offsets;
  if (offsets_out) {
    offsets.assign(count + 1, 0);
    for (int i = 0; i < count; i++) offsets[i + 1] = offsets[i] + set_size(qc.counters[i]);
    memcpy(offsets_out, offsets.data(), sizeof(int64_t) * (count + 1));
    if (corr_csr && (uint64_t)offsets[count] > capacity) {
      char msg[160];
      snprintf(msg, sizeof msg, "the final correspondences number %lld; corr_out holds %zu", (long long)offsets[count], capacity);
      return fail(B200REG_ESTATE, msg);
    }
    if (corr_csr)
      for (int i = 0; i < count; i++)
        if (qc.counters[i].n_wide == 0 && qc.counters[i].n_corr > 0)
          CU(cudaMemcpyAsync(corr_csr + 2 * offsets[i], qc.pairs[i].out_corr, (size_t)qc.counters[i].n_corr * 8, cudaMemcpyDeviceToHost, s));
  }
  if (qc.record && (rc = record_begin(qc, count))) return rc;
  if (!big.empty() && (rc = solve_opt_big(qc, big))) return rc;
  if (!wide.empty() && (rc = solve_wide(qc, wide, corr_csr, offsets))) return rc;
  CU(cudaStreamSynchronize(s));
  for (int i = 0; i < count; i++) fill_info(qc.counters[i], out[i]);
  return qc.record ? record_finish(qc, count) : B200REG_OK;
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
      Layout l;
      const FeatureLayout fl(l, cl->dev.n, true);
      char* fs = nullptr;
      CU(cudaMallocFromPoolAsync((void**)&fs, l.size, c->pool, s));
      cl->fslab = fs;
      fl.bind(fs, cl->dev);
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
  Recording rec(c, REC_MATCHES);
  return rec.commit(quatro_align_impl(c, count, src, dst, prm, out, corr_out, nullptr, 0, nullptr), count);
}

int b200reg_quatro_align_ex(b200reg_ctx* c, int count, b200reg_cloud* const* src, b200reg_cloud* const* dst,
                            const b200reg_quatro_params* prm, b200reg_quatro_info* out, int64_t* offsets_out, size_t capacity,
                            int32_t* corr_out) {
  Recording rec(c, REC_MATCHES);
  if (!offsets_out) return fail(B200REG_EINVAL, "bad argument");
  return rec.commit(quatro_align_impl(c, count, src, dst, prm, out, nullptr, offsets_out, capacity, corr_out), count);
}

int b200reg_quatro_solve_tap(b200reg_ctx* c, int n, const float* src_xyz, const float* dst_xyz, int wide,
                             const b200reg_quatro_params* prm, b200reg_quatro_info* info, int32_t* clique_out) {
  if (!c || n < 1 || n >= BIG_NMAX || !src_xyz || !dst_xyz || !prm || !info) return fail(B200REG_EINVAL, "bad argument");
  if (!wide && n > BIGC) return fail(B200REG_EINVAL, "wide = 0 solves at most B200REG_ADV_CORR_CAPACITY correspondences");
  if (wide == 2 && n > MAXC) return fail(B200REG_EINVAL, "wide = 2 solves at most B200REG_CORR_CAPACITY correspondences");
  CU(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Scratch scratch(c);
  MatchCounters counters{};  // as the matcher leaves a set of n mutual pairs, all of them kept
  counters.n_mutual = counters.n_corr = n;
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
    const MatchLayout ml(l, 0, 0, n);
    const size_t o_pts = l.take(pts.size() * 16), o_rank = l.take((size_t)n * 4), o_clq = l.take((size_t)n * 4),
                 o_pair = l.take(sizeof(MatchDev));
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    ml.bind(slab, m);
    m.fi.n = m.fj.n = n;
    m.fi.pts = (float4*)(slab + o_pts);
    m.fj.pts = m.fi.pts + n;
    m.fi.rank = m.fj.rank = (int*)(slab + o_rank);
    m.swapped = 0;
    m.clique = (int*)(slab + o_clq);
    d_clique = m.clique;
    d_pair = (const MatchDev*)(slab + o_pair);
    CU(cudaMemcpyAsync(m.fi.pts, pts.data(), pts.size() * 16, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.fi.rank, ident.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.out_corr, corr.data(), corr.size() * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.counters, &counters, sizeof counters, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(slab + o_pair, &m, sizeof m, cudaMemcpyHostToDevice, s));
    c->launches += launch_teaser_solve(d_pair, 1, quatro_params_dev(prm, false), s);
  } else {
    std::vector<double> S(3 * (size_t)n), D(3 * (size_t)n);
    for (size_t k = 0; k < 3 * (size_t)n; k++) {
      S[k] = src_xyz[k];  // k_big_gather's float -> double
      D[k] = dst_xyz[k];
    }
    Layout l;
    const MatchLayout ml(l, 0, 0, 0);
    const size_t o_big = l.take(sizeof(BigSolveWs)), o_pair = l.take(sizeof(MatchDev));
    const BigWsLayout wl(l, solve_ws_cap(wide ? SolveTier::wide : SolveTier::first, n), 0);
    char* slab = nullptr;
    CU(scratch.alloc((void**)&slab, l.size));
    const BigSolveWs w = wl.bind(slab);
    ml.bind(slab, m);
    m.big = (BigSolveWs*)(slab + o_big);
    d_clique = w.clique;
    d_pair = (const MatchDev*)(slab + o_pair);
    double T[16];
    for (int k = 0; k < 16; k++) T[k] = (k % 5 == 0) ? 1.0 : 0.0;
    CU(cudaMemcpyAsync(w.S, S.data(), S.size() * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(w.D, D.data(), D.size() * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(w.deg, 0, (size_t)n * 4, s));
    CU(cudaMemcpyAsync(m.counters, &counters, sizeof counters, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.T, T, sizeof T, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(m.big, &w, sizeof w, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(slab + o_pair, &m, sizeof m, cudaMemcpyHostToDevice, s));
    c->launches += launch_big_graph_solve(d_pair, 1, quatro_params_dev(prm, true), wide ? n : 0, s);
  }
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(&counters, m.counters, sizeof counters, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(info->T, m.T, 128, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (clique_out && counters.clique_size > 0)
    CU(cudaMemcpyAsync(clique_out, d_clique, (size_t)counters.clique_size * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  fill_info(counters, *info);  // the solve leaves n_mutual and n_corr as uploaded: n
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
  std::vector<FeatureLayout> fls;
  std::vector<SortLayout> sls;
  std::vector<MatchLayout> mls;
  int max_ni = 0, max_nj = 0;
  for (int q = 0; q < 2 * count; q++) {
    cl[q].n = q & 1 ? nj[q / 2] : ni[q / 2];
    fls.emplace_back(l, cl[q].n, false);
    sls.emplace_back(l, l, cl[q].n, 32);
  }
  for (int k = 0; k < count; k++) {
    mls.emplace_back(l, ni[k], nj[k], 0);
    max_ni = std::max(max_ni, (int)ni[k]);
    max_nj = std::max(max_nj, (int)nj[k]);
  }
  char* slab = nullptr;
  CU(scratch.alloc((void**)&slab, l.size));
  for (int q = 0; q < 2 * count; q++) {
    CloudDev& d = cl[q];
    fls[q].bind(slab, d);
    sorts[q] = sls[q].bind(slab, slab);
    CU(cudaMemsetAsync(sorts[q].hist, 0, sls[q].ws, s));
    // the caller's rows into slots 0..32 of the record table; k_load_records completes the records in place
    CU(cudaMemcpy2DAsync(d.fpfh, FPAD * 4, q & 1 ? fj[q / 2] : fi[q / 2], FDIM * 4, FDIM * 4, d.n, cudaMemcpyHostToDevice, s));
  }
  for (int k = 0; k < count; k++) {
    pairs[k].fi = cl[2 * k];
    pairs[k].fj = cl[2 * k + 1];
    mls[k].bind(slab, pairs[k]);
  }
  CloudDev* d_cl = nullptr;
  SortDev* d_sorts = nullptr;
  MatchDev* d_pairs = nullptr;
  CU(scratch.upload(&d_cl, cl.data(), sizeof(CloudDev) * cl.size()));
  CU(scratch.upload(&d_sorts, sorts.data(), sizeof(SortDev) * sorts.size()));
  CU(scratch.upload(&d_pairs, pairs.data(), sizeof(MatchDev) * count));
  {
    ProfScope ps(c, CLS_MATCH);
    c->launches += launch_load_records(d_cl, 2 * count, max_ni, s);
    c->launches += launch_feature_order(d_cl, d_sorts, 2 * count, max_ni, s);
    c->launches += launch_feature_match(d_pairs, count, max_ni, max_nj, match_thr2(distance_threshold, !!advanced), advanced ? 1 : 0, s);
  }
  CU(cudaGetLastError());
  std::vector<MatchCounters> counters(count);
  for (int k = 0; k < count; k++) {
    CU(cudaMemcpyAsync(nn_out[k], pairs[k].nn, (size_t)nj[k] * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(dis_out[k], pairs[k].dis, (size_t)nj[k] * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(rnn_out[k], pairs[k].rnn, (size_t)ni[k] * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&counters[k], pairs[k].counters, sizeof(MatchCounters), cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  for (int k = 0; k < count; k++) {
    n_mutual_out[k] = counters[k].n_mutual;
    if (n_mutual_out[k] > 0)
      CU(cudaMemcpyAsync(mutual_out[k], pairs[k].corres, (size_t)n_mutual_out[k] * 8, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaStreamSynchronize(s));
  return B200REG_OK;
}

int b200reg_loop_closure(b200reg_ctx* c, int count, const float* const* src_xyz, const size_t* src_n, const float* const* tgt_xyz,
                         const size_t* tgt_n, size_t stride_bytes, int on_device, const b200reg_quatro_params* qp,
                         const b200reg_gicp_params* gp, b200reg_result* out, b200reg_quatro_info* quatro_out) {
  Recording rec(c, REC_ALL);
  if (!c || count <= 0 || !src_xyz || !src_n || !tgt_xyz || !tgt_n || !qp || !gp || !out) return fail(B200REG_EINVAL, "bad argument");
  CU(cudaSetDevice(c->device));
  LoopCapture cap(c);
  ResidualSlab rslab(c);
  int rc = rslab.reserve(count, src_n);  // the fine stage's source clouds have the sizes of the sources
  if (rc) return rc;
  CloudBag bag(c);
  std::vector<b200reg_cloud*> sc(count), tc(count);
  rc = create_pair_clouds(c, count, src_xyz, src_n, tgt_xyz, tgt_n, stride_bytes, on_device, cap.on(), bag, sc.data(), tc.data());
  if (!rc) rc = cap.clouds(count, sc.data(), tc.data(), false, true);
  std::vector<b200reg_quatro_info> own(quatro_out ? 0 : count);  // the capture reads the coarse stage's infos
  b200reg_quatro_info* qi = quatro_out ? quatro_out : own.data();
  std::vector<float> fine_tf(cap.on() ? 16 * (size_t)count : 0);
  if (!rc) rc = coarse_to_fine_on_clouds(c, count, sc.data(), tc.data(), qp, gp, out, qi, cap.on() ? fine_tf.data() : nullptr);
  if (!rc) rc = cap.finish(qi, fine_tf.data());
  return rec.commit(rc, count);
}

}  // extern "C"
