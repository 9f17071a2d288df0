// compat/mvicp_compat.hpp -- drop-in bodies for the reference's hot-path entry points on top of the C ABI.
//
// A maintainer of adrelino/mv-lm-icp replaces the bodies of
//     Frame::computePoseNeighboursKnn / computeClosestPointsToNeighbours        (src/internal/frame.cpp:67-185)
//     ICP_Ceres::ceresOptimizer / _ceresAngleAxis / _sophusSE3                  (src/internal/icp-ceres.cpp:220-475)
//     ICP_Ceres::pointToPoint_* / pointToPlane_*                                (src/internal/icp-ceres.cpp:137-218,525-565)
// by calls into this header (see INTEGRATION.md) and links libmvicp.so; main_multiview.cpp / main_pairwise.cpp stay as
// they are.  Only the reference's own types are used: Frame, OutgoingEdge, Correspondance (include/frame.h:18-102),
// Eigen::Vector3d (contiguous 24-byte xyz) and Eigen::Isometry3d (16 doubles, column-major).
//
// The engine processes ALL frames in one call, whereas the reference loops `for src: src.computeClosestPoints...`
// (main_multiview.cpp:119-127): the per-frame member functions below therefore trigger the batched call when invoked
// for the first non-fixed frame of a round and serve the other frames from the same result.
#pragma once
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../include/mvicp.h"

namespace mvicp_compat {

inline void check(int rc) { if (rc != MVICP_OK) throw std::runtime_error(std::string("mvicp: ") + mvicp_last_error()); }

// One engine per frame set (the reference's `vector<shared_ptr<Frame>> frames`), created lazily and cached.
template <class FrameT>
struct Session {
  mvicp_ctx* ctx = nullptr;
  const std::vector<std::shared_ptr<FrameT>>* frames = nullptr;
  std::vector<int32_t> e_src, e_dst;
  bool corr_valid = false, graph_pushed = false;
  struct Rec { int32_t first, second; double dist; };   // == struct Correspondance (frame.h:18-22)
  Rec* records = nullptr; int64_t records_cap = 0;       // page-locked staging of mvicp_get_all_edges (mvicp_host_alloc)
  ~Session() { mvicp_host_free(records); mvicp_destroy(ctx); }
  void reserve_records(int64_t cap) {
    if (cap <= records_cap) return;
    mvicp_host_free(records); records = nullptr; records_cap = 0;
    void* p = nullptr; check(mvicp_host_alloc(sizeof(Rec) * (size_t)cap, &p));
    records = static_cast<Rec*>(p); records_cap = cap;
  }

  void bind(const std::vector<std::shared_ptr<FrameT>>& fr) {
    if (ctx && frames == &fr) return;
    if (ctx) { mvicp_destroy(ctx); ctx = nullptr; }
    graph_pushed = false;
    mvicp_config cfg{0, 0, nullptr};
    check(mvicp_create(&cfg, &ctx));
    frames = &fr;
    std::vector<const double*> P, N; std::vector<int64_t> n;
    for (auto& f : fr) { P.push_back(f->pts[0].data()); N.push_back(f->nor.empty() ? nullptr : f->nor[0].data()); n.push_back((int64_t)f->pts.size()); }
    check(mvicp_set_frames(ctx, (int32_t)fr.size(), P.data(), N.data(), n.data()));
  }
  void push_poses() {
    std::vector<double> P; std::vector<uint8_t> fx;
    for (auto& f : *frames) { P.insert(P.end(), f->pose.data(), f->pose.data() + 16); fx.push_back(f->fixed ? 1 : 0); }
    check(mvicp_set_poses(ctx, P.data(), fx.data()));
  }
  void pull_poses() {
    std::vector<double> P(16 * frames->size());
    check(mvicp_get_poses(ctx, P.data()));
    for (size_t i = 0; i < frames->size(); ++i) std::copy(P.begin() + 16 * i, P.begin() + 16 * (i + 1), (*frames)[i]->pose.data());
  }
  void push_graph() {   // Frame::neighbours[*].neighbourIdx, in the reference's iteration order
    std::vector<int32_t> ns, nd;
    for (size_t i = 0; i < frames->size(); ++i)
      for (auto& ne : (*frames)[i]->neighbours) { ns.push_back((int32_t)i); nd.push_back(ne.neighbourIdx); }
    if (graph_pushed && ns == e_src && nd == e_dst) return;   // unchanged: keep the engine's per-edge search seeds
    e_src.swap(ns); e_dst.swap(nd);
    check(mvicp_set_graph(ctx, (int32_t)e_src.size(), e_src.data(), e_dst.data()));
    graph_pushed = true;
  }
};

// Frame::recomputeNormals for every frame (frame.cpp:244-255; loadFrames calls it per frame, main_multiview.cpp:68).
template <class FrameT>
void recomputeNormals(Session<FrameT>& s, std::vector<std::shared_ptr<FrameT>>& frames, int k = 10) {
  s.bind(frames);
  check(mvicp_recompute_normals(s.ctx, k));
  for (size_t i = 0; i < frames.size(); ++i) {
    frames[i]->nor.resize(frames[i]->pts.size());
    check(mvicp_get_normals(s.ctx, (int32_t)i, frames[i]->nor[0].data(), nullptr));
  }
}

// ApproachComponents::computeClosestPoints (main_multiview.cpp:119-127).  materialize = fill OutgoingEdge::correspondances
// on the host (the viewer reads them, Visualize.cpp:470-479); the optimiser itself never needs them on the host.
template <class FrameT>
void computeClosestPoints(Session<FrameT>& s, std::vector<std::shared_ptr<FrameT>>& frames, float cutoff, bool materialize) {
  s.bind(frames);
  s.push_graph();
  s.push_poses();
  check(mvicp_correspond(s.ctx, cutoff));
  s.corr_valid = true;
  // one call for every edge: counts / weights always, the 16-byte Correspondance records (bit-compatible with frame.h:18-22) on request
  int32_t E = 0; for (auto& f : frames) E += (int32_t)f->neighbours.size();
  std::vector<int64_t> off(E + 1); std::vector<float> w(E);
  int64_t cap = 0; for (auto& f : frames) cap += (int64_t)f->neighbours.size() * (int64_t)f->pts.size();
  if (materialize) s.reserve_records(cap);
  check(mvicp_get_all_edges(s.ctx, materialize ? (void*)s.records : nullptr, cap, off.data(), w.data()));
  int32_t e = 0;
  for (auto& f : frames)
    for (auto& ne : f->neighbours) {
      if (!f->fixed) {
        if (materialize) {
          static_assert(sizeof(ne.correspondances[0]) == 16, "Correspondance {int, int, double}");
          ne.correspondances.resize((size_t)(off[e + 1] - off[e]));
          if (off[e + 1] > off[e]) std::memcpy((void*)ne.correspondances.data(), &s.records[(size_t)off[e]], 16 * (size_t)(off[e + 1] - off[e]));
        }
        ne.weight = w[e];
      }
      ++e;
    }
}

// ICP_Ceres::ceresOptimizer* (include/icp-ceres.h:40-42): param = MVICP_PARAM_QUAT / _AA / _SE3.
template <class FrameT>
mvicp_lm_summary optimize(Session<FrameT>& s, std::vector<std::shared_ptr<FrameT>>& frames, int param, bool pointToPlane, bool robust) {
  s.bind(frames);
  frames[0]->fixed = true;   // side effect of every ceresOptimizer* (icp-ceres.cpp:242-244,342-344,417-419)
  if (!s.corr_valid) {       // caller filled OutgoingEdge::correspondances itself: hand them over
    s.push_graph(); s.push_poses();
    int32_t e = 0;
    for (auto& f : frames)
      for (auto& ne : f->neighbours) {
        std::vector<int32_t> a, b;
        for (auto& c : ne.correspondances) { a.push_back(c.first); b.push_back(c.second); }
        check(mvicp_set_edge(s.ctx, e++, a.data(), b.data(), (int64_t)a.size(), ne.weight));
      }
  }
  mvicp_lm_summary sum{};
  check(mvicp_optimize(s.ctx, param, pointToPlane ? MVICP_COST_P2PLANE : MVICP_COST_P2P, robust ? 1 : 0, nullptr, &sum));
  s.pull_poses();
  s.corr_valid = false;
  return sum;
}

// ICP_Ceres::pointToPoint_* / pointToPlane_* (include/icp-ceres.h:30-36): returns the src -> dst transform as 16 doubles.
template <class Vec3>
void pairwise(int param, bool pointToPlane, const std::vector<Vec3>& src, const std::vector<Vec3>& dst, const std::vector<Vec3>* nor,
              double pose16_out[16]) {
  mvicp_config cfg{0, 0, nullptr};
  check(mvicp_pairwise(&cfg, param, pointToPlane ? MVICP_COST_P2PLANE : MVICP_COST_P2P, src[0].data(), dst[0].data(),
                       nor ? (*nor)[0].data() : nullptr, (int64_t)src.size(), nullptr, pose16_out, nullptr));
}

// ICP_G2O::g2oOptimizer (include/icp-g2o.h:14, icp-g2o.cpp:149-303): the g2o backend on the same session; frame 0 becomes fixed.
// chi2 (nullable) receives chi2 before the first optimize() call and after every call (what icp-g2o.cpp:264,283 print).
template <class FrameT>
mvicp_g2o_summary g2oOptimizer(Session<FrameT>& s, std::vector<std::shared_ptr<FrameT>>& frames, bool pointToPlane,
                               std::vector<double>* chi2 = nullptr) {
  s.bind(frames);
  frames[0]->fixed = true;   // icp-g2o.cpp:182-186
  if (!s.corr_valid) {       // caller filled OutgoingEdge::correspondances itself: hand them over
    s.push_graph(); s.push_poses();
    int32_t e = 0;
    for (auto& f : frames)
      for (auto& ne : f->neighbours) {
        std::vector<int32_t> a, b;
        for (auto& c : ne.correspondances) { a.push_back(c.first); b.push_back(c.second); }
        check(mvicp_set_edge(s.ctx, e++, a.data(), b.data(), (int64_t)a.size(), ne.weight));
      }
  }
  mvicp_g2o_summary sum{};
  mvicp_g2o_options opt; mvicp_default_g2o_options(&opt);
  std::vector<double> chi((size_t)opt.max_calls + 1, 0.0);
  check(mvicp_optimize_g2o(s.ctx, pointToPlane ? MVICP_COST_P2PLANE : MVICP_COST_P2P, &opt, &sum, chi.data()));
  if (chi2) chi2->assign(chi.begin(), chi.begin() + sum.calls + 1);
  s.pull_poses();
  s.corr_valid = false;
  return sum;
}

// ICP_G2O::pointToPoint / pointToPlane (include/icp-g2o.h:10-11, icp-g2o.cpp:26-147): the src -> dst transform as 16 doubles.
template <class Vec3>
void pairwiseG2O(bool pointToPlane, const std::vector<Vec3>& src, const std::vector<Vec3>& dst, const std::vector<Vec3>* nor,
                 double pose16_out[16]) {
  mvicp_config cfg{0, 0, nullptr};
  check(mvicp_pairwise_g2o(&cfg, pointToPlane ? MVICP_COST_P2PLANE : MVICP_COST_P2P, src[0].data(), dst[0].data(),
                           nor ? (*nor)[0].data() : nullptr, (int64_t)src.size(), nullptr, pose16_out, nullptr));
}

// ICP_Closedform::pointToPoint / pointToPlane (include/icp-closedform.h; icp-closedform.cpp:9-54).
template <class Vec3>
void closedForm(bool pointToPlane, const std::vector<Vec3>& src, const std::vector<Vec3>& dst, const std::vector<Vec3>* nor, double pose16_out[16]) {
  mvicp_config cfg{0, 0, nullptr};
  check(mvicp_pairwise_closed(&cfg, pointToPlane ? MVICP_COST_P2PLANE : MVICP_COST_P2P, src[0].data(), dst[0].data(),
                              nor ? (*nor)[0].data() : nullptr, (int64_t)src.size(), pose16_out));
}

}  // namespace mvicp_compat
