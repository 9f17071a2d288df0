// lm_eval.cuh -- residual / Jacobian streaming kernel of the LM step (replaces Ceres' evaluator).
//
// Reference semantics (SURVEY 8(a) A7/A8/A9): per correspondence (p = src point, q = dst point, n = dst normal)
//   point-to-point  r = (R_s p + t_s) - (R_k q + t_k)                 include/icp-ceres.h:49-99,143-185,236-275
//   point-to-plane  r = ((R_s p + t_s) - (R_k q + t_k)) . (R_k n)     include/icp-ceres.h:101-141,187-234,277-316
//   robust          SoftLOneLoss(a = edge.weight): rho(s) = 2b(sqrt(1+s/b)-1), b = a^2; since rho'' < 0 Ceres'
//                   corrector scales the block's residuals and Jacobian rows by sqrt(rho')  (icp-ceres.cpp:284,374,449)
//   cost            1/2 sum rho(|r|^2)   (1/2 sum |r|^2 without loss)
//
// Formulation.  Both residuals are invariant under the dst rotation, so they are evaluated in the dst frame:
// x = T_k^-1 T_s p = R_rel p + t_rel, d = x - q; p2p: r = d, p2plane: r = d . n.  With the canonical body tangent
// xi = (upsilon, omega) of T_s <- T_s exp(xi):   dr/dxi_s = [m ; p x m],  m = R_rel^T n   (p2plane)
//                                                 J_s = R_rel [I | -[p]x]               (p2p)
// point-to-plane (scalar residual): the dst-side row is J_k = -J_s Ad(T_rel^-1), so ONE 6x6 block A = sum w J_s^T J_s,
// one 6-vector b = sum w J_s^T r and the cost are accumulated per edge; lm_step.cuh expands them to the (s,s),(s,k),
// (k,k) blocks and maps the canonical tangent to the active parameterisation (tangent_map()).
// point-to-point (3-vector residual expressed in WORLD axes by the reference): the cost and the gradient are the
// same in any frame, but the Gauss-Newton matrix is not (the residual axes rotate with T_k), so the world-frame rows
// J_s = R_s [I | -[p]x], J_k = -R_k [I | -[q]x] are used: J^T J is then a function of the moments sum w, sum w p,
// sum w q, sum w pp^T, sum w qq^T, sum w pq^T (28 doubles) which is what the kernel accumulates.
// Bytes per correspondence: idx 4 + src 16 + dst 16 (+ normal 16) = 36 / 52 B in the fp32-storage mode.
#pragma once
#include <cuda_runtime.h>
#include "knn.cuh"
#include "se3_math.cuh"
#include "types.cuh"

namespace mv {

enum { COST_P2P = 0, COST_P2PLANE = 1, COST_MIXED = 2 };

template <bool F32> __device__ __forceinline__ typename Rec<F32>::type rec_load(const void* base, int64_t i);
template <> __device__ __forceinline__ float4 rec_load<true>(const void* base, int64_t i) {
  return __ldg(reinterpret_cast<const float4*>(base) + i);
}
template <> __device__ __forceinline__ double4a rec_load<false>(const void* base, int64_t i) {
  const double2* p = reinterpret_cast<const double2*>(reinterpret_cast<const double4a*>(base) + i);
  const double2 a = __ldg(p), b = __ldg(p + 1);
  double4a r; r.x = a.x; r.y = a.y; r.z = b.x; r.w = b.y;
  return r;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// partial[tile][NBLK]: layout BLK_* of types.cuh
template <bool F32, bool NF32, int COST>
__global__ void __launch_bounds__(EVAL_THREADS, 2)
lm_eval_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const Tile* __restrict__ tiles,
               int tile_len, const int32_t* __restrict__ corr, const Rt* __restrict__ frame_Rt,
               const float* __restrict__ weight, int robust, double* __restrict__ partial, DoneGate gate) {
  const Tile t = tiles[blockIdx.x];
  if (gate.skip(t.edge)) return;   // issued speculatively after the solve (of this edge's component) terminated
  const EdgeDev e = edges[t.edge];
  __shared__ double sRel[12];
  __shared__ double sred[EVAL_THREADS / 32][NBLK];
  if (threadIdx.x == 0) {
    const Rt a = frame_Rt[e.src], k = frame_Rt[e.dst];
    double R[9]; matTmul(k.R, a.R, R);
    const double dt[3] = {a.t[0] - k.t[0], a.t[1] - k.t[1], a.t[2] - k.t[2]};
    double tr[3]; matTvec(k.R, dt, tr);
    for (int i = 0; i < 9; ++i) sRel[i] = R[i];
    sRel[9] = tr[0]; sRel[10] = tr[1]; sRel[11] = tr[2];
  }
  __syncthreads();
  double R[9], tr[3];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = sRel[i];
  tr[0] = sRel[9]; tr[1] = sRel[10]; tr[2] = sRel[11];
  const double a_w = (double)weight[t.edge];
  const double bb = a_w * a_w, cc = 1.0 / bb;

  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  double A[21], g[6], cost = 0.0;
#pragma unroll
  for (int i = 0; i < 21; ++i) A[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = 0.0;
  double sw = 0.0, swp[3] = {0, 0, 0}, swq[3] = {0, 0, 0}, swpp[6] = {0, 0, 0, 0, 0, 0}, swqq[6] = {0, 0, 0, 0, 0, 0},
         swpq[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // point-to-point moments

  const int end = min(t.start + tile_len, e.n_src);
  typedef typename Rec<F32>::type rec_t;
  constexpr int U = F32 ? 4 : 2;   // slots in flight per thread: all index loads, then all gathers, then the math
  for (int k0 = t.start + threadIdx.x; k0 < end; k0 += U * EVAL_THREADS) {
    int cidx[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = k0 + u * EVAL_THREADS;
      cidx[u] = (k < end) ? __ldg(corr + e.off + k) : -1;
    }
    typedef typename Rec<NF32>::type nrec_t;   // normals keep fp32 records only while they are fp32-exact (not after mvicp_recompute_normals)
    rec_t P[U], Q[U]; nrec_t Nn[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (cidx[u] >= 0) {
        P[u] = rec_load<F32>(fs.pts_o, k0 + u * EVAL_THREADS);
        if (F32 && NF32 && COST != COST_P2P) {   // point and normal of the match from one 32-byte record: one sector per gather
          const float4* pn = fd.pn_o + 2 * (size_t)cidx[u];
          const float4 a = __ldg(pn), b = __ldg(pn + 1);
          Q[u].x = a.x; Q[u].y = a.y; Q[u].z = a.z; Nn[u].x = b.x; Nn[u].y = b.y; Nn[u].z = b.z;
        } else {
          Q[u] = rec_load<F32>(fd.pts_o, cidx[u]);
          if (COST != COST_P2P) Nn[u] = rec_load<NF32>(fd.nor_o, cidx[u]);
        }
      }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (cidx[u] < 0) continue;
      const double px = (double)P[u].x, py = (double)P[u].y, pz = (double)P[u].z;
      const double qx = (double)Q[u].x, qy = (double)Q[u].y, qz = (double)Q[u].z;
      const double x0 = R[0] * px + R[1] * py + R[2] * pz + tr[0];
      const double x1 = R[3] * px + R[4] * py + R[5] * pz + tr[1];
      const double x2 = R[6] * px + R[7] * py + R[8] * pz + tr[2];
      const double d0 = x0 - qx, d1 = x1 - qy, d2 = x2 - qz;
      if (COST == COST_P2PLANE || COST == COST_MIXED) {
        const double nx = (double)Nn[u].x, ny = (double)Nn[u].y, nz = (double)Nn[u].z;
        const double r = d0 * nx + d1 * ny + d2 * nz;
        const double s = r * r;
        double w = 1.0;
        if (robust) { const double arg = 1.0 + s * cc; w = rsqrt(arg); cost += bb * (arg * w - 1.0); }
        else cost += 0.5 * s;
        double a[6];
        a[0] = R[0] * nx + R[3] * ny + R[6] * nz;   // m = R_rel^T n
        a[1] = R[1] * nx + R[4] * ny + R[7] * nz;
        a[2] = R[2] * nx + R[5] * ny + R[8] * nz;
        a[3] = py * a[2] - pz * a[1];               // p x m
        a[4] = pz * a[0] - px * a[2];
        a[5] = px * a[1] - py * a[0];
        const double wr = w * r;
        int idx = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          const double wa = w * a[i];
          g[i] += wr * a[i];
#pragma unroll
          for (int j = i; j < 6; ++j) A[idx++] += wa * a[j];
        }
      }
      if (COST == COST_P2P || COST == COST_MIXED) {
        const double s = d0 * d0 + d1 * d1 + d2 * d2;
        double w = 1.0;
        if (robust) { const double arg = 1.0 + s * cc; w = rsqrt(arg); cost += bb * (arg * w - 1.0); }
        else cost += 0.5 * s;
        const double u0 = R[0] * d0 + R[3] * d1 + R[6] * d2;   // u = R_rel^T d
        const double u1 = R[1] * d0 + R[4] * d1 + R[7] * d2;
        const double u2 = R[2] * d0 + R[5] * d1 + R[8] * d2;
        g[0] += w * u0; g[1] += w * u1; g[2] += w * u2;
        g[3] += w * (py * u2 - pz * u1); g[4] += w * (pz * u0 - px * u2); g[5] += w * (px * u1 - py * u0);
        sw += w;
        const double wx = w * px, wy = w * py, wz = w * pz;
        const double vx = w * qx, vy = w * qy, vz = w * qz;
        swp[0] += wx; swp[1] += wy; swp[2] += wz;
        swq[0] += vx; swq[1] += vy; swq[2] += vz;
        swpp[0] += wx * px; swpp[1] += wx * py; swpp[2] += wx * pz; swpp[3] += wy * py; swpp[4] += wy * pz; swpp[5] += wz * pz;
        swqq[0] += vx * qx; swqq[1] += vx * qy; swqq[2] += vx * qz; swqq[3] += vy * qy; swqq[4] += vy * qz; swqq[5] += vz * qz;
        swpq[0] += wx * qx; swpq[1] += wx * qy; swpq[2] += wx * qz;
        swpq[3] += wy * qx; swpq[4] += wy * qy; swpq[5] += wy * qz;
        swpq[6] += wz * qx; swpq[7] += wz * qy; swpq[8] += wz * qz;
      }
    }
  }
  // block reduction: warp shuffles, then one value per warp through shared memory, fixed order
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  constexpr int NUSED = (COST == COST_P2PLANE) ? NBLK_PLANE : NBLK;
#define MV_RED(val, slot) { const double v_ = warp_sum(val); if (lane == 0) sred[wid][slot] = v_; }
  if (COST != COST_P2P) {
#pragma unroll
    for (int i = 0; i < 21; ++i) MV_RED(A[i], BLK_A + i)
  } else if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 21; ++i) sred[wid][BLK_A + i] = 0.0;
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) MV_RED(g[i], BLK_B + i)
  MV_RED(cost, BLK_COST)
  if (COST != COST_P2PLANE) {
    MV_RED(sw, BLK_SW)
#pragma unroll
    for (int i = 0; i < 3; ++i) { MV_RED(swp[i], BLK_SWP + i) MV_RED(swq[i], BLK_SWQ + i) }
#pragma unroll
    for (int i = 0; i < 6; ++i) { MV_RED(swpp[i], BLK_SWPP + i) MV_RED(swqq[i], BLK_SWQQ + i) }
#pragma unroll
    for (int i = 0; i < 9; ++i) MV_RED(swpq[i], BLK_SWPQ + i)
  }
#undef MV_RED
  __syncthreads();
  if (threadIdx.x < NUSED) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < EVAL_THREADS / 32; ++w) v += sred[w][threadIdx.x];
    partial[(size_t)blockIdx.x * NBLK + threadIdx.x] = v;
  }
}

// One CTA per edge: (1) sum the edge's tile partials in tile order (deterministic), (2) expand the block into the edge's
// 12x12 pair matrix and 12-vector over the two frames' parameterisation tangents:
//   canonical pair matrix (over [xi_s, xi_k]):
//     point-to-plane part  [I | -Q]^T A [I | -Q],  Q = Ad(T_rel^-1) = [[R^T, -R^T [t]x], [0, R^T]]  (R = R_rel, t = t_rel)
//     point-to-point part  from the moments, world-frame rows J_s = R_s [I | -[p]x], J_k = -R_k [I | -[q]x]
//   then Hp = Kpair^T Hcan Kpair with Kpair = diag(K_s, K_k) (tangent_map), gp = Kpair^T [b ; -Q^T b].
// out[e] = Hp (144) | gp (12) | cost | pad; zeros for edges this rank does not own (an all-reduce then gathers).
constexpr int EDGE_THREADS = 64;
constexpr int EOUT_ = 160;

// Sharded runs: the per-edge result is pushed straight into every peer GPU's exchange buffer over NVLink (each edge has
// exactly one owner, so the "all-reduce" of the pair matrices is really an all-to-all broadcast with no arithmetic and
// no ordering issue), and the last CTA of the grid raises this rank's flag on every peer; lm_step_kernel waits for all
// ranks' flags.  Compute and collective are one kernel; NCCL is not on the LM loop's critical path.
constexpr int MAX_PEERS = 16;
struct PeerTable {
  int world, rank;
  double* eout[MAX_PEERS];          // peer p's exchange area for the current buffer half (IPC-mapped), [E][EOUT]
  volatile int* flags[MAX_PEERS];   // peer p's flag array: flags[p][r] = last sequence number rank r completed
};

__device__ __forceinline__ void edge_publish(const PeerTable& pt, int e, int r, double v, double* __restrict__ o) {
  o[r] = v;
  for (int p = 0; p < pt.world; ++p) if (p != pt.rank) pt.eout[p][(size_t)EOUT_ * e + r] = v;
}
// every CTA of the edge kernels ends here: fence the remote stores, count, and let the last CTA raise the flags
__device__ __forceinline__ void edge_signal(const PeerTable& pt, int seq, unsigned int* counter) {
  if (pt.world <= 1) return;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(counter, 1u);
    if (prev == gridDim.x - 1) {
      *counter = 0u;
      __threadfence_system();
      for (int p = 0; p < pt.world; ++p) pt.flags[p][pt.rank] = seq;
      __threadfence_system();
    }
  }
}
__global__ void __launch_bounds__(EDGE_THREADS)
lm_edge_kernel(const EdgeDev* __restrict__ edges, const int32_t* __restrict__ edge_tile_begin, const double* __restrict__ partial,
               int nused, const Rt* __restrict__ frame_Rt, const double* __restrict__ K_eval, double* __restrict__ out,
               DoneGate gate, PeerTable pt, int seq, unsigned int* counter) {
  if (gate.skip(blockIdx.x)) return;
  const int e = blockIdx.x, tid = threadIdx.x;
  __shared__ double blk[NBLK], Q[36], AQ[36], Hcan[144], T1[144], Rt_[9];
  double* o = out + (size_t)EOUT_ * e;
  if (!edges[e].owned) {   // NCCL mode: zeros for the sum; peer mode: the owner writes this edge into our buffer
    if (pt.world <= 1) for (int i = tid; i < EOUT_; i += EDGE_THREADS) o[i] = 0.0;
    edge_signal(pt, seq, counter);
    return;
  }
  if (tid < NBLK) {
    double v = 0.0;
    if (tid < nused) for (int t = edge_tile_begin[e]; t < edge_tile_begin[e + 1]; ++t) v += partial[(size_t)t * NBLK + tid];
    blk[tid] = v;
  }
  if (tid == 0) {
    const Rt a = frame_Rt[edges[e].src], k = frame_Rt[edges[e].dst];
    double R[9]; matTmul(k.R, a.R, R);
    const double dt[3] = {a.t[0] - k.t[0], a.t[1] - k.t[1], a.t[2] - k.t[2]};
    double t[3]; matTvec(k.R, dt, t);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt_[3 * i + j] = R[3 * j + i];
    const double tx[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
    double RtTx[9]; matmul(Rt_, tx, RtTx);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        Q[6 * i + j] = Rt_[3 * i + j]; Q[6 * i + 3 + j] = -RtTx[3 * i + j];
        Q[6 * (3 + i) + j] = 0.0;      Q[6 * (3 + i) + 3 + j] = Rt_[3 * i + j];
      }
  }
  for (int i = tid; i < 144; i += EDGE_THREADS) Hcan[i] = 0.0;
  __syncthreads();
  if (tid == 0 && blk[BLK_SW] != 0.0) {   // point-to-point part of the canonical pair matrix
    const double* m = blk;
    const double sw = m[BLK_SW];
    const double* sp = m + BLK_SWP; const double* sq = m + BLK_SWQ;
    const double pp[9] = {m[BLK_SWPP], m[BLK_SWPP + 1], m[BLK_SWPP + 2], m[BLK_SWPP + 1], m[BLK_SWPP + 3], m[BLK_SWPP + 4],
                          m[BLK_SWPP + 2], m[BLK_SWPP + 4], m[BLK_SWPP + 5]};
    const double qq[9] = {m[BLK_SWQQ], m[BLK_SWQQ + 1], m[BLK_SWQQ + 2], m[BLK_SWQQ + 1], m[BLK_SWQQ + 3], m[BLK_SWQQ + 4],
                          m[BLK_SWQQ + 2], m[BLK_SWQQ + 4], m[BLK_SWQQ + 5]};
    const double* pq = m + BLK_SWPQ;
    const double px[9] = {0, -sp[2], sp[1], sp[2], 0, -sp[0], -sp[1], sp[0], 0};   // [sum w p]x
    const double qx[9] = {0, -sq[2], sq[1], sq[2], 0, -sq[0], -sq[1], sq[0], 0};
    const double trp = pp[0] + pp[4] + pp[8], trq = qq[0] + qq[4] + qq[8];
    double RtQx[9]; matmul(Rt_, qx, RtQx);      // R^T [swq]x
    double PxRt[9]; matmul(px, Rt_, PxRt);      // [swp]x R^T
    double* Hc_ = Hcan;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const double dij = (i == j) ? 1.0 : 0.0;
        // (s,s) and (k,k): [[w I, -[wp]x], [[wp]x, tr(wpp) I - wpp]]
        Hc_[12 * i + j] = sw * dij;                         Hc_[12 * (6 + i) + 6 + j] = sw * dij;
        Hc_[12 * i + 3 + j] = -px[3 * i + j];               Hc_[12 * (6 + i) + 9 + j] = -qx[3 * i + j];
        Hc_[12 * (3 + i) + j] = px[3 * i + j];              Hc_[12 * (9 + i) + 6 + j] = qx[3 * i + j];
        Hc_[12 * (3 + i) + 3 + j] = trp * dij - pp[3 * i + j];
        Hc_[12 * (9 + i) + 9 + j] = trq * dij - qq[3 * i + j];
        // (s,k) = -[I | -[p]x]^T R^T [I | -[q]x]
        double ww = 0.0;   // sum_{c,d} wpq[c][d] (E_c R^T E_d)_{ij},  (E_c)_{ik} = eps(i,c,k)
        for (int c2 = 0; c2 < 3; ++c2)
          for (int d2 = 0; d2 < 3; ++d2) {
            double acc = 0.0;
            for (int kk = 0; kk < 3; ++kk)
              for (int ll = 0; ll < 3; ++ll) {
                const int e1 = (i - c2) * (c2 - kk) * (kk - i), e2 = (ll - d2) * (d2 - j) * (j - ll);
                if (e1 && e2) acc += 0.25 * (double)(e1 * e2) * Rt_[3 * kk + ll];
              }
            ww += pq[3 * c2 + d2] * acc;
          }
        const double sk_uu = -sw * Rt_[3 * i + j], sk_uw = RtQx[3 * i + j], sk_wu = -PxRt[3 * i + j], sk_ww = ww;
        Hc_[12 * i + 6 + j] = sk_uu;        Hc_[12 * (6 + j) + i] = sk_uu;
        Hc_[12 * i + 9 + j] = sk_uw;        Hc_[12 * (9 + j) + i] = sk_uw;
        Hc_[12 * (3 + i) + 6 + j] = sk_wu;  Hc_[12 * (6 + j) + 3 + i] = sk_wu;
        Hc_[12 * (3 + i) + 9 + j] = sk_ww;  Hc_[12 * (9 + j) + 3 + i] = sk_ww;
      }
  }
  if (tid < 36) {      // AQ = A Q
    const int i = tid / 6, j = tid - 6 * i;
    double s = 0;
    for (int m = 0; m < 6; ++m) {
      const int a = min(i, m), b = max(i, m);
      s += blk[BLK_A + a * 6 - (a * (a - 1)) / 2 + (b - a)] * Q[6 * m + j];
    }
    AQ[tid] = s;
  }
  __syncthreads();
  for (int r = tid; r < 144; r += EDGE_THREADS) {     // Hcan += [I | -Q]^T A [I | -Q]
    const int a = r / 12, b = r - 12 * a;
    double v;
    if (a < 6 && b < 6) { const int lo = min(a, b), hi = max(a, b); v = blk[BLK_A + lo * 6 - (lo * (lo - 1)) / 2 + (hi - lo)]; }
    else if (a < 6) v = -AQ[6 * a + (b - 6)];
    else if (b < 6) v = -AQ[6 * b + (a - 6)];
    else { v = 0; for (int i = 0; i < 6; ++i) v += Q[6 * i + (a - 6)] * AQ[6 * i + (b - 6)]; }
    Hcan[r] += v;
  }
  __syncthreads();
  const double* Ks = K_eval + 36 * edges[e].src; const double* Kk = K_eval + 36 * edges[e].dst;
  for (int r = tid; r < 144; r += EDGE_THREADS) {     // T1 = Hcan Kpair
    const int a = r / 12, b = r - 12 * a;
    const double* Kb = b < 6 ? Ks : Kk; const int off = b < 6 ? 0 : 6;
    double v = 0; for (int m = 0; m < 6; ++m) v += Hcan[12 * a + off + m] * Kb[6 * m + (b - off)];
    T1[r] = v;
  }
  __syncthreads();
  for (int r = tid; r < 157; r += EDGE_THREADS) {     // Hp = Kpair^T T1 (144), gp = Kpair^T [b ; -Q^T b] (12), cost
    if (r < 144) {
      const int a = r / 12, b = r - 12 * a;
      const double* Ka = a < 6 ? Ks : Kk; const int off = a < 6 ? 0 : 6;
      double v = 0; for (int m = 0; m < 6; ++m) v += Ka[6 * m + (a - off)] * T1[12 * (off + m) + b];
      edge_publish(pt, e, r, v, o);
    } else if (r < 156) {
      const int a = r - 144;
      const double* bv = blk + BLK_B;
      const double* Ka = a < 6 ? Ks : Kk; const int off = a < 6 ? 0 : 6;
      double v = 0;
      for (int m = 0; m < 6; ++m) {
        double gm;
        if (a < 6) gm = bv[m];
        else { gm = 0; for (int i = 0; i < 6; ++i) gm -= Q[6 * i + m] * bv[i]; }
        v += Ka[6 * m + (a - off)] * gm;
      }
      edge_publish(pt, e, r, v, o);
    } else edge_publish(pt, e, r, blk[BLK_COST], o);
  }
  if (tid < 3) o[157 + tid] = 0.0;
  edge_signal(pt, seq, counter);
}


// ---- general path: non-unit quaternions (non-rigid input poses, or quaternion poses that drifted) ----------------------
// Same contract as lm_eval_kernel, for the frame model of frame_general(): y = F v + t with F no rotation, Jacobian rows
// through the per-frame matrices D_j, c_j (the relative-pose shortcut needs orthogonal F), the 12x12 pair matrix accumulated
// directly: 78 + 12 + 1 sums per correspondence.  That is too many fp64 accumulators for one thread, and splitting them over
// passes (rounds 1-2: three) recomputes the Jacobian row in each -- 70 % of the arithmetic.  So TWO LANES share a
// correspondence: the even lane owns the src frame's half of the row, the odd lane the dst frame's; they swap halves with one
// shuffle per entry, and each accumulates its own diagonal block (21), half of the off-diagonal block (18), its half of the
// gradient (6) -- 46 sums per lane, one pass, the row computed once.  Both lanes run the same instruction stream (role-selected
// operands, no divergence).  The tangent is handled in the order (rotation, translation): D_j = 0 for translation directions
// and c_j = 0 for rotation directions in both parameterisations (frame_general), which halves the row's cost; `rot0` (0:
// quaternion, 3: SE3) maps that order back when the sums are written.
constexpr int GBLK = 96;   // stride of a general partial: 78 (upper 12x12) | 12 | 1
constexpr int GACC = 46;   // per lane: 21 own block | 18 half of the (s,k) block | 6 gradient | cost
__device__ __forceinline__ int u12(int i, int j) { return i * 12 - (i * (i - 1)) / 2 + (j - i); }

template <bool F32, bool NF32, int COST>
__global__ void __launch_bounds__(EVAL_THREADS)
lm_eval_general_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const Tile* __restrict__ tiles,
                       int tile_len, const int32_t* __restrict__ corr, const FrameGen* __restrict__ frame_gen,
                       const float* __restrict__ weight, int robust, int rot0, double* __restrict__ partial, DoneGate gate) {
  const Tile t = tiles[blockIdx.x];
  if (gate.skip(t.edge)) return;
  const EdgeDev e = edges[t.edge];
  __shared__ FrameGen g2[2];                                    // [0] src frame, [1] dst frame
  __shared__ double sred[EVAL_THREADS / 32][2][GACC];
  {
    const double* a = reinterpret_cast<const double*>(frame_gen + e.src); const double* b = reinterpret_cast<const double*>(frame_gen + e.dst);
    double* sa = reinterpret_cast<double*>(&g2[0]); double* sb = reinterpret_cast<double*>(&g2[1]);
    for (int i = threadIdx.x; i < (int)(sizeof(FrameGen) / sizeof(double)); i += blockDim.x) { sa[i] = a[i]; sb[i] = b[i]; }
  }
  __syncthreads();
  const int role = threadIdx.x & 1;                              // 0: src half of the row, 1: dst half
  const FrameGen& gs = g2[0]; const FrameGen& gk = g2[1]; const FrameGen& gm = g2[role];
  const int tra0 = 3 - rot0;
  const double sgn = role ? -1.0 : 1.0;
  const double a_w = (double)weight[t.edge];
  const double bb = a_w * a_w, cc = 1.0 / bb;
  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  double acc[GACC];
#pragma unroll
  for (int i = 0; i < GACC; ++i) acc[i] = 0.0;
  const int end = min(t.start + tile_len, e.n_src);
  for (int k0 = t.start; k0 < end; k0 += EVAL_THREADS / 2) {    // uniform trip count: the pair shuffles need every lane
    const int k = k0 + (threadIdx.x >> 1);
    const int c = k < end ? __ldg(corr + e.off + k) : -1;
    const bool ok = c >= 0;
    if (!__any_sync(0xffffffffu, ok)) continue;
    double p[3] = {0, 0, 0}, q[3] = {0, 0, 0}, n[3] = {0, 0, 0}; int dummy;
    if (ok) {
      Rec<F32>::load(fs.pts_o, k, p[0], p[1], p[2], dummy);
      Rec<F32>::load(fd.pts_o, c, q[0], q[1], q[2], dummy);
      if (COST != COST_P2P) Rec<NF32>::load(fd.nor_o, c, n[0], n[1], n[2], dummy);
    }
    const double live = ok ? 1.0 : 0.0;                          // an empty slot adds exact zeros
    double ys[3], yk[3], n2[3], d[3];
    matvec(gs.F, p, ys); matvec(gk.F, q, yk); matvec(gk.F, n, n2);
#pragma unroll
    for (int i = 0; i < 3; ++i) d[i] = (ys[i] + gs.t[i]) - (yk[i] + gk.t[i]);
    // this lane's half of the point Jacobians: rotation directions D_j v, translation directions c_j  (v = p | q)
    const double v[3] = {role ? q[0] : p[0], role ? q[1] : p[1], role ? q[2] : p[2]};
    const double dk[3] = {role ? d[0] : 0.0, role ? d[1] : 0.0, role ? d[2] : 0.0};      // the d . (D_j n) term exists on the dst side only
    double a3[3][3], cn[3][3];
#pragma unroll
    for (int j = 0; j < 3; ++j) { matvec(gm.D[rot0 + j], v, a3[j]); if (COST != COST_P2P) matvec(gm.D[rot0 + j], n, cn[j]); }
#pragma unroll
    for (int blk = 0; blk < 2; ++blk) {
      const bool plane = blk == 1;
      if (plane && COST == COST_P2P) continue;
      if (!plane && COST == COST_P2PLANE) continue;
      const int nr = plane ? 1 : 3;
      double r[3];
      if (plane) r[0] = d[0] * n2[0] + d[1] * n2[1] + d[2] * n2[2]; else { r[0] = d[0]; r[1] = d[1]; r[2] = d[2]; }
      double s = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) if (i < nr) s += r[i] * r[i];
      double w = 1.0, cst;
      if (robust) { const double arg = 1.0 + s * cc; w = rsqrt(arg); cst = bb * (arg * w - 1.0); } else cst = 0.5 * s;
      w *= live; cst *= live;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        if (i >= nr) continue;
        double Jm[6], Jo[6];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const double* cj = gm.c[tra0 + j];
          if (plane) {
            Jm[j] = sgn * (n2[0] * a3[j][0] + n2[1] * a3[j][1] + n2[2] * a3[j][2]) + (dk[0] * cn[j][0] + dk[1] * cn[j][1] + dk[2] * cn[j][2]);
            Jm[3 + j] = sgn * (n2[0] * cj[0] + n2[1] * cj[1] + n2[2] * cj[2]);
          } else { Jm[j] = sgn * a3[j][i]; Jm[3 + j] = sgn * cj[i]; }
        }
#pragma unroll
        for (int j = 0; j < 6; ++j) Jo[j] = __shfl_xor_sync(0xffffffffu, Jm[j], 1);
        int idx = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) { const double wa = w * Jm[a];
#pragma unroll
          for (int b = a; b < 6; ++b) acc[idx++] += wa * Jm[b]; }
        // (s,k) block: rows 0-2 of it on the even lane, rows 3-5 on the odd lane; X = src-side entries of those rows, Y = the dst side
#pragma unroll
        for (int a = 0; a < 3; ++a) { const double wx = w * (role ? Jo[3 + a] : Jm[a]);
#pragma unroll
          for (int b = 0; b < 6; ++b) acc[21 + 6 * a + b] += wx * (role ? Jm[b] : Jo[b]); }
        const double wr = w * r[i];
#pragma unroll
        for (int a = 0; a < 6; ++a) acc[39 + a] += wr * Jm[a];
      }
      acc[45] += cst;
    }
  }
  // sum over the lanes of equal role (xor 16, 8, 4, 2), then over the warps in order
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < GACC; ++i) {
    double v = acc[i];
#pragma unroll
    for (int o = 16; o > 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane < 2) sred[wid][lane][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 2 * GACC) {
    const int rl = threadIdx.x / GACC, i = threadIdx.x - GACC * rl;
    double v = 0.0;
    for (int w = 0; w < EVAL_THREADS / 32; ++w) v += sred[w][rl][i];
    // (rotation, translation) order -> the parameterisation's tangent order, then the 12x12 upper-triangle layout
    auto real = [&](int a) { return (a + rot0) % 6; };
    int dst = -1;
    if (i < 21) {
      int a = 0, rem = i; while (rem >= 6 - a) { rem -= 6 - a; ++a; }
      const int ra = real(a), rb = real(a + rem);
      dst = u12(6 * rl + min(ra, rb), 6 * rl + max(ra, rb));
    } else if (i < 39) {
      const int a = (i - 21) / 6, b = (i - 21) - 6 * a;
      dst = u12(real(rl ? 3 + a : a), 6 + real(b));
    } else if (i < 45) dst = 78 + 6 * rl + real(i - 39);
    else if (rl == 0) dst = 90;
    if (dst >= 0) partial[(size_t)blockIdx.x * GBLK + dst] = v;
  }
}

// general-path counterpart of lm_edge_kernel: the partials already are the pair matrix in the parameterisation tangent
__global__ void __launch_bounds__(EDGE_THREADS)
lm_edge_general_kernel(const EdgeDev* __restrict__ edges, const int32_t* __restrict__ edge_tile_begin, const double* __restrict__ partial,
                       double* __restrict__ out, DoneGate gate, PeerTable pt, int seq, unsigned int* counter) {
  if (gate.skip(blockIdx.x)) return;
  const int e = blockIdx.x, tid = threadIdx.x;
  __shared__ double blk[GBLK];
  double* o = out + (size_t)EOUT_ * e;
  if (!edges[e].owned) {
    if (pt.world <= 1) for (int i = tid; i < EOUT_; i += EDGE_THREADS) o[i] = 0.0;
    edge_signal(pt, seq, counter);
    return;
  }
  for (int j = tid; j < 91; j += EDGE_THREADS) {
    double v = 0.0;
    for (int t = edge_tile_begin[e]; t < edge_tile_begin[e + 1]; ++t) v += partial[(size_t)t * GBLK + j];
    blk[j] = v;
  }
  __syncthreads();
  for (int r = tid; r < 160; r += EDGE_THREADS) {
    if (r < 144) { const int a = r / 12, b = r - 12 * a; edge_publish(pt, e, r, blk[u12(min(a, b), max(a, b))], o); }
    else if (r < 156) edge_publish(pt, e, r, blk[78 + (r - 144)], o);
    else if (r == 156) edge_publish(pt, e, r, blk[90], o);
    else o[r] = 0.0;
  }
  edge_signal(pt, seq, counter);
}

}  // namespace mv
