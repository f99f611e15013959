// goliath_b200/csrc/lbs.cu — linear blend skinning of the tracked mesh (sm_90a).
//
// The reference poses the mesh with LBSModule.pose (ca_code/utils/lbs.py:725-731): ParameterTransform (a [7J, P+S]
// matrix-vector product), solve_skeleton_state (a Python loop over the J joints with about a dozen small torch ops
// per joint), states_to_matrix, and a skinning step that materialises mat[:, skin_indices] as [B, V, 8, 3, 4].
// Here:
//   1. skeleton: one CTA per batch item.  A warp per joint computes the joint's seven transformed parameters and its
//      local (t, q, s); the joint chain then runs level by level of the tree (host-computed order, one
//      __syncthreads per level), so its length is the tree's depth, not J; the last pass writes the skinning
//      matrices of states_to_matrix(bind_state, states).  Joint states live in shared memory, which bounds J.
//   2. skin: one thread per (item, vertex): out = gs * sum_k w_k M[idx_k] [v + template; 1], slots in order.
//      Its backward sends the gradient to the vertices only and sums a batch-1 input over B inside the thread, in
//      order, so the result is deterministic.
//   3. unskin (LBSModule.unpose, lbs.py:273-306,733-739): one thread per (item, vertex) blends the same matrices,
//      inverts the blended affine map in registers and applies it; no [B,V,4,4] temporary and no host loop.
// Quaternions are (x, y, z, w), as ca_code/utils/quaternion.py:178-320 (batchMul, batchRot, batchInvert,
// batchFromXYZ) stores them.
#include "common.cuh"

namespace {

constexpr int kMaxJoints = 1024;  // 32 KB of joint states per CTA
constexpr int kSkelThreads = 256;
constexpr int kSlots = 8;          // LinearBlendSkinning's num_max_skin_joints
constexpr int kThreads = 256;

struct Q { float x, y, z, w; };
struct V3 { float x, y, z; };

// batchMul(q, r), quaternion.py:178-249
__device__ __forceinline__ Q qmul(Q q, Q r) {
  return {q.x * r.w + q.y * r.z - q.z * r.y + q.w * r.x,
          -q.x * r.z + q.y * r.w + q.z * r.x + q.w * r.y,
          q.x * r.y - q.y * r.x + q.z * r.w + q.w * r.z,
          -q.x * r.x - q.y * r.y - q.z * r.z + q.w * r.w};
}
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
// batchRot(q, v) = v + 2 (w (a x v) + a x (a x v)), a = q.xyz;  quaternion.py:251-265
__device__ __forceinline__ V3 qrot(Q q, V3 v) {
  const V3 a = {q.x, q.y, q.z};
  const V3 av = cross(a, v), aav = cross(a, av);
  return {v.x + 2.f * (av.x * q.w + aav.x), v.y + 2.f * (av.y * q.w + aav.y), v.z + 2.f * (av.z * q.w + aav.z)};
}
// batchInvert, quaternion.py:267-282
__device__ __forceinline__ Q qinv(Q q) {
  const float r = 1.f / (q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return {-q.x * r, -q.y * r, -q.z * r, q.w * r};
}
// batchFromXYZ, quaternion.py:284-320: half-angles (-x/2, y/2, z/2)
__device__ __forceinline__ Q from_xyz(float rx, float ry, float rz) {
  float s0, c0, s1, c1, s2, c2;
  sincosf(-0.5f * rx, &s0, &c0);
  sincosf(0.5f * ry, &s1, &c1);
  sincosf(0.5f * rz, &s2, &c2);
  return {-s0 * (c1 * c2) - c0 * (s1 * s2), c0 * (s1 * c2) - s0 * (c1 * s2), c0 * (c1 * s2) + s0 * (s1 * c2),
          c0 * (c1 * c2) - s0 * (s1 * s2)};
}

struct SkelArgs {
  int B, J, P, S, scale_stride, n_levels;
  const float *motion, *scale, *transform, *offsets, *joint_offset, *joint_rotation, *bind_state;
  const int32_t *parents, *order, *level_start;
  float *mats, *states;
};

__global__ void __launch_bounds__(kSkelThreads) skeleton_kernel(SkelArgs a) {
  __shared__ float st[kMaxJoints * 8];  // per joint: t[3], q[4], s
  const int b = blockIdx.x, lane = gb::lane_id(), warp = threadIdx.x >> 5, n_warps = kSkelThreads / 32;
  const int PS = a.P + a.S;
  const float* mo = a.motion + (size_t)b * a.P;
  const float* sc = a.scale + (size_t)b * a.scale_stride;

  // ParameterTransform (lbs.py:39-46) + the local transforms of solve_skeleton_state (lbs.py:353-361)
  for (int j = warp; j < a.J; j += n_warps) {
    float jp[7];
#pragma unroll
    for (int c = 0; c < 7; ++c) {
      const float* row = a.transform + (size_t)(7 * j + c) * PS;
      float acc = 0.f;
      for (int k = lane; k < PS; k += 32) acc += row[k] * (k < a.P ? mo[k] : sc[k - a.P]);
      jp[c] = gb::warp_sum(acc) + a.offsets[7 * j + c];
    }
    if (lane == 0) {
      const float* jr = a.joint_rotation + 4 * j;
      const Q lr = qmul({jr[0], jr[1], jr[2], jr[3]}, from_xyz(jp[3], jp[4], jp[5]));
      float* s = st + 8 * j;
      s[0] = jp[0] + a.joint_offset[3 * j];
      s[1] = jp[1] + a.joint_offset[3 * j + 1];
      s[2] = jp[2] + a.joint_offset[3 * j + 2];
      s[3] = lr.x; s[4] = lr.y; s[5] = lr.z; s[6] = lr.w;
      s[7] = exp2f(jp[6]);
    }
  }

  // the joint chain (lbs.py:363-383), one tree level at a time; level 0 holds the roots, which keep their local state
  for (int l = 1; l < a.n_levels; ++l) {
    __syncthreads();
    const int lo = a.level_start[l], hi = a.level_start[l + 1];
    for (int i = lo + threadIdx.x; i < hi; i += kSkelThreads) {
      const int j = a.order[i], p = a.parents[j];
      float* s = st + 8 * j;
      const float* ps = st + 8 * p;
      const Q pq = {ps[3], ps[4], ps[5], ps[6]};
      const float pscale = ps[7];
      const Q gr = qmul(pq, {s[3], s[4], s[5], s[6]});
      const V3 gt = qrot(pq, {s[0] * pscale, s[1] * pscale, s[2] * pscale});
      s[0] = gt.x + ps[0]; s[1] = gt.y + ps[1]; s[2] = gt.z + ps[2];
      s[3] = gr.x; s[4] = gr.y; s[5] = gr.z; s[6] = gr.w;
      s[7] = pscale * s[7];
    }
  }
  __syncthreads();

  // states_to_matrix(bind_state, states), lbs.py:388-426
  for (int j = threadIdx.x; j < a.J; j += kSkelThreads) {
    const float* s = st + 8 * j;
    if (a.states) {
#pragma unroll
      for (int c = 0; c < 8; ++c) a.states[((size_t)b * a.J + j) * 8 + c] = s[c];
    }
    const float* bs_ = a.bind_state + 8 * j;
    const Q br = qinv({bs_[3], bs_[4], bs_[5], bs_[6]});
    const float bs = 1.f / bs_[7];
    const V3 bt0 = qrot(br, {-bs_[0], -bs_[1], -bs_[2]});
    const Q q = {s[3], s[4], s[5], s[6]};
    const Q tr = qmul(q, br);
    const float ts = s[7] * bs;
    const V3 tt0 = qrot(q, {(bt0.x * bs) * s[7], (bt0.y * bs) * s[7], (bt0.z * bs) * s[7]});
    const float tx = tt0.x + s[0], ty = tt0.y + s[1], tz = tt0.z + s[2];
    const float twx = 2.f * tr.x * tr.w, twy = 2.f * tr.y * tr.w, twz = 2.f * tr.z * tr.w;
    const float txx = 2.f * tr.x * tr.x, txy = 2.f * tr.y * tr.x, txz = 2.f * tr.z * tr.x;
    const float tyy = 2.f * tr.y * tr.y, tyz = 2.f * tr.z * tr.y, tzz = 2.f * tr.z * tr.z;
    float* m = a.mats + ((size_t)b * a.J + j) * 12;  // row-major [3, 4]: columns = the three stacked rows, then tt
    m[0] = (1.f - (tyy + tzz)) * ts; m[1] = (txy - twz) * ts;         m[2] = (txz + twy) * ts;         m[3] = tx;
    m[4] = (txy + twz) * ts;         m[5] = (1.f - (txx + tzz)) * ts; m[6] = (tyz - twx) * ts;         m[7] = ty;
    m[8] = (txz - twy) * ts;         m[9] = (tyz + twx) * ts;         m[10] = (1.f - (txx + tyy)) * ts; m[11] = tz;
  }
}

struct SkinArgs {
  int B, V, J, vb;
  const float *mats, *verts, *templ, *w, *gs;
  const int32_t* idx;
};

__global__ void __launch_bounds__(kThreads) skin_fwd_kernel(SkinArgs a, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long long)a.B * a.V) return;
  const int v = (int)(i % a.V), b = (int)(i / a.V);
  const float* x = a.verts + ((size_t)(a.vb == 1 ? 0 : b) * a.V + v) * 3;
  float x0 = x[0], x1 = x[1], x2 = x[2];
  if (a.templ) { x0 += a.templ[3 * v]; x1 += a.templ[3 * v + 1]; x2 += a.templ[3 * v + 2]; }
  float o0 = 0.f, o1 = 0.f, o2 = 0.f;
#pragma unroll
  for (int k = 0; k < kSlots; ++k) {
    const float wk = a.w[(size_t)v * kSlots + k];
    const float* m = a.mats + ((size_t)b * a.J + a.idx[(size_t)v * kSlots + k]) * 12;
    o0 += wk * (m[0] * x0 + m[1] * x1 + m[2] * x2 + m[3]);
    o1 += wk * (m[4] * x0 + m[5] * x1 + m[6] * x2 + m[7]);
    o2 += wk * (m[8] * x0 + m[9] * x1 + m[10] * x2 + m[11]);
  }
  if (a.gs) { o0 *= a.gs[0]; o1 *= a.gs[1]; o2 *= a.gs[2]; }
  float* o = out + (size_t)i * 3;
  o[0] = o0; o[1] = o1; o[2] = o2;
}

// g_v = sum_k w_k M[b, idx_k][:, :3]^T (gs * g); thread = (row of g_verts, vertex); a batch-1 input sums b in order
__global__ void __launch_bounds__(kThreads) skin_bwd_kernel(SkinArgs a, const float* __restrict__ g_out,
                                                            float* __restrict__ g_verts) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long long)a.vb * a.V) return;
  const int v = (int)(i % a.V), r = (int)(i / a.V);
  const int b0 = a.vb == 1 ? 0 : r, b1 = a.vb == 1 ? a.B : r + 1;
  float w[kSlots];
  int id[kSlots];
#pragma unroll
  for (int k = 0; k < kSlots; ++k) { w[k] = a.w[(size_t)v * kSlots + k]; id[k] = a.idx[(size_t)v * kSlots + k]; }
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (int b = b0; b < b1; ++b) {
    const float* g = g_out + ((size_t)b * a.V + v) * 3;
    float g0 = g[0], g1 = g[1], g2 = g[2];
    if (a.gs) { g0 *= a.gs[0]; g1 *= a.gs[1]; g2 *= a.gs[2]; }
#pragma unroll
    for (int k = 0; k < kSlots; ++k) {
      const float* m = a.mats + ((size_t)b * a.J + id[k]) * 12;
      s0 += w[k] * (m[0] * g0 + m[4] * g1 + m[8] * g2);
      s1 += w[k] * (m[1] * g0 + m[5] * g1 + m[9] * g2);
      s2 += w[k] * (m[2] * g0 + m[6] * g1 + m[10] * g2);
    }
  }
  float* o = g_verts + (size_t)i * 3;
  o[0] = s0; o[1] = s1; o[2] = s2;
}

// out = (sum_k w_k M[idx_k])^-1 [verts / gs; 1] - template.  The reference appends the row (0,0,0,1) to the blended
// [3,4] matrix [A | t] and calls inverse() on the 4x4 (lbs.py:293-301); the inverse of such a matrix is
// [A^-1 | -A^-1 t] over the same bottom row, so A^-1 (x - t) is the same result.  A^-1 = adj(A) / det(A).  A blend of
// unrelated joint rotations can be close to singular and x - t cancels, so everything after the loads runs in double
// (a few hundred operations per vertex).  det(A) == 0 gives NaN for that vertex (the reference's inverse() raises).
__global__ void __launch_bounds__(kThreads) unskin_fwd_kernel(SkinArgs a, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long long)a.B * a.V) return;
  const int v = (int)(i % a.V), b = (int)(i / a.V);
  const float* x = a.verts + ((size_t)(a.vb == 1 ? 0 : b) * a.V + v) * 3;
  double x0 = x[0], x1 = x[1], x2 = x[2];
  if (a.gs) { x0 /= (double)a.gs[0]; x1 /= (double)a.gs[1]; x2 /= (double)a.gs[2]; }
  double m[12];
#pragma unroll
  for (int c = 0; c < 12; ++c) m[c] = 0.0;
#pragma unroll
  for (int k = 0; k < kSlots; ++k) {
    const double wk = a.w[(size_t)v * kSlots + k];
    const float* mk = a.mats + ((size_t)b * a.J + a.idx[(size_t)v * kSlots + k]) * 12;
#pragma unroll
    for (int c = 0; c < 12; ++c) m[c] += wk * (double)mk[c];
  }
  const double c00 = m[5] * m[10] - m[6] * m[9], c01 = m[6] * m[8] - m[4] * m[10], c02 = m[4] * m[9] - m[5] * m[8];
  const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  const double d0 = x0 - m[3], d1 = x1 - m[7], d2 = x2 - m[11];
  float o0, o1, o2;
  if (det == 0.0) {
    o0 = o1 = o2 = __int_as_float(0x7fc00000);
  } else {
    const double r = 1.0 / det;
    double u0 = r * (c00 * d0 + (m[2] * m[9] - m[1] * m[10]) * d1 + (m[1] * m[6] - m[2] * m[5]) * d2);
    double u1 = r * (c01 * d0 + (m[0] * m[10] - m[2] * m[8]) * d1 + (m[2] * m[4] - m[0] * m[6]) * d2);
    double u2 = r * (c02 * d0 + (m[1] * m[8] - m[0] * m[9]) * d1 + (m[0] * m[5] - m[1] * m[4]) * d2);
    if (a.templ) { u0 -= (double)a.templ[3 * v]; u1 -= (double)a.templ[3 * v + 1]; u2 -= (double)a.templ[3 * v + 2]; }
    o0 = (float)u0; o1 = (float)u1; o2 = (float)u2;
  }
  float* o = out + (size_t)i * 3;
  o[0] = o0; o[1] = o1; o[2] = o2;
}

}  // namespace

GB_API int gb_lbs_max_joints(void) { return kMaxJoints; }

GB_API int gb_lbs_skeleton_fwd(int B, int J, int P, int S, const float* motion, const float* scale, int scale_stride,
                               const float* transform, const float* transform_offsets, const float* joint_offset,
                               const float* joint_rotation, const int32_t* parents, const int32_t* level_order,
                               const int32_t* level_start, int n_levels, const float* bind_state, float* mats,
                               float* states, void* stream) {
  if (B <= 0 || J <= 0) return 0;
  if (J > kMaxJoints || P < 0 || S < 0 || n_levels < 1 || n_levels > J || scale_stride < 0) return (int)cudaErrorInvalidValue;
  SkelArgs a{B, J, P, S, scale_stride, n_levels, motion, scale, transform, transform_offsets, joint_offset,
             joint_rotation, bind_state, parents, level_order, level_start, mats, states};
  return gb::launch<skeleton_kernel>(B, kSkelThreads, 0, (cudaStream_t)stream, a);
}

GB_API int gb_lbs_skin_fwd(int B, int V, int J, int vb, const float* mats, const float* verts, const float* templ,
                           const int32_t* skin_indices, const float* skin_weights, const float* global_scaling,
                           float* out, void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (J <= 0 || (vb != 1 && vb != B)) return (int)cudaErrorInvalidValue;
  SkinArgs a{B, V, J, vb, mats, verts, templ, skin_weights, global_scaling, skin_indices};
  return gb::launch<skin_fwd_kernel>((unsigned)gb::cdiv64((long long)B * V, kThreads), kThreads, 0,
                                     (cudaStream_t)stream, a, out);
}

GB_API int gb_lbs_skin_bwd(int B, int V, int J, int vb, const float* mats, const int32_t* skin_indices,
                           const float* skin_weights, const float* global_scaling, const float* g_out, float* g_verts,
                           void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (J <= 0 || (vb != 1 && vb != B)) return (int)cudaErrorInvalidValue;
  SkinArgs a{B, V, J, vb, mats, nullptr, nullptr, skin_weights, global_scaling, skin_indices};
  return gb::launch<skin_bwd_kernel>((unsigned)gb::cdiv64((long long)vb * V, kThreads), kThreads, 0,
                                     (cudaStream_t)stream, a, g_out, g_verts);
}

GB_API int gb_lbs_unskin_fwd(int B, int V, int J, int vb, const float* mats, const float* verts, const float* templ,
                             const int32_t* skin_indices, const float* skin_weights, const float* global_scaling,
                             float* out, void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (J <= 0 || (vb != 1 && vb != B)) return (int)cudaErrorInvalidValue;
  SkinArgs a{B, V, J, vb, mats, verts, templ, skin_weights, global_scaling, skin_indices};
  return gb::launch<unskin_fwd_kernel>((unsigned)gb::cdiv64((long long)B * V, kThreads), kThreads, 0,
                                       (cudaStream_t)stream, a, out);
}
