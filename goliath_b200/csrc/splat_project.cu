// goliath_b200/csrc/splat_project.cu — EWA projection of 3-D Gaussians, forward + backward (sm_90a).
//
// COMPILED WITH -fmad=false AND WITHOUT FAST-MATH: tile binning is a bit-exact contract
// (BASELINE.json north_star), so every fp32 operation here is a single IEEE rounding in a fixed
// order — the same order oracle/splat_oracle.c uses on the CPU.  The kernel is HBM-bound
// (40 B in / 92 B out per Gaussian), so unfused multiplies cost nothing measurable.
//
// Replaces (third-party, absent from the reference tree) gsplat 0.1.11
// project_gaussians_forward_kernel / project_gaussians_backward_kernel as called from
// ca_code/utils/render_gsplat.py:49-63; behaviour restated in SURVEY.md Appendix A.
#include "common.cuh"

namespace {

constexpr int kBlock = 256;

struct M3 { float m[9]; };  // row-major

__device__ __forceinline__ M3 mm3(const M3& a, const M3& b) {
  M3 o;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      o.m[r * 3 + c] = a.m[r * 3 + 0] * b.m[0 * 3 + c] + a.m[r * 3 + 1] * b.m[1 * 3 + c] + a.m[r * 3 + 2] * b.m[2 * 3 + c];
  return o;
}
__device__ __forceinline__ M3 tr3(const M3& a) {
  M3 o;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) o.m[r * 3 + c] = a.m[c * 3 + r];
  return o;
}

__device__ __forceinline__ M3 quat_to_rotmat(float4 q /* (w,x,y,z) in (.x,.y,.z,.w) */) {
  float w = q.x, x = q.y, y = q.z, z = q.w;
  const float n = sqrtf(w * w + x * x + y * y + z * z);
  const float s = 1.0f / n;
  w = w * s; x = x * s; y = y * s; z = z * s;
  M3 R;
  R.m[0] = 1.f - 2.f * (y * y + z * z);
  R.m[1] = 2.f * (x * y - w * z);
  R.m[2] = 2.f * (x * z + w * y);
  R.m[3] = 2.f * (x * y + w * z);
  R.m[4] = 1.f - 2.f * (x * x + z * z);
  R.m[5] = 2.f * (y * z - w * x);
  R.m[6] = 2.f * (x * z - w * y);
  R.m[7] = 2.f * (y * z + w * x);
  R.m[8] = 1.f - 2.f * (x * x + y * y);
  return R;
}

// inclusive-min / exclusive-max tile box; float->int conversion saturates (cvt.rzi)
__device__ __forceinline__ void tile_bbox(float cx, float cy, float radius, int tbx, int tby, int bw, int& x0,
                                          int& y0, int& x1, int& y1) {
  const float fb = (float)bw;
  const float tcx = cx / fb, tcy = cy / fb, tr = radius / fb;
  x0 = min(max(0, __float2int_rz(tcx - tr)), tbx);
  x1 = min(max(0, __float2int_rz(tcx + tr + 1.f)), tbx);
  y0 = min(max(0, __float2int_rz(tcy - tr)), tby);
  y1 = min(max(0, __float2int_rz(tcy + tr + 1.f)), tby);
}

__global__ void __launch_bounds__(kBlock) project_fwd_kernel(
    int G, const float* __restrict__ means3d, const float* __restrict__ scales, float glob_scale,
    const float4* __restrict__ quats, const float* __restrict__ viewmat, float fx, float fy, float cx, float cy,
    int img_h, int img_w, int block_width, float clip_thresh, float* __restrict__ cov3d, float2* __restrict__ xys,
    float* __restrict__ depths, int* __restrict__ radii, float* __restrict__ conics,
    float* __restrict__ compensation, int* __restrict__ num_tiles_hit, float* __restrict__ grad_acc) {
  __shared__ float V[12];
  if (threadIdx.x < 12) V[threadIdx.x] = viewmat[threadIdx.x];
  __syncthreads();
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= G) return;
  const int tbx = (img_w + block_width - 1) / block_width;
  const int tby = (img_h + block_width - 1) / block_width;

  // defaults for culled Gaussians (the reference pre-zeroes its outputs)
  int o_radius = 0, o_tiles = 0;
  float2 o_xy = make_float2(0.f, 0.f);
  float o_depth = 0.f, o_comp = 0.f;
  float o_conic[3] = {0.f, 0.f, 0.f};
  float c3[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};

  const float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];
  const float vx = V[0] * px + V[1] * py + V[2] * pz + V[3];
  const float vy = V[4] * px + V[5] * py + V[6] * pz + V[7];
  const float vz = V[8] * px + V[9] * py + V[10] * pz + V[11];
  if (vz > clip_thresh) {
    const M3 R = quat_to_rotmat(quats[i]);
    const float sx = glob_scale * scales[3 * i], sy = glob_scale * scales[3 * i + 1], sz = glob_scale * scales[3 * i + 2];
    M3 M;
    M.m[0] = R.m[0] * sx; M.m[1] = R.m[1] * sy; M.m[2] = R.m[2] * sz;
    M.m[3] = R.m[3] * sx; M.m[4] = R.m[4] * sy; M.m[5] = R.m[5] * sz;
    M.m[6] = R.m[6] * sx; M.m[7] = R.m[7] * sy; M.m[8] = R.m[8] * sz;
    const M3 S3 = mm3(M, tr3(M));
    c3[0] = S3.m[0]; c3[1] = S3.m[1]; c3[2] = S3.m[2]; c3[3] = S3.m[4]; c3[4] = S3.m[5]; c3[5] = S3.m[8];

    const float tan_fovx = 0.5f * (float)img_w / fx;
    const float tan_fovy = 0.5f * (float)img_h / fy;
    const float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
    const float tz = vz;
    const float tx = tz * fminf(lim_x, fmaxf(-lim_x, vx / tz));
    const float ty = tz * fminf(lim_y, fmaxf(-lim_y, vy / tz));
    const float rz = 1.f / tz, rz2 = rz * rz;
    const float j00 = fx * rz, j02 = -fx * tx * rz2, j11 = fy * rz, j12 = -fy * ty * rz2;
    const float t00 = j00 * V[0] + j02 * V[8], t01 = j00 * V[1] + j02 * V[9], t02 = j00 * V[2] + j02 * V[10];
    const float t10 = j11 * V[4] + j12 * V[8], t11 = j11 * V[5] + j12 * V[9], t12 = j11 * V[6] + j12 * V[10];
    const float a0 = t00 * c3[0] + t01 * c3[1] + t02 * c3[2];
    const float a1 = t00 * c3[1] + t01 * c3[3] + t02 * c3[4];
    const float a2 = t00 * c3[2] + t01 * c3[4] + t02 * c3[5];
    const float b0 = t10 * c3[0] + t11 * c3[1] + t12 * c3[2];
    const float b1 = t10 * c3[1] + t11 * c3[3] + t12 * c3[4];
    const float b2 = t10 * c3[2] + t11 * c3[4] + t12 * c3[5];
    const float c00 = a0 * t00 + a1 * t01 + a2 * t02;
    const float c01 = a0 * t10 + a1 * t11 + a2 * t12;
    const float c11 = b0 * t10 + b1 * t11 + b2 * t12;

    const float det0 = c00 * c11 - c01 * c01;
    const float A = c00 + 0.3f, B = c01, C = c11 + 0.3f;
    const float det1 = A * C - B * B;
    const float comp = sqrtf(fmaxf(0.f, det0 / det1));
    if (det1 != 0.f) {
      const float inv_det = 1.f / det1;
      o_conic[0] = C * inv_det; o_conic[1] = -B * inv_det; o_conic[2] = A * inv_det;
      const float mid = 0.5f * (A + C);
      const float disc = sqrtf(fmaxf(0.1f, mid * mid - det1));
      const float v1 = mid + disc, v2 = mid - disc;
      const float radius = ceilf(3.f * sqrtf(fmaxf(v1, v2)));
      const float rw = 1.f / (vz + 1e-6f);
      const float ctr_x = vx * rw * fx + cx, ctr_y = vy * rw * fy + cy;
      int x0, y0, x1, y1;
      tile_bbox(ctr_x, ctr_y, radius, tbx, tby, block_width, x0, y0, x1, y1);
      const int area = (x1 - x0) * (y1 - y0);
      if (area > 0) {
        o_tiles = area; o_depth = vz; o_radius = __float2int_rz(radius);
        o_xy = make_float2(ctr_x, ctr_y); o_comp = comp;
      }
    }
  }
  radii[i] = o_radius; num_tiles_hit[i] = o_tiles; xys[i] = o_xy; depths[i] = o_depth; compensation[i] = o_comp;
  conics[3 * i] = o_conic[0]; conics[3 * i + 1] = o_conic[1]; conics[3 * i + 2] = o_conic[2];
#pragma unroll
  for (int k = 0; k < 6; ++k) cov3d[6 * i + k] = c3[k];
  if (grad_acc) {  // this Gaussian's row of the blend backward's accumulator (layout: gb_project_gaussians_fwd_acc)
    reinterpret_cast<float4*>(grad_acc)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float2*>(grad_acc + 4 * (size_t)G)[i] = make_float2(0.f, 0.f);
    float* vc = grad_acc + 6 * (size_t)G + 3 * (size_t)i;
    vc[0] = 0.f; vc[1] = 0.f; vc[2] = 0.f;
    grad_acc[9 * (size_t)G + i] = 0.f;
  }
}

// The projection backward of Gaussian i (radii[i] > 0) from the gradients of its xy, depth, conic and compensation, in
// one fixed order of single IEEE roundings; the outputs are zero-initialised by the caller.
__device__ __forceinline__ void project_bwd_one(int i, const float* V, const float* __restrict__ means3d,
                                                const float* __restrict__ scales, float glob_scale,
                                                const float4* __restrict__ quats, float fx, float fy,
                                                const float* __restrict__ cov3d, const float* __restrict__ conics,
                                                const float* __restrict__ compensation, float2 gxy, float vzg,
                                                const float vcon[3], float vcomp, float vm[3], float vc2[3],
                                                float vc3[6], float vsc[3], float4& vq) {
  {
    const float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];
    const float vx = V[0] * px + V[1] * py + V[2] * pz + V[3];
    const float vy = V[4] * px + V[5] * py + V[6] * pz + V[7];
    const float vz = V[8] * px + V[9] * py + V[10] * pz + V[11];
    const float rw = 1.f / (vz + 1e-6f);
    const float vpx = fx * gxy.x, vpy = fy * gxy.y;
    const float gvx = vpx * rw, gvy = vpy * rw, gvz = -(vpx * vx + vpy * vy) * rw * rw;
    vm[0] = V[0] * gvx + V[4] * gvy + V[8] * gvz;
    vm[1] = V[1] * gvx + V[5] * gvy + V[9] * gvz;
    vm[2] = V[2] * gvx + V[6] * gvy + V[10] * gvz;
    vm[0] += V[8] * vzg; vm[1] += V[9] * vzg; vm[2] += V[10] * vzg;

    const float X00 = conics[3 * i], X01 = conics[3 * i + 1], X11 = conics[3 * i + 2];
    const float G00 = vcon[0], G01 = 0.5f * vcon[1], G11 = vcon[2];
    const float xg00 = X00 * G00 + X01 * G01, xg01 = X00 * G01 + X01 * G11;
    const float xg10 = X01 * G00 + X11 * G01, xg11 = X01 * G01 + X11 * G11;
    const float s00 = -(xg00 * X00 + xg01 * X01), s01 = -(xg00 * X01 + xg01 * X11);
    const float s10 = -(xg10 * X00 + xg11 * X01), s11 = -(xg10 * X01 + xg11 * X11);
    vc2[0] = s00; vc2[1] = s01 + s10; vc2[2] = s11;
    {
      const float comp = compensation[i];
      const float inv_det = X00 * X11 - X01 * X01;
      const float omc = 1.f - comp * comp;
      const float vsq = vcomp * 0.5f / (comp + 1e-6f);
      vc2[0] += vsq * (omc * X00 - 0.3f * inv_det);
      vc2[1] += 2.f * vsq * (omc * X01);
      vc2[2] += vsq * (omc * X11 - 0.3f * inv_det);
    }

    const float* c3 = cov3d + 6 * i;
    const float tx = vx, ty = vy, tz = vz;
    const float rz = 1.f / tz, rz2 = rz * rz, rz3 = rz2 * rz;
    M3 W, J, Vm, Gc;
    W.m[0] = V[0]; W.m[1] = V[1]; W.m[2] = V[2]; W.m[3] = V[4]; W.m[4] = V[5]; W.m[5] = V[6];
    W.m[6] = V[8]; W.m[7] = V[9]; W.m[8] = V[10];
    J.m[0] = fx * rz; J.m[1] = 0.f; J.m[2] = -fx * tx * rz2; J.m[3] = 0.f; J.m[4] = fy * rz; J.m[5] = -fy * ty * rz2;
    J.m[6] = 0.f; J.m[7] = 0.f; J.m[8] = 0.f;
    Vm.m[0] = c3[0]; Vm.m[1] = c3[1]; Vm.m[2] = c3[2]; Vm.m[3] = c3[1]; Vm.m[4] = c3[3]; Vm.m[5] = c3[4];
    Vm.m[6] = c3[2]; Vm.m[7] = c3[4]; Vm.m[8] = c3[5];
    Gc.m[0] = vc2[0]; Gc.m[1] = 0.5f * vc2[1]; Gc.m[2] = 0.f; Gc.m[3] = 0.5f * vc2[1]; Gc.m[4] = vc2[2]; Gc.m[5] = 0.f;
    Gc.m[6] = 0.f; Gc.m[7] = 0.f; Gc.m[8] = 0.f;
    const M3 T = mm3(J, W);
    const M3 vV = mm3(mm3(tr3(T), Gc), T);
    const M3 gtv = mm3(mm3(Gc, T), Vm);
    M3 vT;
#pragma unroll
    for (int k = 0; k < 9; ++k) vT.m[k] = gtv.m[k] + gtv.m[k];
    vc3[0] = vV.m[0]; vc3[1] = vV.m[1] + vV.m[3]; vc3[2] = vV.m[2] + vV.m[6];
    vc3[3] = vV.m[4]; vc3[4] = vV.m[5] + vV.m[7]; vc3[5] = vV.m[8];
    const M3 vJ = mm3(vT, tr3(W));
    const float vt0 = -fx * rz2 * vJ.m[2];
    const float vt1 = -fy * rz2 * vJ.m[5];
    const float vt2 = -fx * rz2 * vJ.m[0] + 2.f * fx * tx * rz3 * vJ.m[2] - fy * rz2 * vJ.m[4] + 2.f * fy * ty * rz3 * vJ.m[5];
    vm[0] += vt0 * W.m[0] + vt1 * W.m[3] + vt2 * W.m[6];
    vm[1] += vt0 * W.m[1] + vt1 * W.m[4] + vt2 * W.m[7];
    vm[2] += vt0 * W.m[2] + vt1 * W.m[5] + vt2 * W.m[8];

    M3 vVs;
    vVs.m[0] = vc3[0]; vVs.m[1] = 0.5f * vc3[1]; vVs.m[2] = 0.5f * vc3[2]; vVs.m[3] = 0.5f * vc3[1]; vVs.m[4] = vc3[3];
    vVs.m[5] = 0.5f * vc3[4]; vVs.m[6] = 0.5f * vc3[2]; vVs.m[7] = 0.5f * vc3[4]; vVs.m[8] = vc3[5];
    const float4 q = quats[i];
    const M3 R = quat_to_rotmat(q);
    const float sx = glob_scale * scales[3 * i], sy = glob_scale * scales[3 * i + 1], sz = glob_scale * scales[3 * i + 2];
    M3 Mm;
    Mm.m[0] = R.m[0] * sx; Mm.m[1] = R.m[1] * sy; Mm.m[2] = R.m[2] * sz;
    Mm.m[3] = R.m[3] * sx; Mm.m[4] = R.m[4] * sy; Mm.m[5] = R.m[5] * sz;
    Mm.m[6] = R.m[6] * sx; Mm.m[7] = R.m[7] * sy; Mm.m[8] = R.m[8] * sz;
    M3 vM = mm3(vVs, Mm);
#pragma unroll
    for (int k = 0; k < 9; ++k) vM.m[k] = 2.f * vM.m[k];
    vsc[0] = (R.m[0] * vM.m[0] + R.m[3] * vM.m[3] + R.m[6] * vM.m[6]) * glob_scale;
    vsc[1] = (R.m[1] * vM.m[1] + R.m[4] * vM.m[4] + R.m[7] * vM.m[7]) * glob_scale;
    vsc[2] = (R.m[2] * vM.m[2] + R.m[5] * vM.m[5] + R.m[8] * vM.m[8]) * glob_scale;
    float vR[9];
    vR[0] = vM.m[0] * sx; vR[1] = vM.m[1] * sy; vR[2] = vM.m[2] * sz;
    vR[3] = vM.m[3] * sx; vR[4] = vM.m[4] * sy; vR[5] = vM.m[5] * sz;
    vR[6] = vM.m[6] * sx; vR[7] = vM.m[7] * sy; vR[8] = vM.m[8] * sz;
    const float qn = 1.f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float w = q.x * qn, x = q.y * qn, y = q.z * qn, z = q.w * qn;
#define VR(r, c) vR[(r) * 3 + (c)]
    vq.x = 2.f * (x * (VR(2, 1) - VR(1, 2)) + y * (VR(0, 2) - VR(2, 0)) + z * (VR(1, 0) - VR(0, 1)));
    vq.y = 2.f * (-2.f * x * (VR(1, 1) + VR(2, 2)) + y * (VR(1, 0) + VR(0, 1)) + z * (VR(2, 0) + VR(0, 2)) + w * (VR(2, 1) - VR(1, 2)));
    vq.z = 2.f * (x * (VR(1, 0) + VR(0, 1)) - 2.f * y * (VR(0, 0) + VR(2, 2)) + z * (VR(2, 1) + VR(1, 2)) + w * (VR(0, 2) - VR(2, 0)));
    vq.w = 2.f * (x * (VR(2, 0) + VR(0, 2)) + y * (VR(2, 1) + VR(1, 2)) - 2.f * z * (VR(0, 0) + VR(1, 1)) + w * (VR(1, 0) - VR(0, 1)));
#undef VR
  }
}

__global__ void __launch_bounds__(kBlock) project_bwd_kernel(
    int G, const float* __restrict__ means3d, const float* __restrict__ scales, float glob_scale,
    const float4* __restrict__ quats, const float* __restrict__ viewmat, float fx, float fy,
    const float* __restrict__ cov3d, const int* __restrict__ radii, const float* __restrict__ conics,
    const float* __restrict__ compensation, const float2* __restrict__ v_xy, const float* __restrict__ v_depth,
    const float* __restrict__ v_conic, const float* __restrict__ v_compensation, float* __restrict__ v_cov2d,
    float* __restrict__ v_cov3d, float* __restrict__ v_mean3d, float* __restrict__ v_scale,
    float4* __restrict__ v_quat) {
  __shared__ float V[12];
  if (threadIdx.x < 12) V[threadIdx.x] = viewmat[threadIdx.x];
  __syncthreads();
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= G) return;
  float vm[3] = {0.f, 0.f, 0.f}, vc2[3] = {0.f, 0.f, 0.f}, vsc[3] = {0.f, 0.f, 0.f};
  float vc3[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float4 vq = make_float4(0.f, 0.f, 0.f, 0.f);
  if (radii[i] > 0) {
    project_bwd_one(i, V, means3d, scales, glob_scale, quats, fx, fy, cov3d, conics, compensation, v_xy[i], v_depth[i],
                    v_conic + 3 * i, v_compensation[i], vm, vc2, vc3, vsc, vq);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) { v_cov2d[3 * i + k] = vc2[k]; v_mean3d[3 * i + k] = vm[k]; v_scale[3 * i + k] = vsc[k]; }
#pragma unroll
  for (int k = 0; k < 6; ++k) v_cov3d[6 * i + k] = vc3[k];
  v_quat[i] = vq;
}

// The fused render's per-Gaussian backward in one pass: the blend's accumulator row (layout:
// gb_project_gaussians_fwd_acc) -> the colour and opacity gradients (splat_grad_unpack_kernel's products) and, through
// project_bwd_one, those of the means, scales and rotations.  v_cov2d / v_cov3d are not written.
__global__ void __launch_bounds__(kBlock) splat_project_bwd_kernel(
    int G, const float* __restrict__ means3d, const float* __restrict__ scales, float glob_scale,
    const float4* __restrict__ quats, const float* __restrict__ viewmat, float fx, float fy,
    const float* __restrict__ cov3d, const int* __restrict__ radii, const float* __restrict__ conics,
    const float* __restrict__ compensation, const float* __restrict__ opacity, const float* __restrict__ grad_acc,
    float* __restrict__ v_colors, float* __restrict__ v_opacity, float* __restrict__ v_mean3d,
    float* __restrict__ v_scale, float4* __restrict__ v_quat) {
  __shared__ float V[12];
  if (threadIdx.x < 12) V[threadIdx.x] = viewmat[threadIdx.x];
  __syncthreads();
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= G) return;
  const float4 c4 = reinterpret_cast<const float4*>(grad_acc)[i];  // (v_rgb, v_depth)
  const float e = grad_acc[9 * (size_t)G + i];                     // gradient of opacity * compensation
  v_colors[3 * i] = c4.x; v_colors[3 * i + 1] = c4.y; v_colors[3 * i + 2] = c4.z;
  v_opacity[i] = e * compensation[i];
  float vm[3] = {0.f, 0.f, 0.f}, vc2[3] = {0.f, 0.f, 0.f}, vsc[3] = {0.f, 0.f, 0.f};
  float vc3[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float4 vq = make_float4(0.f, 0.f, 0.f, 0.f);
  if (radii[i] > 0) {
    project_bwd_one(i, V, means3d, scales, glob_scale, quats, fx, fy, cov3d, conics, compensation,
                    reinterpret_cast<const float2*>(grad_acc + 4 * (size_t)G)[i], c4.w,
                    grad_acc + 6 * (size_t)G + 3 * (size_t)i, e * opacity[i], vm, vc2, vc3, vsc, vq);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) { v_mean3d[3 * i + k] = vm[k]; v_scale[3 * i + k] = vsc[k]; }
  v_quat[i] = vq;
}

}  // namespace

// replaces gsplat._C.project_gaussians_forward (call site ca_code/utils/render_gsplat.py:49-63).
// Every output is written for every Gaussian (culled ones get zeros), so the caller need not pre-zero.
GB_API int gb_project_gaussians_fwd(int G, const float* means3d, const float* scales, float glob_scale,
                                    const float* quats, const float* viewmat, float fx, float fy, float cx, float cy,
                                    int img_h, int img_w, int block_width, float clip_thresh, float* cov3d,
                                    float* xys, float* depths, int32_t* radii, float* conics, float* compensation,
                                    int32_t* num_tiles_hit, void* stream) {
  if (G <= 0) return 0;
  if (block_width < 2 || block_width > 16) return (int)cudaErrorInvalidValue;
  return gb::launch<project_fwd_kernel>(gb::cdiv(G, kBlock), kBlock, 0, (cudaStream_t)stream,
      G, means3d, scales, glob_scale, (const float4*)quats, viewmat, fx, fy, cx, cy, img_h, img_w, block_width,
      clip_thresh, cov3d, (float2*)xys, depths, radii, conics, compensation, num_tiles_hit, nullptr);
}

// gb_project_gaussians_fwd that also zeroes grad_acc [10 G] fp32, the accumulator the fused render's blend backward
// adds into: v_rgbd [G,4] | v_xy [G,2] | v_conic [G,3] | v_opacity_eff [G], each part aligned for the blend's vector
// reductions.  gb_splat_project_bwd reads it.
GB_API int gb_project_gaussians_fwd_acc(int G, const float* means3d, const float* scales, float glob_scale,
                                        const float* quats, const float* viewmat, float fx, float fy, float cx,
                                        float cy, int img_h, int img_w, int block_width, float clip_thresh,
                                        float* cov3d, float* xys, float* depths, int32_t* radii, float* conics,
                                        float* compensation, int32_t* num_tiles_hit, float* grad_acc, void* stream) {
  if (G <= 0) return 0;
  if (block_width < 2 || block_width > 16 || !grad_acc) return (int)cudaErrorInvalidValue;
  return gb::launch<project_fwd_kernel>(gb::cdiv(G, kBlock), kBlock, 0, (cudaStream_t)stream,
      G, means3d, scales, glob_scale, (const float4*)quats, viewmat, fx, fy, cx, cy, img_h, img_w, block_width,
      clip_thresh, cov3d, (float2*)xys, depths, radii, conics, compensation, num_tiles_hit, grad_acc);
}

// replaces gsplat._C.project_gaussians_backward (autograd of the call at render_gsplat.py:49-63)
GB_API int gb_project_gaussians_bwd(int G, const float* means3d, const float* scales, float glob_scale,
                                    const float* quats, const float* viewmat, float fx, float fy,
                                    const float* cov3d, const int32_t* radii, const float* conics,
                                    const float* compensation, const float* v_xy, const float* v_depth,
                                    const float* v_conic, const float* v_compensation, float* v_cov2d,
                                    float* v_cov3d, float* v_mean3d, float* v_scale, float* v_quat, void* stream) {
  if (G <= 0) return 0;
  return gb::launch<project_bwd_kernel>(gb::cdiv(G, kBlock), kBlock, 0, (cudaStream_t)stream,
      G, means3d, scales, glob_scale, (const float4*)quats, viewmat, fx, fy, cov3d, radii, conics, compensation,
      (const float2*)v_xy, v_depth, v_conic, v_compensation, v_cov2d, v_cov3d, v_mean3d, v_scale, (float4*)v_quat);
}

// Backward of the fused render per Gaussian, after its blend backward: grad_acc as gb_project_gaussians_fwd_acc left it
// and the blend filled it, opacity [G] and the projection's saved tensors -> v_colors [G,3], v_opacity [G] and
// v_mean3d / v_scale / v_quat, bit for bit gb_splat_grad_unpack followed by gb_project_gaussians_bwd.
GB_API int gb_splat_project_bwd(int G, const float* means3d, const float* scales, float glob_scale, const float* quats,
                                const float* viewmat, float fx, float fy, const float* cov3d, const int32_t* radii,
                                const float* conics, const float* compensation, const float* opacity,
                                const float* grad_acc, float* v_colors, float* v_opacity, float* v_mean3d,
                                float* v_scale, float* v_quat, void* stream) {
  if (G <= 0) return 0;
  return gb::launch<splat_project_bwd_kernel>(gb::cdiv(G, kBlock), kBlock, 0, (cudaStream_t)stream,
      G, means3d, scales, glob_scale, (const float4*)quats, viewmat, fx, fy, cov3d, radii, conics, compensation, opacity,
      grad_acc, v_colors, v_opacity, v_mean3d, v_scale, (float4*)v_quat);
}
