// goliath_b200/csrc/mvp_prims.cu — the two glue stages between the hand-MVP decoders and the raymarcher (sm_90a):
//
//  1. slab -> primitive templates.  The reference turns the decoders' UV slabs into the raymarcher's template with
//     five full-size passes: relu(25*rgb+100) (hand_mvp.py:472), relu(alpha) (:434), cat (:172), the
//     view/permute/reshape copy (:172-185, 134 MB per item) and the valid-primitive gather
//     (render_raymarcher.py:44-46).  Here it is one kernel: read 4 floats per voxel from the NCHW slabs, apply the
//     output activations, write the float4 texel of the (compacted) primitive.  Backward is the mirrored scatter.
//
//  2. primitive transforms.  TransDecoder's head scaling (hand_mvp.py:317-321) and GeomDecoder's composition with
//     the mesh-attached base frame (hand_mvp.py:410-425: base + R_base*dpos, R_base*axisangle(drvec), 512*dscale)
//     are ~35 tiny PyTorch kernels over [B,4096,3]; here one kernel forward, one backward.
#include "common.cuh"

namespace {

struct SlabGeom {
  int B, PZ, U, PSX, PSY, NPX, NPY, Kout;
};

// thread = one (b, z, Y, X) voxel; X fastest so slab reads are coalesced and 16 consecutive lanes write one 256 B row
template <bool BWD>
__global__ void __launch_bounds__(256) slab_prims_kernel(SlabGeom g, const float* __restrict__ rgb /* [B,PZ,3,U,U] */,
                                                         const float* __restrict__ alpha /* [B,PZ,1,U,U] */,
                                                         const int* __restrict__ prim_slot /* [NPY*NPX] or null */,
                                                         float rgb_mul, float rgb_add, int apply_relu,
                                                         float4* __restrict__ tpl /* fwd: out, bwd: grad in */,
                                                         float* __restrict__ g_rgb, float* __restrict__ g_alpha) {
  const long long total = (long long)g.B * g.PZ * g.U * g.U;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % g.U), Y = (int)((i / g.U) % g.U);
  const int z = (int)((i / ((long long)g.U * g.U)) % g.PZ), b = (int)(i / ((long long)g.U * g.U * g.PZ));
  const int ix = X / g.PSX, x = X % g.PSX, iy = Y / g.PSY, y = Y % g.PSY;
  const int prim = iy * g.NPX + ix;
  const int slot = prim_slot ? prim_slot[prim] : prim;
  const size_t plane = (size_t)g.U * g.U, pix = (size_t)Y * g.U + X;
  const size_t o_rgb = ((size_t)(b * g.PZ + z) * 3) * plane + pix, o_a = (size_t)(b * g.PZ + z) * plane + pix;
  const size_t o_t = ((((size_t)b * g.Kout + slot) * g.PZ + z) * g.PSY + y) * g.PSX + x;
  if (!BWD) {
    if (slot < 0) return;
    // separate multiply and add (no FMA contraction): the reference's `25.0 * rgb + 100.0` is two rounded ops
    float r = __fadd_rn(__fmul_rn(rgb[o_rgb], rgb_mul), rgb_add);
    float gg = __fadd_rn(__fmul_rn(rgb[o_rgb + plane], rgb_mul), rgb_add);
    float bb = __fadd_rn(__fmul_rn(rgb[o_rgb + 2 * plane], rgb_mul), rgb_add), a = alpha[o_a];
    if (apply_relu) { r = fmaxf(r, 0.f); gg = fmaxf(gg, 0.f); bb = fmaxf(bb, 0.f); a = fmaxf(a, 0.f); }
    tpl[o_t] = make_float4(r, gg, bb, a);
  } else {
    float4 gt = make_float4(0.f, 0.f, 0.f, 0.f);
    if (slot >= 0) gt = tpl[o_t];
    float gr = gt.x * rgb_mul, ggg = gt.y * rgb_mul, gbb = gt.z * rgb_mul, ga = gt.w;
    if (apply_relu) {
      if (!(__fadd_rn(__fmul_rn(rgb[o_rgb], rgb_mul), rgb_add) > 0.f)) gr = 0.f;
      if (!(__fadd_rn(__fmul_rn(rgb[o_rgb + plane], rgb_mul), rgb_add) > 0.f)) ggg = 0.f;
      if (!(__fadd_rn(__fmul_rn(rgb[o_rgb + 2 * plane], rgb_mul), rgb_add) > 0.f)) gbb = 0.f;
      if (!(alpha[o_a] > 0.f)) ga = 0.f;
    }
    g_rgb[o_rgb] = gr; g_rgb[o_rgb + plane] = ggg; g_rgb[o_rgb + 2 * plane] = gbb;
    g_alpha[o_a] = ga;
  }
}

// ---------------------------------------------------------------------------------------------------------------
struct Rot {
  float a[9];
};
__device__ __forceinline__ Rot axisangle(float r0, float r1, float r2, float& theta, float& c, float& s) {
  theta = sqrtf(1e-5f + (r0 * r0 + r1 * r1 + r2 * r2));  // hand_mvp.py:478
  const float u0 = r0 / theta, u1 = r1 / theta, u2 = r2 / theta;
  c = cosf(theta); s = sinf(theta);
  Rot R;
  R.a[0] = u0 * u0 + (1.f - u0 * u0) * c; R.a[1] = u0 * u1 * (1.f - c) - u2 * s; R.a[2] = u0 * u2 * (1.f - c) + u1 * s;
  R.a[3] = u0 * u1 * (1.f - c) + u2 * s; R.a[4] = u1 * u1 + (1.f - u1 * u1) * c; R.a[5] = u1 * u2 * (1.f - c) - u0 * s;
  R.a[6] = u0 * u2 * (1.f - c) - u1 * s; R.a[7] = u1 * u2 * (1.f - c) + u0 * s; R.a[8] = u2 * u2 + (1.f - u2 * u2) * c;
  return R;
}

constexpr float kPosMul = 1.0e-4f, kRvecMul = 0.01f, kScaleMul = 0.01f;  // hand_mvp.py:318-320

template <bool BWD>
__global__ void __launch_bounds__(128) prim_transform_kernel(int B, int K, const float* __restrict__ dec /* [B,9,K] */,
                                                             const float* __restrict__ posbase /* [B,K,3] */,
                                                             const float* __restrict__ rotbase /* [B,K,3,3] */,
                                                             float prim_scale, int zero_delta, float* primpos,
                                                             float* primrot, float* primscale,
                                                             float* __restrict__ g_dec /* [B,9,K] (bwd) */) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  const int b = i / K, k = i % K;
  float d[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) d[c] = dec[((size_t)b * 9 + c) * K + k];
  float Rb[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) Rb[c] = rotbase[(size_t)i * 9 + c];
  float p0 = d[0] * kPosMul, p1 = d[1] * kPosMul, p2 = d[2] * kPosMul;
  float r0 = d[3] * kRvecMul, r1 = d[4] * kRvecMul, r2 = d[5] * kRvecMul;
  float s0 = expf(kScaleMul * d[6]), s1 = expf(kScaleMul * d[7]), s2 = expf(kScaleMul * d[8]);
  if (zero_delta) {  // training warm start, hand_mvp.py:412-415
    p0 = p1 = p2 = 0.f; r0 = r1 = r2 = 0.f; s0 = s1 = s2 = 1.f;
  }
  float theta, c, s;
  const Rot A = axisangle(r0, r1, r2, theta, c, s);
  if (!BWD) {
    primpos[(size_t)i * 3 + 0] = posbase[(size_t)i * 3 + 0] + (Rb[0] * p0 + Rb[1] * p1 + Rb[2] * p2);
    primpos[(size_t)i * 3 + 1] = posbase[(size_t)i * 3 + 1] + (Rb[3] * p0 + Rb[4] * p1 + Rb[5] * p2);
    primpos[(size_t)i * 3 + 2] = posbase[(size_t)i * 3 + 2] + (Rb[6] * p0 + Rb[7] * p1 + Rb[8] * p2);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int cc = 0; cc < 3; ++cc)
        primrot[(size_t)i * 9 + r * 3 + cc] = Rb[r * 3] * A.a[cc] + Rb[r * 3 + 1] * A.a[3 + cc] + Rb[r * 3 + 2] * A.a[6 + cc];
    primscale[(size_t)i * 3 + 0] = prim_scale * s0;
    primscale[(size_t)i * 3 + 1] = prim_scale * s1;
    primscale[(size_t)i * 3 + 2] = prim_scale * s2;
  } else {
    // here primpos / primrot / primscale hold the incoming gradients (any may be null)
    float gd[9];
#pragma unroll
    for (int cc = 0; cc < 9; ++cc) gd[cc] = 0.f;
    if (!zero_delta) {
      if (primpos) {
        const float g0 = primpos[(size_t)i * 3], g1 = primpos[(size_t)i * 3 + 1], g2 = primpos[(size_t)i * 3 + 2];
        gd[0] = kPosMul * (Rb[0] * g0 + Rb[3] * g1 + Rb[6] * g2);
        gd[1] = kPosMul * (Rb[1] * g0 + Rb[4] * g1 + Rb[7] * g2);
        gd[2] = kPosMul * (Rb[2] * g0 + Rb[5] * g1 + Rb[8] * g2);
      }
      if (primscale) {
        gd[6] = primscale[(size_t)i * 3] * prim_scale * s0 * kScaleMul;
        gd[7] = primscale[(size_t)i * 3 + 1] * prim_scale * s1 * kScaleMul;
        gd[8] = primscale[(size_t)i * 3 + 2] * prim_scale * s2 * kScaleMul;
      }
      if (primrot) {
        float G[9], g[9];
#pragma unroll
        for (int cc = 0; cc < 9; ++cc) G[cc] = primrot[(size_t)i * 9 + cc];
#pragma unroll
        for (int r = 0; r < 3; ++r)  // g = Rb^T G
#pragma unroll
          for (int cc = 0; cc < 3; ++cc) g[r * 3 + cc] = Rb[r] * G[cc] + Rb[3 + r] * G[3 + cc] + Rb[6 + r] * G[6 + cc];
        const float u0 = r0 / theta, u1 = r1 / theta, u2 = r2 / theta, omc = 1.f - c;
        const float s01 = g[1] + g[3], s02 = g[2] + g[6], s12 = g[5] + g[7];
        const float dc = g[0] * (1.f - u0 * u0) + g[4] * (1.f - u1 * u1) + g[8] * (1.f - u2 * u2) - s01 * u0 * u1 -
                         s02 * u0 * u2 - s12 * u1 * u2;
        const float ds = u2 * (g[3] - g[1]) + u1 * (g[2] - g[6]) + u0 * (g[7] - g[5]);
        const float du0 = omc * (2.f * g[0] * u0 + s01 * u1 + s02 * u2) + s * (g[7] - g[5]);
        const float du1 = omc * (2.f * g[4] * u1 + s01 * u0 + s12 * u2) + s * (g[2] - g[6]);
        const float du2 = omc * (2.f * g[8] * u2 + s02 * u0 + s12 * u1) + s * (g[3] - g[1]);
        const float dtheta = (c * ds - s * dc) - (du0 * r0 + du1 * r1 + du2 * r2) / (theta * theta);
        gd[3] = kRvecMul * (du0 / theta + dtheta * u0);
        gd[4] = kRvecMul * (du1 / theta + dtheta * u1);
        gd[5] = kRvecMul * (du2 / theta + dtheta * u2);
      }
    }
#pragma unroll
    for (int cc = 0; cc < 9; ++cc) g_dec[((size_t)b * 9 + cc) * K + k] = gd[cc];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// primitive base frames on the posed mesh: make_postex + compute_tbn (geom.py:355-397,515-520) and the texel gather of
// compute_view_cos (geom.py:349-352) through values_to_uv (geom.py:308-324)
struct F3 {
  float x, y, z;
};
__device__ __forceinline__ F3 ld3(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ F3 sub3(F3 a, F3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ F3 cross3(F3 a, F3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
// F.normalize(x, dim=-1): x / max(|x|, 1e-12); an infinite component gives NaN, as in torch
__device__ __forceinline__ F3 normalize3(F3 a) {
  const float d = fmaxf(sqrtf(a.x * a.x + a.y * a.y + a.z * a.z), 1e-12f);
  return {a.x / d, a.y / d, a.z / d};
}
// torch's indexing of a negative index: -1 is the last row
__device__ __forceinline__ int wrap(int i, int n) { return i < 0 ? i + n : i; }

__global__ void __launch_bounds__(128) prim_frames_kernel(int B, int V, int NT, int T, const float* __restrict__ v,
                                                          const int* __restrict__ vidx, const int* __restrict__ vtidx,
                                                          const float* __restrict__ bary, const float* __restrict__ vt,
                                                          const float* __restrict__ vn, const float* __restrict__ campos,
                                                          float* posbase, float* rotbase, float* view_cos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * T) return;
  const int b = i / T, t = i % T;
  const int r0 = vidx[3 * t], r1 = vidx[3 * t + 1], r2 = vidx[3 * t + 2];
  const int i0 = wrap(r0, V), i1 = wrap(r1, V), i2 = wrap(r2, V);
  const float* vb = v + (size_t)b * V * 3;
  const F3 p0 = ld3(vb + 3 * i0), p1 = ld3(vb + 3 * i1), p2 = ld3(vb + 3 * i2);
  const float w0 = bary[3 * t], w1 = bary[3 * t + 1], w2 = bary[3 * t + 2];
  if (posbase) {
    float* o = posbase + (size_t)i * 3;
    o[0] = w0 * p0.x + w1 * p1.x + w2 * p2.x;
    o[1] = w0 * p0.y + w1 * p1.y + w2 * p2.y;
    o[2] = w0 * p0.z + w1 * p1.z + w2 * p2.z;
  }
  if (rotbase) {
    const int j0 = wrap(vtidx[3 * t], NT), j1 = wrap(vtidx[3 * t + 1], NT), j2 = wrap(vtidx[3 * t + 2], NT);
    const float u01 = vt[2 * j1] - vt[2 * j0], w01 = vt[2 * j1 + 1] - vt[2 * j0 + 1];
    const float u02 = vt[2 * j2] - vt[2 * j0], w02 = vt[2 * j2 + 1] - vt[2 * j0 + 1];
    const F3 e01 = sub3(p1, p0), e02 = sub3(p2, p0);
    // no guard on the determinant: a degenerate UV triangle gives inf here and NaN below, as in the reference
    const float f = 1.f / (u01 * w02 - w01 * u02);
    const F3 tg = normalize3({f * (e01.x * w02 - e02.x * w01), f * (e01.y * w02 - e02.y * w01), f * (e01.z * w02 - e02.z * w01)});
    const F3 nm = normalize3(cross3(e01, e02));
    const F3 bt = normalize3(cross3(tg, nm));
    float* R = rotbase + (size_t)i * 9;  // columns T, B, N
    R[0] = tg.x; R[1] = bt.x; R[2] = nm.x;
    R[3] = tg.y; R[4] = bt.y; R[5] = nm.y;
    R[6] = tg.z; R[7] = bt.z; R[8] = nm.z;
  }
  if (view_cos) {
    float c = 0.f;
    if (r0 != -1 && r1 != -1 && r2 != -1) {
      const float* nb = vn + (size_t)b * V * 3;
      const F3 cp = ld3(campos + 3 * b);
      const int id[3] = {i0, i1, i2};
      const F3 p[3] = {p0, p1, p2};
      const float w[3] = {w0, w1, w2};
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const F3 n = normalize3(ld3(nb + 3 * id[k])), d = normalize3(sub3(p[k], cp));
        c += (n.x * d.x + n.y * d.y + n.z * d.z) * w[k];
      }
    }
    view_cos[i] = c;
  }
}

}  // namespace

// hand_mvp.py:172-185 (+ the output activations :434,:472 and the valid-primitive gather render_raymarcher.py:44-46).
// rgb [B,PZ,3,U,U], alpha [B,PZ,1,U,U] (raw decoder outputs when apply_relu / rgb_mul / rgb_add carry the output
// activation, or already-activated tensors with rgb_mul=1, rgb_add=0, apply_relu=0); prim_slot [NPY*NPX] i32 maps a
// primitive to its slot in the output (-1 = dropped) or NULL for identity; tpl [B,Kout,PZ,PSY,PSX,4].
GB_API int gb_mvp_slab_to_prims_fwd(int B, int PZ, int U, int PSX, int PSY, int Kout, const float* rgb,
                                    const float* alpha, const int* prim_slot, float rgb_mul, float rgb_add,
                                    int apply_relu, float* tpl, void* stream) {
  if (B <= 0 || PZ <= 0 || U <= 0) return 0;
  if (PSX <= 0 || PSY <= 0 || U % PSX || U % PSY) return (int)cudaErrorInvalidValue;
  SlabGeom g{B, PZ, U, PSX, PSY, U / PSX, U / PSY, Kout};
  const long long total = (long long)B * PZ * U * U;
  return gb::launch<slab_prims_kernel<false>>((unsigned)gb::cdiv64(total, 256), 256, 0, (cudaStream_t)stream,
      g, rgb, alpha, prim_slot, rgb_mul, rgb_add, apply_relu, reinterpret_cast<float4*>(tpl), nullptr, nullptr);
}

// Backward: g_tpl [B,Kout,PZ,PSY,PSX,4] -> g_rgb [B,PZ,3,U,U], g_alpha [B,PZ,1,U,U] (every element written; dropped
// primitives get zeros).
GB_API int gb_mvp_slab_to_prims_bwd(int B, int PZ, int U, int PSX, int PSY, int Kout, const float* rgb,
                                    const float* alpha, const int* prim_slot, float rgb_mul, float rgb_add,
                                    int apply_relu, const float* g_tpl, float* g_rgb, float* g_alpha, void* stream) {
  if (B <= 0 || PZ <= 0 || U <= 0) return 0;
  if (PSX <= 0 || PSY <= 0 || U % PSX || U % PSY) return (int)cudaErrorInvalidValue;
  SlabGeom g{B, PZ, U, PSX, PSY, U / PSX, U / PSY, Kout};
  const long long total = (long long)B * PZ * U * U;
  return gb::launch<slab_prims_kernel<true>>((unsigned)gb::cdiv64(total, 256), 256, 0, (cudaStream_t)stream,
      g, rgb, alpha, prim_slot, rgb_mul, rgb_add, apply_relu,
      reinterpret_cast<float4*>(const_cast<float*>(g_tpl)), g_rgb, g_alpha);
}

// hand_mvp.py:317-321 + :410-425.  dec [B,9,K] = TransDecoder.dec0 output viewed [B,9,64*64]; posbase [B,K,3],
// rotbase [B,K,3,3]; zero_delta = the `iteration < primposstart` training warm start.
GB_API int gb_mvp_prim_transform_fwd(int B, int K, const float* dec, const float* posbase, const float* rotbase,
                                     float prim_scale, int zero_delta, float* primpos, float* primrot, float* primscale,
                                     void* stream) {
  if (B <= 0 || K <= 0) return 0;
  return gb::launch<prim_transform_kernel<false>>(gb::cdiv(B * K, 128), 128, 0, (cudaStream_t)stream,
      B, K, dec, posbase, rotbase, prim_scale, zero_delta, primpos, primrot, primscale, nullptr);
}

// hand_mvp.py:386-408 (make_postex, compute_tbn) and :230-236 (compute_view_cos + values_to_uv) on the posed mesh.
GB_API int gb_mvp_prim_frames_fwd(int B, int V, int NT, int T, const float* verts, const int32_t* vidx,
                                  const int32_t* vtidx, const float* bary, const float* vt, const float* vn,
                                  const float* campos, float* posbase, float* rotbase, float* view_cos, void* stream) {
  if (B <= 0 || T <= 0) return 0;
  if (V <= 0 || (rotbase && (NT <= 0 || !vtidx || !vt)) || (view_cos && (!vn || !campos)))
    return (int)cudaErrorInvalidValue;
  return gb::launch<prim_frames_kernel>(gb::cdiv(B * T, 128), 128, 0, (cudaStream_t)stream, B, V, NT, T, verts, vidx,
                                        vtidx, bary, vt, vn, campos, posbase, rotbase, view_cos);
}

// g_primpos / g_primrot / g_primscale may be NULL (no gradient arrived); g_dec [B,9,K] is written.
GB_API int gb_mvp_prim_transform_bwd(int B, int K, const float* dec, const float* posbase, const float* rotbase,
                                     float prim_scale, int zero_delta, const float* g_primpos, const float* g_primrot,
                                     const float* g_primscale, float* g_dec, void* stream) {
  if (B <= 0 || K <= 0) return 0;
  return gb::launch<prim_transform_kernel<true>>(gb::cdiv(B * K, 128), 128, 0, (cudaStream_t)stream,
      B, K, dec, posbase, rotbase, prim_scale, zero_delta, const_cast<float*>(g_primpos), const_cast<float*>(g_primrot),
      const_cast<float*>(g_primscale), g_dec);
}
