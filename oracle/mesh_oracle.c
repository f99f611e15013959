/* oracle/mesh_oracle.c — CPU restatement of the body render (goliath_b200/csrc/mesh_raster.cu), TEST ONLY.
 *
 * Restates drtk's rasterize / render / interpolate, the grid_sample of ca_code/utils/render_drtk.py:45-63 and the
 * project's formulation of drtk's edge_grad_estimator (render_drtk.py:65-72).  drtk is outside the reference tree:
 * PARITY UNPINNED (DESIGN.md R9'').  Conventions, as in include/goliath_b200.h: pixel (x, y) samples (x + 0.5,
 * y + 0.5); a face is drawn if its three z > 0 and its screen area is non-zero; inclusive inside test for either
 * winding; perspective-correct barycentrics; per pixel the smallest (depth, face id).
 *
 *   orc_mesh_raster      fp32, the same expressions in the same order as the kernel (built with -ffp-contract=off),
 *                        so the index image is bit-exact; brute force over every face's pixel box.
 *   orc_mesh_render_fwd  fp64 depth, barycentrics, vt_img, mask and render at a given index image.
 *   orc_mesh_render_bwd  fp64 gradients of sum(g_render * render) with respect to v_pix (interior term, and the edge
 *                        term when edge_grad != 0) and tex, at a given index image.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PIX_OFF 0.5

/* ------------------------------------------------------------------ rasteriser (fp32, bit-exact) */

static float edge_f(float ax, float ay, float bx, float by, float px, float py) {
  return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}

void orc_mesh_raster(int B, int V, int F, int H, int W, const float* v_pix, const int32_t* vi, int32_t* index_img) {
  const size_t HW = (size_t)H * W;
  uint64_t* zb = (uint64_t*)malloc(sizeof(uint64_t) * (HW ? HW : 1));
  for (int b = 0; b < B; ++b) {
    for (size_t i = 0; i < HW; ++i) zb[i] = ~(uint64_t)0;
    const float* vp = v_pix + (size_t)b * V * 3;
    for (int f = 0; f < F; ++f) {
      float x[3], y[3], z[3];
      int ok = 1;
      for (int k = 0; k < 3; ++k) {
        const int v = vi[3 * f + k];
        x[k] = vp[3 * v];
        y[k] = vp[3 * v + 1];
        z[k] = vp[3 * v + 2];
        if (!(z[k] > 0.f) || !isfinite(x[k]) || !isfinite(y[k]) || !isfinite(z[k])) ok = 0;
      }
      if (!ok) continue;
      const float area = edge_f(x[0], y[0], x[1], y[1], x[2], y[2]);
      if (!(area != 0.f && isfinite(area))) continue;
      const float xmin = fminf(fminf(x[0], x[1]), x[2]), xmax = fmaxf(fmaxf(x[0], x[1]), x[2]);
      const float ymin = fminf(fminf(y[0], y[1]), y[2]), ymax = fmaxf(fmaxf(y[0], y[1]), y[2]);
      const float fx0 = fmaxf(ceilf(xmin - 0.5f), 0.f), fx1 = fminf(floorf(xmax - 0.5f), (float)(W - 1));
      const float fy0 = fmaxf(ceilf(ymin - 0.5f), 0.f), fy1 = fminf(floorf(ymax - 0.5f), (float)(H - 1));
      if (!(fx0 <= fx1) || !(fy0 <= fy1)) continue;
      for (int py = (int)fy0; py <= (int)fy1; ++py)
        for (int px = (int)fx0; px <= (int)fx1; ++px) {
          const float sx = (float)px + 0.5f, sy = (float)py + 0.5f;
          float l[3], q[3];
          l[0] = edge_f(x[1], y[1], x[2], y[2], sx, sy) / area;
          l[1] = edge_f(x[2], y[2], x[0], y[0], sx, sy) / area;
          l[2] = edge_f(x[0], y[0], x[1], y[1], sx, sy) / area;
          if (!(l[0] >= 0.f && l[1] >= 0.f && l[2] >= 0.f)) continue;
          q[0] = l[0] / z[0];
          q[1] = l[1] / z[1];
          q[2] = l[2] / z[2];
          const float depth = 1.f / (q[0] + q[1] + q[2]);
          uint32_t bits;
          memcpy(&bits, &depth, 4);
          const uint64_t key = ((uint64_t)bits << 32) | (uint32_t)f;
          uint64_t* d = zb + (size_t)py * W + px;
          if (key < *d) *d = key;
        }
    }
    for (size_t i = 0; i < HW; ++i)
      index_img[(size_t)b * HW + i] = zb[i] == ~(uint64_t)0 ? -1 : (int32_t)(uint32_t)(zb[i] & 0xffffffffu);
  }
  free(zb);
}

/* ------------------------------------------------------------------ fp64 render and gradients */

typedef struct {
  double x[3], y[3], z[3], area;
} Tri;

static double edge_d(double ax, double ay, double bx, double by, double px, double py) {
  return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}

static Tri tri(const float* vp, const int32_t* vi, int f) {
  Tri t;
  for (int k = 0; k < 3; ++k) {
    const int v = vi[3 * f + k];
    t.x[k] = vp[3 * v];
    t.y[k] = vp[3 * v + 1];
    t.z[k] = vp[3 * v + 2];
  }
  t.area = edge_d(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
  return t;
}

static void bary_d(const Tri* t, double px, double py, double l[3]) {
  l[0] = edge_d(t->x[1], t->y[1], t->x[2], t->y[2], px, py) / t->area;
  l[1] = edge_d(t->x[2], t->y[2], t->x[0], t->y[0], px, py) / t->area;
  l[2] = edge_d(t->x[0], t->y[0], t->x[1], t->y[1], px, py) / t->area;
}

static int inside_d(const double l[3]) { return l[0] >= 0 && l[1] >= 0 && l[2] >= 0; }

typedef struct {
  double l[3], q[3], zi, b[3], u[3], v[3], U, V, ix, iy, wx0, wx1, wy0, wy1;
  int x0, y0;
} PixelEval;

static void eval_pixel(const Tri* t, const int32_t* vti, const float* vt, int f, int x, int y, int Ht, int Wt,
                       PixelEval* e) {
  bary_d(t, x + PIX_OFF, y + PIX_OFF, e->l);
  e->zi = 0;
  for (int k = 0; k < 3; ++k) {
    e->q[k] = e->l[k] / t->z[k];
    e->zi += e->q[k];
  }
  e->U = e->V = 0;
  for (int k = 0; k < 3; ++k) {
    e->b[k] = e->q[k] / e->zi;
    const int j = vti[3 * f + k];
    e->u[k] = 2.0 * vt[2 * j] - 1.0;
    e->v[k] = 2.0 * vt[2 * j + 1] - 1.0;
    e->U += e->b[k] * e->u[k];
    e->V += e->b[k] * e->v[k];
  }
  e->ix = ((e->U + 1.0) * Wt - 1.0) / 2.0;
  e->iy = ((e->V + 1.0) * Ht - 1.0) / 2.0;
  e->x0 = (int)floor(e->ix);
  e->y0 = (int)floor(e->iy);
  e->wx1 = e->ix - e->x0;
  e->wx0 = 1.0 - e->wx1;
  e->wy1 = e->iy - e->y0;
  e->wy0 = 1.0 - e->wy1;
}

static double texel(const float* tc, int Ht, int Wt, int x, int y) {
  return (x >= 0 && x < Wt && y >= 0 && y < Ht) ? (double)tc[(size_t)y * Wt + x] : 0.0;
}

static double sample(const float* tc, int Ht, int Wt, const PixelEval* e) {
  return e->wy0 * (e->wx0 * texel(tc, Ht, Wt, e->x0, e->y0) + e->wx1 * texel(tc, Ht, Wt, e->x0 + 1, e->y0)) +
         e->wy1 * (e->wx0 * texel(tc, Ht, Wt, e->x0, e->y0 + 1) + e->wx1 * texel(tc, Ht, Wt, e->x0 + 1, e->y0 + 1));
}

void orc_mesh_render_fwd(int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* v_pix,
                         const int32_t* vi, const int32_t* vti, const float* vt, const float* tex,
                         const int32_t* index_img, double* depth, double* bary, double* vt_img, double* mask,
                         double* render) {
  (void)F;
  const size_t HW = (size_t)H * W, tHW = (size_t)Ht * Wt;
  for (int b = 0; b < B; ++b)
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const size_t p = (size_t)y * W + x, i = (size_t)b * HW + p;
        const int f = index_img[i];
        if (f < 0) {
          depth[i] = mask[i] = 0;
          for (int k = 0; k < 3; ++k) bary[((size_t)b * 3 + k) * HW + p] = 0;
          for (int k = 0; k < 2; ++k) vt_img[((size_t)b * 2 + k) * HW + p] = 0;
          for (int c = 0; c < C; ++c) render[((size_t)b * C + c) * HW + p] = 0;
          continue;
        }
        const Tri t = tri(v_pix + (size_t)b * V * 3, vi, f);
        PixelEval e;
        eval_pixel(&t, vti, vt, f, x, y, Ht, Wt, &e);
        depth[i] = 1.0 / e.zi;
        mask[i] = 1;
        for (int k = 0; k < 3; ++k) bary[((size_t)b * 3 + k) * HW + p] = e.b[k];
        vt_img[(size_t)b * 2 * HW + p] = e.U;
        vt_img[((size_t)b * 2 + 1) * HW + p] = e.V;
        for (int c = 0; c < C; ++c)
          render[((size_t)b * C + c) * HW + p] = sample(tex + ((size_t)b * C + c) * tHW, Ht, Wt, &e);
      }
}

/* gradient of edge_d(v_a, v_b, p) with respect to v_a, v_b (p fixed), times g, added to gv [3 vertices][3] */
static void edge_bwd_d(const Tri* t, int a, int b, double px, double py, double g, double gv[3][3]) {
  gv[a][0] += g * (t->y[b] - py);
  gv[a][1] += g * (px - t->x[b]);
  gv[b][0] += g * (py - t->y[a]);
  gv[b][1] -= g * (px - t->x[a]);
}

static int share_edge(const int32_t* vi, int f, int g) {
  int n = 0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) n += vi[3 * f + a] == vi[3 * g + b];
  return n >= 2;
}

void orc_mesh_render_bwd(int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* v_pix,
                         const int32_t* vi, const int32_t* vti, const float* vt, const float* tex,
                         const int32_t* index_img, const float* g_render, int edge_grad, double* g_v_pix,
                         double* g_tex) {
  (void)F;
  const size_t HW = (size_t)H * W, tHW = (size_t)Ht * Wt;
  memset(g_v_pix, 0, sizeof(double) * (size_t)B * V * 3);
  memset(g_tex, 0, sizeof(double) * (size_t)B * C * tHW);
  /* the fp64 render, for the edge term's colour differences */
  double* img = (double*)calloc((size_t)B * C * HW + 1, sizeof(double));
  for (int b = 0; b < B; ++b)
    for (size_t p = 0; p < HW; ++p) {
      const int f = index_img[(size_t)b * HW + p];
      if (f < 0) continue;
      const Tri t = tri(v_pix + (size_t)b * V * 3, vi, f);
      PixelEval e;
      eval_pixel(&t, vti, vt, f, (int)(p % W), (int)(p / W), Ht, Wt, &e);
      for (int c = 0; c < C; ++c)
        img[((size_t)b * C + c) * HW + p] = sample(tex + ((size_t)b * C + c) * tHW, Ht, Wt, &e);
    }
  for (int b = 0; b < B; ++b) {
    const float* vp = v_pix + (size_t)b * V * 3;
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const size_t p = (size_t)y * W + x;
        const int f = index_img[(size_t)b * HW + p];
        if (f < 0) continue;
        const Tri t = tri(vp, vi, f);
        PixelEval e;
        eval_pixel(&t, vti, vt, f, x, y, Ht, Wt, &e);
        const double px = x + PIX_OFF, py = y + PIX_OFF;
        double gv[3][3] = {{0}};
        /* interior: texture taps and d render / d (ix, iy) */
        double gix = 0, giy = 0;
        for (int c = 0; c < C; ++c) {
          const float* tc = tex + ((size_t)b * C + c) * tHW;
          const double g = g_render[((size_t)b * C + c) * HW + p];
          const double t00 = texel(tc, Ht, Wt, e.x0, e.y0), t01 = texel(tc, Ht, Wt, e.x0 + 1, e.y0);
          const double t10 = texel(tc, Ht, Wt, e.x0, e.y0 + 1), t11 = texel(tc, Ht, Wt, e.x0 + 1, e.y0 + 1);
          gix += g * (e.wy0 * (t01 - t00) + e.wy1 * (t11 - t10));
          giy += g * (e.wx0 * (t10 - t00) + e.wx1 * (t11 - t01));
          const int xs[4] = {e.x0, e.x0 + 1, e.x0, e.x0 + 1}, ys[4] = {e.y0, e.y0, e.y0 + 1, e.y0 + 1};
          const double ws[4] = {e.wy0 * e.wx0, e.wy0 * e.wx1, e.wy1 * e.wx0, e.wy1 * e.wx1};
          for (int d = 0; d < 4; ++d)
            if (xs[d] >= 0 && xs[d] < Wt && ys[d] >= 0 && ys[d] < Ht)
              g_tex[((size_t)b * C + c) * tHW + (size_t)ys[d] * Wt + xs[d]] += g * ws[d];
        }
        const double gU = gix * Wt / 2.0, gV = giy * Ht / 2.0;
        double gb[3], sb = 0, gA = 0, gw[3];
        for (int k = 0; k < 3; ++k) {
          gb[k] = gU * e.u[k] + gV * e.v[k];
          sb += gb[k] * e.b[k];
        }
        for (int k = 0; k < 3; ++k) {
          const double gq = (gb[k] - sb) / e.zi, gl = gq / t.z[k];
          gv[k][2] += -gq * e.q[k] / t.z[k];
          gw[k] = gl / t.area;
          gA -= gl * e.l[k] / t.area;
        }
        edge_bwd_d(&t, 1, 2, px, py, gw[0], gv);
        edge_bwd_d(&t, 2, 0, px, py, gw[1], gv);
        edge_bwd_d(&t, 0, 1, px, py, gw[2], gv);
        edge_bwd_d(&t, 0, 1, t.x[2], t.y[2], gA, gv);
        gv[2][0] -= gA * (t.y[1] - t.y[0]);
        gv[2][1] += gA * (t.x[1] - t.x[0]);
        /* edge term: neighbour pairs (p, q) in which this pixel's face occludes */
        for (int nb = 0; edge_grad && nb < 4; ++nb) {
          const int dx = nb == 0 ? 1 : (nb == 2 ? -1 : 0), dy = nb == 1 ? 1 : (nb == 3 ? -1 : 0);
          const int qx = x + dx, qy = y + dy;
          if (qx < 0 || qx >= W || qy < 0 || qy >= H) continue;
          const size_t pq = (size_t)qy * W + qx;
          const int fq = index_img[(size_t)b * HW + pq];
          if (fq == f) continue;
          const double qpx = qx + PIX_OFF, qpy = qy + PIX_OFF;
          double lo[3];
          bary_d(&t, qpx, qpy, lo);
          if (fq >= 0) {
            if (share_edge(vi, f, fq)) continue;
            const Tri tq = tri(vp, vi, fq);
            double lq[3];
            bary_d(&tq, px, py, lq);
            const int in_p = inside_d(lo), in_q = inside_d(lq);
            if (in_p) continue; /* interpenetration, or the other face occludes */
            if (!in_q) {
              bary_d(&tq, qpx, qpy, lq);
              const double dq = 1.0 / (lq[0] / tq.z[0] + lq[1] / tq.z[1] + lq[2] / tq.z[2]);
              const double dp = 1.0 / e.zi;
              if (!(dp < dq || (dp == dq && f < fq))) continue;
            }
          }
          int ks = -1;
          double smin = 0;
          for (int k = 0; k < 3; ++k)
            if (lo[k] < 0) {
              const double sk = e.l[k] / (e.l[k] - lo[k]);
              if (ks < 0 || sk < smin) {
                ks = k;
                smin = sk;
              }
            }
          if (ks < 0) continue;
          double dLds = 0;
          for (int c = 0; c < C; ++c) {
            const size_t o = ((size_t)b * C + c) * HW;
            dLds += ((double)g_render[o + p] + g_render[o + pq]) * (img[o + p] - img[o + pq]);
          }
          dLds *= 0.5;
          const int a = (ks + 1) % 3, ee = (ks + 2) % 3;
          const double ex = fabs(t.x[ee] - t.x[a]), ey = fabs(t.y[ee] - t.y[a]);
          const double wgt = (dx != 0 ? ey : ex) / (ex + ey);
          const double wo = edge_d(t.x[a], t.y[a], t.x[ee], t.y[ee], px, py);
          const double wt = edge_d(t.x[a], t.y[a], t.x[ee], t.y[ee], qpx, qpy);
          const double den = wo - wt, gs = wgt * dLds / (den * den);
          edge_bwd_d(&t, a, ee, px, py, -gs * wt, gv);
          edge_bwd_d(&t, a, ee, qpx, qpy, gs * wo, gv);
        }
        for (int k = 0; k < 3; ++k)
          for (int d = 0; d < 3; ++d) g_v_pix[((size_t)b * V + vi[3 * f + k]) * 3 + d] += gv[k][d];
      }
  }
  free(img);
}
