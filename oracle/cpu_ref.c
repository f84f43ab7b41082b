/* cpu_ref.c -- TEST / BENCH INFRASTRUCTURE, not product code (only tests/, bench.py's CPU legs and __graft_entry__.build() touch oracle/).
 *
 * A C + OpenMP restatement of how DL4J 1.0.0-beta3 with the nd4j-native CPU backend (P:104-108 of the reference's Java/pom.xml; the
 * reference's "reference plumbing" configuration) executes the adversarial G+D step of J:408-471: NCHW fp32 activations, every layer
 * op-by-op -- explicit im2col buffer + SGEMM + separate bias / activation / BatchNorm passes, col2im scatter for the transposed
 * convolutions and the input gradients, a multi-pass Adam updater -- on all host cores.  DL4J itself cannot run here (no JVM, no jars:
 * SURVEY.md section 8c), so this is the "DL4J-algorithm CPU baseline (restated)" SURVEY section 8d(i) asks for.  The arithmetic is the
 * NumPy oracle's (oracle/dl4j_oracle.py: Conv2D / Deconv2D / BatchNorm / Dense / xent_score_and_grad / Net.apply_update / gan_step, each
 * of which cites its DL4J source) and tests/test_oracle.py::test_c_reference_matches_numpy_oracle pins it to that oracle.
 *
 * Scope: the layer vocabulary of the DCGAN (C2 / C4) and MLP-GAN (C5) configurations -- conv, transposed conv, batch norm, activation,
 * dense, binary cross-entropy on logits, Adam.  The SGEMM is a packed, cache-blocked, OpenMP-parallel kernel whose micro-kernel is plain C
 * that gcc vectorises per ISA (target_clones: AVX-512 / AVX2 / baseline, picked at load time), standing in for nd4j-native's OpenBLAS.
 *
 * build: gcc -O3 -fopenmp -shared -fPIC -o oracle/_build/libcpuref.so oracle/cpu_ref.c -lm      (oracle/Makefile)
 */
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { L_CONV = 0, L_DECONV = 1, L_BN = 2, L_ACT = 3, L_DENSE = 4 };
enum { A_ID = 0, A_TANH = 1, A_SIGMOID = 2, A_RELU = 3, A_LRELU = 4 };

typedef struct {            /* mirrors the layer specs of gan_deeplearning4j_b200/models.py */
  int32_t type, cin, cout, k, s, p, has_bias, act;
  float alpha;
} cr_layer;

typedef struct {
  cr_layer d;
  int ih, iw, oh, ow;                 /* per-example spatial dims (dense: 1x1) */
  int64_t off_b, off_w, off_gamma;    /* offsets into the flattened parameter vector (DL4J order), -1 if absent */
  float *out, *z, *xhat;              /* activations [N][C][H][W]; pre-activation (layers with a non-identity activation); BN x-hat */
  float *mu, *var, *std;              /* BN batch statistics of the latest forward */
} cr_l;

typedef struct {
  int nl, in_c, in_h, in_w, maxn; cr_l* L; int64_t np;
  float *params, *grads, *m, *v; int iteration;
  float lr, b1, b2, eps;
  float *eps_a, *eps_b, *col; size_t col_floats, act_floats;
} cr_net;

typedef struct { cr_net G, D; float* xfake; float* gsave; } cr_gan;

/* ------------------------------------------------------------------ SGEMM: C[M][N] (+)= op(A)[M][K] * op(B)[K][N] ---------------- */
#define MR 6
#define NR 32
#define KC 256
#define MC 96
#define NC 2048
__attribute__((target_clones("avx512f", "avx2", "default")))
static void micro(int kc, const float* __restrict a /* [kc][MR] */, const float* __restrict b /* [kc][NR] */, float* __restrict c, int ldc, int mr, int nr, int add) {
  float acc[MR][NR];
  for (int i = 0; i < MR; ++i) for (int j = 0; j < NR; ++j) acc[i][j] = 0.f;
  for (int k = 0; k < kc; ++k) {
    const float* bk = b + (size_t)k * NR; const float* ak = a + (size_t)k * MR;
    for (int i = 0; i < MR; ++i) { const float av = ak[i];
#pragma omp simd
      for (int j = 0; j < NR; ++j) acc[i][j] += av * bk[j]; }
  }
  if (add) { for (int i = 0; i < mr; ++i) for (int j = 0; j < nr; ++j) c[(size_t)i * ldc + j] += acc[i][j]; }
  else { for (int i = 0; i < mr; ++i) for (int j = 0; j < nr; ++j) c[(size_t)i * ldc + j] = acc[i][j]; }
}
/* element (i,k) of op(A) = A[i*sa_i + k*sa_k]; likewise B(k,j) */
static void sgemm(int M, int N, int K, const float* A, int64_t sa_i, int64_t sa_k, const float* B, int64_t sb_k, int64_t sb_j, float* C, int ldc, int accumulate) {
  float* Bp = (float*)aligned_alloc(64, sizeof(float) * (size_t)KC * NC);
  const int nth = omp_get_max_threads();
  float* Ap_all = (float*)aligned_alloc(64, sizeof(float) * (size_t)nth * MC * KC);
  for (int jc = 0; jc < N; jc += NC) {
    const int nc = N - jc < NC ? N - jc : NC, npan = (nc + NR - 1) / NR;
    for (int pc = 0; pc < K; pc += KC) {
      const int kc = K - pc < KC ? K - pc : KC;
#pragma omp parallel for schedule(static)
      for (int jp = 0; jp < npan; ++jp) {                       /* pack B into NR-wide panels [kc][NR] */
        float* dst = Bp + (size_t)jp * kc * NR; const int j0 = jc + jp * NR;
        for (int k = 0; k < kc; ++k) for (int j = 0; j < NR; ++j) dst[(size_t)k * NR + j] = (j0 + j < N) ? B[(int64_t)(pc + k) * sb_k + (int64_t)(j0 + j) * sb_j] : 0.f;
      }
      const int mblocks = (M + MC - 1) / MC, jgroups = (npan + 7) / 8;    /* a task = one MC block of rows x 8 column panels */
#pragma omp parallel for collapse(2) schedule(dynamic)
      for (int ib = 0; ib < mblocks; ++ib) for (int jg = 0; jg < jgroups; ++jg) {
        float* Ap = Ap_all + (size_t)omp_get_thread_num() * MC * KC;
        const int i0 = ib * MC, mc = M - i0 < MC ? M - i0 : MC, mpan = (mc + MR - 1) / MR;
        for (int ip = 0; ip < mpan; ++ip) {                       /* pack A into MR-tall panels [kc][MR] */
          float* dst = Ap + (size_t)ip * kc * MR;
          for (int k = 0; k < kc; ++k) for (int i = 0; i < MR; ++i) { const int r = i0 + ip * MR + i; dst[(size_t)k * MR + i] = r < M ? A[(int64_t)r * sa_i + (int64_t)(pc + k) * sa_k] : 0.f; }
        }
        const int jp1 = (jg + 1) * 8 < npan ? (jg + 1) * 8 : npan;
        for (int jp = jg * 8; jp < jp1; ++jp) for (int ip = 0; ip < mpan; ++ip) {
          const int r0 = i0 + ip * MR, c0 = jc + jp * NR;
          micro(kc, Ap + (size_t)ip * kc * MR, Bp + (size_t)jp * kc * NR, C + (size_t)r0 * ldc + c0, ldc, M - r0 < MR ? M - r0 : MR, N - c0 < NR ? N - c0 : NR, accumulate || pc > 0);
        }
      }
    }
  }
  free(Bp); free(Ap_all);
}

/* ------------------------------------------------------------------ im2col / col2im (NCHW, rows = output pixels) ------------------ */
/* cols [N*OH*OW][C*k*k] with column index (c*k + i)*k + j -- the order of DL4J's W.reshape(nOut, nIn*kH*kW) */
static void im2col(const float* x, int N, int C, int H, int W, int k, int s, int p, int OH, int OW, float* cols) {
#pragma omp parallel for collapse(2) schedule(static)
  for (int n = 0; n < N; ++n) for (int oy = 0; oy < OH; ++oy) for (int ox = 0; ox < OW; ++ox) {
    float* row = cols + ((size_t)(n * OH + oy) * OW + ox) * C * k * k;
    for (int c = 0; c < C; ++c) for (int i = 0; i < k; ++i) { const int iy = oy * s - p + i;
      for (int j = 0; j < k; ++j) { const int ix = ox * s - p + j; row[(c * k + i) * k + j] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? x[((size_t)(n * C + c) * H + iy) * W + ix] : 0.f; } }
  }
}
static void col2im(const float* cols, int N, int C, int H, int W, int k, int s, int p, int OH, int OW, float* x) {
#pragma omp parallel for collapse(2) schedule(static)
  for (int n = 0; n < N; ++n) for (int c = 0; c < C; ++c) {
    float* xc = x + (size_t)(n * C + c) * H * W; memset(xc, 0, sizeof(float) * H * W);
    for (int oy = 0; oy < OH; ++oy) for (int ox = 0; ox < OW; ++ox) { const float* row = cols + ((size_t)(n * OH + oy) * OW + ox) * C * k * k + c * k * k;
      for (int i = 0; i < k; ++i) { const int iy = oy * s - p + i; if (iy < 0 || iy >= H) continue;
        for (int j = 0; j < k; ++j) { const int ix = ox * s - p + j; if (ix >= 0 && ix < W) xc[iy * W + ix] += row[i * k + j]; } } }
  }
}
static inline float actf(int a, float z, float al) { switch (a) { case A_TANH: return tanhf(z); case A_SIGMOID: return 1.f / (1.f + expf(-z)); case A_RELU: return z > 0 ? z : 0.f; case A_LRELU: return z > 0 ? z : al * z; } return z; }
static inline float actg(int a, float z, float al) { switch (a) { case A_TANH: { float t = tanhf(z); return 1.f - t * t; } case A_SIGMOID: { float s = 1.f / (1.f + expf(-z)); return s * (1.f - s); } case A_RELU: return z > 0 ? 1.f : 0.f; case A_LRELU: return z > 0 ? 1.f : al; } return 1.f; }

/* ------------------------------------------------------------------ net ------------------------------------------------------------ */
static int net_init(cr_net* n, const cr_layer* ls, int nl, int in_c, int in_h, int in_w, int maxn, float lr, float b1, float b2, float eps) {
  memset(n, 0, sizeof(*n)); n->nl = nl; n->in_c = in_c; n->in_h = in_h; n->in_w = in_w; n->maxn = maxn; n->lr = lr; n->b1 = b1; n->b2 = b2; n->eps = eps;
  n->L = (cr_l*)calloc(nl, sizeof(cr_l));
  int c = in_c, h = in_h, w = in_w; int64_t off = 0; size_t maxact = (size_t)c * h * w, maxcol = 1;
  for (int i = 0; i < nl; ++i) { cr_l* l = &n->L[i]; l->d = ls[i]; l->ih = h; l->iw = w; l->off_b = l->off_w = l->off_gamma = -1; cr_layer* d = &l->d;
    if (d->cin == 0) d->cin = c;
    switch (d->type) {
      case L_CONV: l->oh = (h - d->k + 2 * d->p) / d->s + 1; l->ow = (w - d->k + 2 * d->p) / d->s + 1;
        if (d->has_bias) { l->off_b = off; off += d->cout; } l->off_w = off; off += (int64_t)d->cout * d->cin * d->k * d->k;
        if ((size_t)l->oh * l->ow * d->cin * d->k * d->k > maxcol) { maxcol = (size_t)l->oh * l->ow * d->cin * d->k * d->k; }
        break;
      case L_DECONV: l->oh = d->s * (h - 1) + d->k - 2 * d->p; l->ow = d->s * (w - 1) + d->k - 2 * d->p;
        if (d->has_bias) { l->off_b = off; off += d->cout; } l->off_w = off; off += (int64_t)d->cin * d->cout * d->k * d->k;
        if ((size_t)h * w * d->cout * d->k * d->k > maxcol) { maxcol = (size_t)h * w * d->cout * d->k * d->k; }
        break;
      case L_DENSE: l->oh = l->ow = 1; d->cin = c * h * w; l->off_w = off; off += (int64_t)d->cin * d->cout; if (d->has_bias) { l->off_b = off; off += d->cout; } break;
      case L_BN: d->cout = c; l->oh = h; l->ow = w; l->off_gamma = off; off += 4 * (int64_t)c; break;
      case L_ACT: d->cout = c; l->oh = h; l->ow = w; break;
      default: return -1;
    }
    c = d->cout; h = l->oh; w = l->ow;
    const size_t oe = (size_t)c * h * w; if (oe > maxact) maxact = oe;
    l->out = (float*)malloc(sizeof(float) * maxn * oe);
    if ((d->type == L_CONV || d->type == L_DECONV || d->type == L_DENSE) && d->act != A_ID) l->z = (float*)malloc(sizeof(float) * maxn * oe);
    if (d->type == L_BN) { l->xhat = (float*)malloc(sizeof(float) * maxn * oe); l->mu = (float*)calloc(c, 4); l->var = (float*)calloc(c, 4); l->std = (float*)calloc(c, 4); }
  }
  n->np = off; n->params = (float*)calloc(off, 4); n->grads = (float*)calloc(off, 4); n->m = (float*)calloc(off, 4); n->v = (float*)calloc(off, 4);
  n->act_floats = (size_t)maxn * maxact; n->eps_a = (float*)malloc(4 * n->act_floats); n->eps_b = (float*)malloc(4 * n->act_floats);
  n->col_floats = (size_t)maxn * maxcol; n->col = (float*)malloc(4 * n->col_floats);
  for (int i = 0; i < nl; ++i) if (n->L[i].d.type == L_BN) { float* p = n->params + n->L[i].off_gamma; const int C = n->L[i].d.cout; for (int k = 0; k < C; ++k) { p[k] = 1.f; p[3 * C + k] = 1.f; } }
  return 0;
}
static void net_free(cr_net* n) { for (int i = 0; i < n->nl; ++i) { free(n->L[i].out); free(n->L[i].z); free(n->L[i].xhat); free(n->L[i].mu); free(n->L[i].var); free(n->L[i].std); }
  free(n->L); free(n->params); free(n->grads); free(n->m); free(n->v); free(n->eps_a); free(n->eps_b); free(n->col); }

/* [rows][C] (row = n*HW + p) -> NCHW (+ bias), optionally keeping z and applying the activation: the separate passes DL4J makes */
static void rows_to_nchw_bias_act(const float* rows, int N, int C, int HW, const float* bias, int act, float al, float* z, float* out) {
#pragma omp parallel for collapse(2) schedule(static)
  for (int n = 0; n < N; ++n) for (int c = 0; c < C; ++c) for (int p = 0; p < HW; ++p) {
    const float v = rows[((size_t)n * HW + p) * C + c] + (bias ? bias[c] : 0.f); const size_t o = ((size_t)n * C + c) * HW + p;
    if (z) { z[o] = v; }
    out[o] = actf(act, v, al); }
}
static void nchw_to_rows(const float* x, int N, int C, int HW, float* rows) {
#pragma omp parallel for collapse(2) schedule(static)
  for (int n = 0; n < N; ++n) for (int p = 0; p < HW; ++p) for (int c = 0; c < C; ++c) rows[((size_t)n * HW + p) * C + c] = x[((size_t)n * C + c) * HW + p];
}

static const float* net_forward(cr_net* n, const float* x, int N, int train) {
  const float* cur = x; int c = n->in_c;
  float* tmp = n->eps_a;      /* row-major GEMM result before the NCHW permute */
  for (int i = 0; i < n->nl; ++i) { cr_l* l = &n->L[i]; const cr_layer* d = &l->d; const float* bias = l->off_b >= 0 ? n->params + l->off_b : NULL;
    switch (d->type) {
      case L_CONV: { const int kk = d->cin * d->k * d->k, P = l->oh * l->ow;
        im2col(cur, N, d->cin, l->ih, l->iw, d->k, d->s, d->p, l->oh, l->ow, n->col);
        sgemm(N * P, d->cout, kk, n->col, kk, 1, n->params + l->off_w, 1, kk, tmp, d->cout, 0);           /* cols x W2d^T */
        rows_to_nchw_bias_act(tmp, N, d->cout, P, bias, d->act, d->alpha, l->z, l->out); } break;
      case L_DECONV: { const int P = l->ih * l->iw, kk = d->cout * d->k * d->k;
        nchw_to_rows(cur, N, d->cin, P, tmp);                                                               /* x2d [N*H*W][Cin] */
        sgemm(N * P, kk, d->cin, tmp, d->cin, 1, n->params + l->off_w, kk, 1, n->col, kk, 0);               /* x2d x W[Cin][Cout*k*k] */
        float* zz = l->z ? l->z : l->out;
        col2im(n->col, N, d->cout, l->oh, l->ow, d->k, d->s, d->p, l->ih, l->iw, zz);
        const size_t HW = (size_t)l->oh * l->ow;
#pragma omp parallel for collapse(2) schedule(static)
        for (int b = 0; b < N; ++b) for (int ch = 0; ch < d->cout; ++ch) { float* zp = zz + ((size_t)b * d->cout + ch) * HW; float* op = l->out + ((size_t)b * d->cout + ch) * HW; const float bb = bias ? bias[ch] : 0.f;
          for (size_t p = 0; p < HW; ++p) { const float v = zp[p] + bb; zp[p] = v; op[p] = actf(d->act, v, d->alpha); } } } break;
      case L_DENSE: {   /* W is 'f'-order [nIn][nOut]: element (i,o) at i + nIn*o */
        sgemm(N, d->cout, d->cin, cur, d->cin, 1, n->params + l->off_w, 1, d->cin, tmp, d->cout, 0);
        rows_to_nchw_bias_act(tmp, N, d->cout, 1, bias, d->act, d->alpha, l->z, l->out); } break;
      case L_BN: { const int C = d->cout; const size_t HW = (size_t)l->oh * l->ow; const float* P = n->params + l->off_gamma; const double m = (double)N * HW;
#pragma omp parallel for schedule(static)
        for (int ch = 0; ch < C; ++ch) {
          float mu, var;
          if (train) { double s = 0; for (int b = 0; b < N; ++b) { const float* xp = cur + ((size_t)b * C + ch) * HW; for (size_t p = 0; p < HW; ++p) s += xp[p]; } mu = (float)(s / m);
            double q = 0; for (int b = 0; b < N; ++b) { const float* xp = cur + ((size_t)b * C + ch) * HW; for (size_t p = 0; p < HW; ++p) { const double dlt = xp[p] - mu; q += dlt * dlt; } } var = (float)(q / m);
            l->mu[ch] = mu; l->var[ch] = var; }
          else { mu = P[2 * C + ch]; var = P[3 * C + ch]; }
          const float sd = sqrtf(var + 1e-5f); l->std[ch] = sd; const float g = P[ch], be = P[C + ch];
          for (int b = 0; b < N; ++b) { const float* xp = cur + ((size_t)b * C + ch) * HW; float* hp = l->xhat + ((size_t)b * C + ch) * HW; float* op = l->out + ((size_t)b * C + ch) * HW;
            for (size_t p = 0; p < HW; ++p) { const float xh = (xp[p] - mu) / sd; hp[p] = xh; op[p] = g * xh + be; } }
        } } break;
      case L_ACT: { const size_t tot = (size_t)N * d->cout * l->oh * l->ow;
#pragma omp parallel for schedule(static)
        for (size_t e = 0; e < tot; ++e) l->out[e] = actf(d->act, cur[e], d->alpha); } break;
    }
    cur = l->out; c = d->cout;
  }
  (void)c; return cur;
}

/* eps: gradient w.r.t. the last layer's output [N][...]; leaves summed gradients in n->grads; returns d/d input if want_in */
static const float* net_backward(cr_net* n, const float* x, const float* eps, int N, int want_wgrad, int want_in) {
  float* bufs[2] = {n->eps_a, n->eps_b}; int bi = 0; const float* cur = eps;
  for (int i = n->nl - 1; i >= 0; --i) { cr_l* l = &n->L[i]; const cr_layer* d = &l->d; const float* lin = i == 0 ? x : n->L[i - 1].out;
    const int need_in = want_in || i > 0;
    float* nx = bufs[bi]; if (nx == cur) { bi ^= 1; nx = bufs[bi]; }
    switch (d->type) {
      case L_CONV: case L_DECONV: case L_DENSE: {
        const size_t oe = (size_t)N * d->cout * l->oh * l->ow;
        /* delta = eps * act'(z) (separate pass), then as rows [N*P][Cout] */
        float* dl = (float*)malloc(4 * oe);
#pragma omp parallel for schedule(static)
        for (size_t e = 0; e < oe; ++e) dl[e] = cur[e] * (l->z ? actg(d->act, l->z[e], d->alpha) : 1.f);
        if (d->type == L_CONV) { const int kk = d->cin * d->k * d->k, P = l->oh * l->ow; float* d2d = (float*)malloc(4 * oe);
          nchw_to_rows(dl, N, d->cout, P, d2d);
          if (want_wgrad) { im2col(lin, N, d->cin, l->ih, l->iw, d->k, d->s, d->p, l->oh, l->ow, n->col);
            sgemm(d->cout, kk, N * P, d2d, 1, d->cout, n->col, kk, 1, n->grads + l->off_w, kk, 0);       /* d2d^T x cols */
            if (l->off_b >= 0) { float* gb = n->grads + l->off_b;
#pragma omp parallel for schedule(static)
              for (int o = 0; o < d->cout; ++o) { double s = 0; for (size_t r = 0; r < (size_t)N * P; ++r) s += d2d[r * d->cout + o]; gb[o] = (float)s; } } }
          if (need_in) { sgemm(N * P, kk, d->cout, d2d, d->cout, 1, n->params + l->off_w, kk, 1, n->col, kk, 0);    /* d2d x W2d */
            col2im(n->col, N, d->cin, l->ih, l->iw, d->k, d->s, d->p, l->oh, l->ow, nx); }
          free(d2d);
        } else if (d->type == L_DECONV) { const int P = l->ih * l->iw, kk = d->cout * d->k * d->k;
          im2col(dl, N, d->cout, l->oh, l->ow, d->k, d->s, d->p, l->ih, l->iw, n->col);                   /* dcols [N*H*W][Cout*k*k] */
          if (want_wgrad) { float* x2d = (float*)malloc(4 * (size_t)N * P * d->cin); nchw_to_rows(lin, N, d->cin, P, x2d);
            sgemm(d->cin, kk, N * P, x2d, 1, d->cin, n->col, kk, 1, n->grads + l->off_w, kk, 0); free(x2d);
            if (l->off_b >= 0) { float* gb = n->grads + l->off_b; const size_t HW = (size_t)l->oh * l->ow;
#pragma omp parallel for schedule(static)
              for (int o = 0; o < d->cout; ++o) { double s = 0; for (int b = 0; b < N; ++b) { const float* p = dl + ((size_t)b * d->cout + o) * HW; for (size_t q = 0; q < HW; ++q) s += p[q]; } gb[o] = (float)s; } } }
          if (need_in) { float* r = (float*)malloc(4 * (size_t)N * P * d->cin);
            sgemm(N * P, d->cin, kk, n->col, kk, 1, n->params + l->off_w, 1, kk, r, d->cin, 0);                /* dcols x W2d^T */
            rows_to_nchw_bias_act(r, N, d->cin, P, NULL, A_ID, 0.f, NULL, nx); free(r); }
        } else {
          if (want_wgrad) { /* dW (f-order [nIn][nOut]) = x^T delta: element (i,o) at i + nIn*o  ->  C[o][i] row-major */
            sgemm(d->cout, d->cin, N, dl, 1, d->cout, lin, d->cin, 1, n->grads + l->off_w, d->cin, 0);
            if (l->off_b >= 0) { float* gb = n->grads + l->off_b; for (int o = 0; o < d->cout; ++o) { double s = 0; for (int b = 0; b < N; ++b) s += dl[(size_t)b * d->cout + o]; gb[o] = (float)s; } } }
          if (need_in) sgemm(N, d->cin, d->cout, dl, d->cout, 1, n->params + l->off_w, d->cin, 1, nx, d->cin, 0);    /* delta x W^T */
        }
        free(dl);
      } break;
      case L_BN: { const int C = d->cout; const size_t HW = (size_t)l->oh * l->ow; const float* P = n->params + l->off_gamma; float* G = n->grads + l->off_gamma; const double m = (double)N * HW;
#pragma omp parallel for schedule(static)
        for (int ch = 0; ch < C; ++ch) { double sb = 0, sg = 0;
          for (int b = 0; b < N; ++b) { const float* ep = cur + ((size_t)b * C + ch) * HW; const float* hp = l->xhat + ((size_t)b * C + ch) * HW; for (size_t p = 0; p < HW; ++p) { sb += ep[p]; sg += (double)ep[p] * hp[p]; } }
          if (want_wgrad) { G[ch] = (float)sg; G[C + ch] = (float)sb; G[2 * C + ch] = 0.1f * (P[2 * C + ch] - l->mu[ch]); G[3 * C + ch] = 0.1f * (P[3 * C + ch] - l->var[ch]); }
          const float g = P[ch], k1 = (float)(g * sb / m), k2 = (float)(g * sg / m), sd = l->std[ch];
          for (int b = 0; b < N; ++b) { const float* ep = cur + ((size_t)b * C + ch) * HW; const float* hp = l->xhat + ((size_t)b * C + ch) * HW; float* op = nx + ((size_t)b * C + ch) * HW;
            for (size_t p = 0; p < HW; ++p) op[p] = (ep[p] * g - k1 - hp[p] * k2) / sd; }
        } } break;
      case L_ACT: { const size_t tot = (size_t)N * d->cout * l->oh * l->ow;
#pragma omp parallel for schedule(static)
        for (size_t e = 0; e < tot; ++e) nx[e] = cur[e] * actg(d->act, lin[e], d->alpha); } break;
    }
    if (!need_in) return NULL;
    cur = nx; bi ^= 1;
  }
  return cur;
}

/* BaseMultiLayerUpdater for Adam: g/=mb -> Adam (DL4J form: eps outside the bias correction) -> theta -= g; BN mean/var: NoOp, no /mb.
 * grads2 (optional): a second worker's gradients -- summed (pseudo-gradients averaged) before the update. */
static void net_update(cr_net* n, int mb, const float* grads2) {
  const int t = n->iteration + 1; const float at = n->lr * sqrtf(1.f - powf(n->b2, (float)t)) / (1.f - powf(n->b1, (float)t));
  for (int i = 0; i < n->nl; ++i) { cr_l* l = &n->L[i]; const cr_layer* d = &l->d;
    int64_t segs[3][3]; int ns = 0;   /* off, len, noop */
    if (l->off_b >= 0) { segs[ns][0] = l->off_b; segs[ns][1] = d->cout; segs[ns][2] = 0; ++ns; }
    if (l->off_w >= 0) { segs[ns][0] = l->off_w; segs[ns][1] = d->type == L_DENSE ? (int64_t)d->cin * d->cout : (int64_t)d->cin * d->cout * d->k * d->k; segs[ns][2] = 0; ++ns; }
    if (l->off_gamma >= 0) { segs[ns][0] = l->off_gamma; segs[ns][1] = 2 * (int64_t)d->cout; segs[ns][2] = 0; ++ns; segs[ns][0] = l->off_gamma + 2 * d->cout; segs[ns][1] = 2 * (int64_t)d->cout; segs[ns][2] = 1; ++ns; }
    for (int s = 0; s < ns; ++s) { const int64_t o0 = segs[s][0], len = segs[s][1]; const int noop = (int)segs[s][2];
#pragma omp parallel for schedule(static)
      for (int64_t e = o0; e < o0 + len; ++e) {
        float g = n->grads[e]; if (grads2) g = noop ? 0.5f * (g + grads2[e]) : g + grads2[e];
        if (noop) { n->params[e] -= g; continue; }
        g /= (float)mb;
        const float mm = n->b1 * n->m[e] + (1.f - n->b1) * g, vv = n->b2 * n->v[e] + (1.f - n->b2) * g * g; n->m[e] = mm; n->v[e] = vv;
        n->params[e] -= at * mm / (sqrtf(vv) + n->eps);
      } }
  }
  n->iteration += 1;
}
/* BCE with logits (LossBinaryXENT + sigmoid with clipEps 0): returns sum of losses, eps = sigmoid(z) - y */
static double bce_logits(const float* z, const float* y, int N, float* eps) { double s = 0; for (int i = 0; i < N; ++i) { const float zi = z[i]; s += fmaxf(zi, 0.f) + log1pf(expf(-fabsf(zi))) - y[i] * zi; eps[i] = 1.f / (1.f + expf(-zi)) - y[i]; } return s; }

/* ------------------------------------------------------------------ exported API (ctypes) ---------------------------------------- */
void* cpuref_create(const cr_layer* g, int ng, const cr_layer* d, int nd, int z_dim, int img_c, int img_h, int img_w, int batch, float lr, float b1, float b2, float eps) {
  cr_gan* q = (cr_gan*)calloc(1, sizeof(cr_gan));
  if (net_init(&q->G, g, ng, z_dim, 1, 1, batch, lr, b1, b2, eps) || net_init(&q->D, d, nd, img_c, img_h, img_w, batch, lr, b1, b2, eps)) { free(q); return NULL; }
  q->xfake = (float*)malloc(4 * (size_t)batch * img_c * img_h * img_w); q->gsave = (float*)malloc(4 * q->D.np);
  return q;
}
void cpuref_destroy(void* h) { cr_gan* q = (cr_gan*)h; if (!q) return; net_free(&q->G); net_free(&q->D); free(q->xfake); free(q->gsave); free(q); }
int64_t cpuref_num_params(void* h, int net) { cr_gan* q = (cr_gan*)h; return net ? q->D.np : q->G.np; }
void cpuref_set_params(void* h, int net, const float* p) { cr_gan* q = (cr_gan*)h; cr_net* n = net ? &q->D : &q->G; memcpy(n->params, p, 4 * n->np); }
void cpuref_get_params(void* h, int net, float* p) { cr_gan* q = (cr_gan*)h; cr_net* n = net ? &q->D : &q->G; memcpy(p, n->params, 4 * n->np); }
int cpuref_threads(void) { return omp_get_max_threads(); }
void cpuref_set_threads(int n) { if (n > 0) omp_set_num_threads(n); }
/* oracle gan_step: x_fake = G(z_d) with inference-mode BN; D on real and fake as two minibatches (own BN statistics), gradients summed /2N,
 * one Adam step; G step through train-mode D with labels y_gen, D untouched; one Adam step.  losses = {d_real, d_fake, g} means. */
void cpuref_step(void* h, const float* x_real, const float* z_d, const float* z_g, const float* y_real, const float* y_fake, const float* y_gen, int N, float* losses) {
  cr_gan* q = (cr_gan*)h; cr_net *G = &q->G, *D = &q->D; float* e = (float*)malloc(4 * (size_t)N);
  const float* xf = net_forward(G, z_d, N, 0); memcpy(q->xfake, xf, 4 * (size_t)N * D->in_c * D->in_h * D->in_w);
  const float* lg = net_forward(D, x_real, N, 1); losses[0] = (float)(bce_logits(lg, y_real, N, e) / N);
  net_backward(D, x_real, e, N, 1, 0); memcpy(q->gsave, D->grads, 4 * D->np);
  lg = net_forward(D, q->xfake, N, 1); losses[1] = (float)(bce_logits(lg, y_fake, N, e) / N);
  net_backward(D, q->xfake, e, N, 1, 0);
  net_update(D, 2 * N, q->gsave);
  const float* xg = net_forward(G, z_g, N, 1); lg = net_forward(D, xg, N, 1); losses[2] = (float)(bce_logits(lg, y_gen, N, e) / N);
  const float* ex = net_backward(D, xg, e, N, 0, 1);
  net_backward(G, z_g, ex, N, 1, 0);
  net_update(G, N, NULL);
  free(e);
}
