/* cosnarks_oracle.c -- CPU restatement of the co-snarks Groth16 hot path in plain C.
 *
 * TEST INFRASTRUCTURE AND CPU BASELINE ONLY: loaded by tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference leg; never by the product (co_snarks_b200/).
 *
 * The reference is Rust and cannot be built in this image (no cargo; the arithmetic lives in the
 * un-vendored crates taceo-ark-algebra 0.1.0 / arkworks 0.6, Cargo.lock:4771), so this file restates
 * the path the reference's CPU prover takes:
 *   field ops        ark-ff Fp<MontBackend<_,4>>: 4x64-bit Montgomery limbs, CIOS multiplication
 *   msm              ark-ec VariableBaseMSM::msm_bigint behind taceo_ark_algebra::msm::msm_unchecked
 *                    (call sites co-groth16/src/mpc/plain.rs:66-74, rep3.rs:124-132, groth16.rs:194)
 *   ntt              fft::Domain::{ifft_in_to_out, fft_out_to_in} (groth16/reduction.rs:141-175)
 *   witness map      CircomReduction::witness_map_from_matrices (groth16/reduction.rs:77-193),
 *                    plain driver (mpc/plain.rs) and Rep3 driver (mpc/rep3.rs:31-106, arithmetic.rs:132-146)
 *   proof assembly   CoGroth16::create_proof_with_assignment (groth16.rs:207-338) with injected (r, s)
 * It is pinned on the same fixtures as the Python oracle (tests/test_oracle_c.py): identical proofs
 * for fixed (r, s) on the reference's multiplier2 / poseidon test vectors.  OpenMP plays the role of
 * rayon.  Data layout = the C ABI of include/cosnarks_gpu.h (Montgomery limbs), so the same buffers
 * feed both sides.
 */
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef unsigned __int128 u128;
typedef struct { u64 l[4]; } fe;
typedef struct { u64 p[4]; u64 inv; fe r2, one; } fctx;
#include "params.h"

/* ------------------------------------------------------------------ Fp (generic over the modulus) */
static inline int fe_is_zero(const fe* a) { return (a->l[0] | a->l[1] | a->l[2] | a->l[3]) == 0; }
static inline int fe_eq(const fe* a, const fe* b) { return memcmp(a, b, sizeof(fe)) == 0; }
static inline int geq_p(const u64* a, const fctx* f) {
  for (int i = 3; i >= 0; i--) if (a[i] != f->p[i]) return a[i] > f->p[i];
  return 1;
}
static inline void sub_p(u64* a, const fctx* f) {
  u128 br = 0;
  for (int i = 0; i < 4; i++) { u128 d = (u128)a[i] - f->p[i] - br; a[i] = (u64)d; br = (d >> 64) & 1; }
}
static inline void fe_add(fe* r, const fe* a, const fe* b, const fctx* f) {
  u128 c = 0; u64 t[4];
  for (int i = 0; i < 4; i++) { c += (u128)a->l[i] + b->l[i]; t[i] = (u64)c; c >>= 64; }
  if (c || geq_p(t, f)) sub_p(t, f);
  memcpy(r->l, t, 32);
}
static inline void fe_sub(fe* r, const fe* a, const fe* b, const fctx* f) {
  u128 br = 0; u64 t[4];
  for (int i = 0; i < 4; i++) { u128 d = (u128)a->l[i] - b->l[i] - br; t[i] = (u64)d; br = (d >> 64) & 1; }
  if (br) { u128 c = 0; for (int i = 0; i < 4; i++) { c += (u128)t[i] + f->p[i]; t[i] = (u64)c; c >>= 64; } }
  memcpy(r->l, t, 32);
}
static inline void fe_neg(fe* r, const fe* a, const fctx* f) {
  if (fe_is_zero(a)) { *r = *a; return; }
  fe z; memset(&z, 0, sizeof(z)); fe_sub(r, &z, a, f);
}
static inline void fe_mul(fe* r, const fe* a, const fe* b, const fctx* f) {
  u64 t[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    u128 c = 0;
    for (int j = 0; j < 4; j++) { c += (u128)a->l[j] * b->l[i] + t[j]; t[j] = (u64)c; c >>= 64; }
    c += t[4]; t[4] = (u64)c; t[5] = (u64)(c >> 64);
    u64 m = t[0] * f->inv;
    c = (u128)m * f->p[0] + t[0]; c >>= 64;
    for (int j = 1; j < 4; j++) { c += (u128)m * f->p[j] + t[j]; t[j - 1] = (u64)c; c >>= 64; }
    c += t[4]; t[3] = (u64)c; t[4] = t[5] + (u64)(c >> 64);
  }
  if (t[4] || geq_p(t, f)) sub_p(t, f);
  memcpy(r->l, t, 32);
}
static void fe_pow(fe* r, const fe* a, const u64 e[4], const fctx* f) {
  fe res = f->one, base = *a;
  for (int i = 0; i < 4; i++)
    for (int b = 0; b < 64; b++) {
      if ((e[i] >> b) & 1) fe_mul(&res, &res, &base, f);
      fe_mul(&base, &base, &base, f);
    }
  *r = res;
}
static void fe_inv(fe* r, const fe* a, const fctx* f) {
  u64 e[4]; memcpy(e, f->p, 32); e[0] -= 2;
  fe_pow(r, a, e, f);
}
static inline void fe_from_mont(fe* r, const fe* a, const fctx* f) { fe o; memset(&o, 0, sizeof(o)); o.l[0] = 1; fe_mul(r, a, &o, f); }
static inline void fe_to_mont(fe* r, const fe* a, const fctx* f) { fe_mul(r, a, &f->r2, f); }
static void fe_from_u64(fe* r, u64 v, const fctx* f) { fe t; memset(&t, 0, sizeof(t)); t.l[0] = v; fe_to_mont(r, &t, f); }

/* ------------------------------------------------------------------ Fq and Fq2 wrappers for curve.inc */
#define Q_ADD(r, a, b) fe_add(r, a, b, &FQ)
#define Q_SUB(r, a, b) fe_sub(r, a, b, &FQ)
#define Q_MUL(r, a, b) fe_mul(r, a, b, &FQ)
#define Q_SQR(r, a) fe_mul(r, a, a, &FQ)
#define Q_NEG(r, a) fe_neg(r, a, &FQ)
#define Q_ONE(r) (*(r) = FQ.one)
#define Q_INV(r, a) fe_inv(r, a, &FQ)

typedef struct { fe c0, c1; } f2;
static inline int f2_is_zero(const f2* a) { return fe_is_zero(&a->c0) && fe_is_zero(&a->c1); }
static inline void f2_add(f2* r, const f2* a, const f2* b) { Q_ADD(&r->c0, &a->c0, &b->c0); Q_ADD(&r->c1, &a->c1, &b->c1); }
static inline void f2_sub(f2* r, const f2* a, const f2* b) { Q_SUB(&r->c0, &a->c0, &b->c0); Q_SUB(&r->c1, &a->c1, &b->c1); }
static inline void f2_neg(f2* r, const f2* a) { Q_NEG(&r->c0, &a->c0); Q_NEG(&r->c1, &a->c1); }
static inline void f2_mul(f2* r, const f2* a, const f2* b) {
  fe v0, v1, s, t, u;
  Q_MUL(&v0, &a->c0, &b->c0); Q_MUL(&v1, &a->c1, &b->c1);
  Q_ADD(&s, &a->c0, &a->c1); Q_ADD(&t, &b->c0, &b->c1); Q_MUL(&u, &s, &t);
  Q_SUB(&u, &u, &v0); Q_SUB(&u, &u, &v1);
  Q_SUB(&r->c0, &v0, &v1); r->c1 = u;
}
static inline void f2_sqr(f2* r, const f2* a) { f2 t = *a; f2_mul(r, &t, &t); }
static inline void f2_one(f2* r) { r->c0 = FQ.one; memset(&r->c1, 0, sizeof(fe)); }
static void f2_inv(f2* r, const f2* a) {
  fe n, t; Q_SQR(&n, &a->c0); Q_SQR(&t, &a->c1); Q_ADD(&n, &n, &t); Q_INV(&n, &n);
  Q_MUL(&r->c0, &a->c0, &n); Q_MUL(&t, &a->c1, &n); Q_NEG(&r->c1, &t);
}

#define G g1
#define FT fe
#define F_ADD Q_ADD
#define F_SUB Q_SUB
#define F_MUL Q_MUL
#define F_SQR Q_SQR
#define F_NEG Q_NEG
#define F_ONE Q_ONE
#define F_INV Q_INV
#define F_ISZERO fe_is_zero
#include "curve.inc"
#undef G
#undef FT
#undef F_ADD
#undef F_SUB
#undef F_MUL
#undef F_SQR
#undef F_NEG
#undef F_ONE
#undef F_INV
#undef F_ISZERO

#define G g2
#define FT f2
#define F_ADD f2_add
#define F_SUB f2_sub
#define F_MUL f2_mul
#define F_SQR f2_sqr
#define F_NEG f2_neg
#define F_ONE f2_one
#define F_INV f2_inv
#define F_ISZERO f2_is_zero
#include "curve.inc"

/* ------------------------------------------------------------------ exported MSM (Montgomery scalars) */
static u64* canonical_scalars(const u64* s_mont, size_t sstride, size_t n) {
  u64* out = (u64*)malloc(n * 32 + 32);
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) {
    fe a, c; memcpy(&a, s_mont + (size_t)i * sstride, 32);
    fe_from_mont(&c, &a, &FR);   /* into_bigint (pointshare.rs:211-214) */
    memcpy(out + (size_t)i * 4, &c, 32);
  }
  return out;
}

int oracle_msm_g1(const u64* points, const u64* scalars_mont, size_t sstride_words, size_t n, u64* out_affine) {
  u64* sc = canonical_scalars(scalars_mont, sstride_words, n);
  g1_xyzz r; g1_msm(&r, (const g1_aff*)points, sc, 4, n);
  free(sc);
  g1_aff a; g1_to_aff(&a, &r); memcpy(out_affine, &a, sizeof(a));
  return 0;
}
int oracle_msm_g2(const u64* points, const u64* scalars_mont, size_t sstride_words, size_t n, u64* out_affine) {
  u64* sc = canonical_scalars(scalars_mont, sstride_words, n);
  g2_xyzz r; g2_msm(&r, (const g2_aff*)points, sc, 4, n);
  free(sc);
  g2_aff a; g2_to_aff(&a, &r); memcpy(out_affine, &a, sizeof(a));
  return 0;
}

/* ------------------------------------------------------------------ roots of unity (groth16.rs:60-100) */
/* fr = the scalar field, s = its two-adicity (r - 1 = 2^s * trace, trace odd) */
static void roots_of_unity(unsigned power, fe* gen, fe* shift, const fctx* fr, unsigned s) {
  u64 half[4], trace[4];
  memcpy(half, fr->p, 32); half[0] -= 1; memcpy(trace, half, 32);
  for (int i = 0; i < 4; i++) half[i] = (half[i] >> 1) | (i < 3 ? half[i + 1] << 63 : 0);
  for (unsigned k = 0; k < s; k++) for (int i = 0; i < 4; i++) trace[i] = (trace[i] >> 1) | (i < 3 ? trace[i + 1] << 63 : 0);
  fe zero, minus_one, q, t; memset(&zero, 0, sizeof(zero)); fe_sub(&minus_one, &zero, &fr->one, fr);
  u64 qv = 1;
  for (;;) { fe_from_u64(&q, qv, fr); fe_pow(&t, &q, half, fr); if (fe_eq(&t, &minus_one)) break; qv++; }
  fe z; fe_pow(&z, &q, trace, fr);
  *gen = z;
  for (unsigned k = 0; k < s - power; k++) fe_mul(gen, gen, gen, fr);
  if (power == s) fe_mul(shift, &q, &q, fr);
  else { *shift = z; for (unsigned k = 0; k + 1 < s - power; k++) fe_mul(shift, shift, shift, fr); }
}

/* ------------------------------------------------------------------ NTT (batch = interleaved components) */
static unsigned bitrev(unsigned x, unsigned lg) { unsigned r = 0; for (unsigned i = 0; i < lg; i++) r |= ((x >> i) & 1u) << (lg - 1 - i); return r; }

static fe* twiddles(const fe* g, size_t half, const fctx* fr) {
  fe* tw = (fe*)malloc((half ? half : 1) * sizeof(fe));
  if (!half) return tw;
  const size_t blk = 4096;
#pragma omp parallel for schedule(static)
  for (long b = 0; b < (long)((half + blk - 1) / blk); b++) {
    size_t lo = (size_t)b * blk, hi = lo + blk < half ? lo + blk : half;
    u64 e[4] = {lo, 0, 0, 0};
    fe cur; fe_pow(&cur, g, e, fr);
    for (size_t k = lo; k < hi; k++) { tw[k] = cur; fe_mul(&cur, &cur, g, fr); }
  }
  return tw;
}

/* natural in -> bit-reversed out (DIF), scaled by 1/n : Domain::ifft_in_to_out.  fr = the scalar field. */
static void ifft_in_to_out(fe* a, unsigned lg, unsigned batch, const fe* gen, const fctx* fr) {
  size_t n = (size_t)1 << lg;
  if (lg == 0) return;
  fe ginv; fe_inv(&ginv, gen, fr);
  fe* tw = twiddles(&ginv, n / 2, fr);
  for (size_t m = n / 2; m >= 1; m >>= 1) {
    size_t step = (n / 2) / m;
#pragma omp parallel for schedule(static)
    for (long bf = 0; bf < (long)(n / 2); bf++) {
      size_t k = ((size_t)bf / m) * 2 * m, j = (size_t)bf % m;
      for (unsigned c = 0; c < batch; c++) {
        fe* x = &a[(k + j) * batch + c]; fe* y = &a[(k + j + m) * batch + c];
        fe s, d; fe_add(&s, x, y, fr); fe_sub(&d, x, y, fr);
        *x = s; fe_mul(y, &d, &tw[j * step], fr);
      }
    }
  }
  fe ninv; fe_from_u64(&ninv, n, fr); fe_inv(&ninv, &ninv, fr);
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)(n * batch); i++) fe_mul(&a[i], &a[i], &ninv, fr);
  free(tw);
}

/* bit-reversed in -> natural out (DIT) : Domain::fft_out_to_in */
static void fft_out_to_in(fe* a, unsigned lg, unsigned batch, const fe* gen, const fctx* fr) {
  size_t n = (size_t)1 << lg;
  if (lg == 0) return;
  fe* tw = twiddles(gen, n / 2, fr);
  for (size_t m = 1; m < n; m <<= 1) {
    size_t step = (n / 2) / m;
#pragma omp parallel for schedule(static)
    for (long bf = 0; bf < (long)(n / 2); bf++) {
      size_t k = ((size_t)bf / m) * 2 * m, j = (size_t)bf % m;
      for (unsigned c = 0; c < batch; c++) {
        fe* x = &a[(k + j) * batch + c]; fe* y = &a[(k + j + m) * batch + c];
        fe t, s, d; fe_mul(&t, y, &tw[j * step], fr);
        fe_add(&s, x, &t, fr); fe_sub(&d, x, &t, fr);
        *x = s; *y = d;
      }
    }
  }
  free(tw);
}

/* curve: 0 = BN254 Fr, 1 = BLS12-381 Fr (the cs_curve ids of include/cosnarks_gpu.h) */
static const fctx* fr_of(int curve) { return curve == 0 ? &FR : curve == 1 ? &FR_BLS12_381 : NULL; }
int oracle_ifft_in_to_out(u64* data, unsigned lg, unsigned batch, const u64* gen, int curve) {
  const fctx* fr = fr_of(curve);
  if (!fr) return -1;
  ifft_in_to_out((fe*)data, lg, batch, (const fe*)gen, fr);
  return 0;
}
int oracle_fft_out_to_in(u64* data, unsigned lg, unsigned batch, const u64* gen, int curve) {
  const fctx* fr = fr_of(curve);
  if (!fr) return -1;
  fft_out_to_in((fe*)data, lg, batch, (const fe*)gen, fr);
  return 0;
}

/* ------------------------------------------------------------------ Groth16 (same key descriptor as the C ABI) */
typedef struct {
  int curve;
  size_t num_constraints, num_instance_variables, num_witness_variables;
  const uint32_t* a_row_ptr; const uint32_t* a_col; const u64* a_coeff; size_t a_nnz;
  const uint32_t* b_row_ptr; const uint32_t* b_col; const u64* b_coeff; size_t b_nnz;
  const u64* alpha_g1; const u64* beta_g1; const u64* beta_g2; const u64* delta_g1; const u64* delta_g2;
  const u64* a_query; size_t a_query_len;
  const u64* b_g1_query; size_t b_g1_query_len;
  const u64* b_g2_query; size_t b_g2_query_len;
  const u64* l_query; size_t l_query_len;
  const u64* h_query; size_t h_query_len;
  int window_bits;
  const uint32_t* c_row_ptr; const uint32_t* c_col; const u64* c_coeff; size_t c_nnz;
} key_desc;

/* evaluate_constraint (reduction.rs:196-210; mpc/plain.rs:29-43, mpc/rep3.rs:31-49) */
static void spmv(fe* out, const uint32_t* rp, const uint32_t* col, const fe* cf, const fe* pub, size_t ni,
                 const fe* wit, unsigned batch, int pub_comp, size_t nrows, size_t npubrows, size_t n, const fctx* fr) {
#pragma omp parallel for schedule(static)
  for (long r = 0; r < (long)n; r++) {
    fe acc[2]; memset(acc, 0, sizeof(acc));
    if ((size_t)r < nrows) {
      for (uint32_t k = rp[r]; k < rp[r + 1]; k++) {
        fe t;
        if (col[k] < ni) {
          if (pub_comp >= 0) { fe_mul(&t, &cf[k], &pub[col[k]], fr); fe_add(&acc[pub_comp], &acc[pub_comp], &t, fr); }
        } else {
          size_t wi = (size_t)(col[k] - ni) * batch;
          for (unsigned c = 0; c < batch; c++) { fe_mul(&t, &cf[k], &wit[wi + c], fr); fe_add(&acc[c], &acc[c], &t, fr); }
        }
      }
    } else if ((size_t)r < nrows + npubrows) {
      if (pub_comp >= 0) acc[pub_comp] = pub[r - nrows];
    }
    for (unsigned c = 0; c < batch; c++) out[(size_t)r * batch + c] = acc[c];
  }
}

/* local_mul_vec (+ optional mask, optional subtraction) -- rep3/arithmetic.rs:132-146, ops.rs:69-76 */
static void local_mul(fe* out, const fe* a, const fe* b, unsigned batch, const fe* mask, const fe* sub, size_t n, const fctx* fr) {
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) {
    fe z;
    if (batch == 1) fe_mul(&z, &a[i], &b[i], fr);
    else {
      fe t1, t2, t3;
      fe_mul(&t1, &a[2 * i], &b[2 * i], fr); fe_mul(&t2, &a[2 * i], &b[2 * i + 1], fr); fe_mul(&t3, &a[2 * i + 1], &b[2 * i], fr);
      fe_add(&z, &t1, &t2, fr); fe_add(&z, &z, &t3, fr);
    }
    if (mask) fe_add(&z, &z, &mask[i], fr);
    if (sub) fe_sub(&z, &z, &sub[i], fr);
    out[i] = z;
  }
}

/* CircomReduction::witness_map_from_matrices.  kind 0 = plain, 1 = rep3 (party 0..2).  h: n elements.
 * The scalar field, two-adicity and roots follow d->curve (0 BN254: s = 28, 1 BLS12-381: s = 32). */
int oracle_witness_map(const key_desc* d, int kind, int party, const u64* pub_, const u64* wit_, const u64* m1,
                       const u64* m2, u64* h_out) {
  const size_t nc = d->num_constraints, ni = d->num_instance_variables;
  const fctx* fr = fr_of(d->curve);
  if (!fr) return -1;
  const unsigned two_adicity = d->curve == 0 ? 28 : 32;
  size_t n = 1; unsigned lg = 0;
  while (n < nc + ni) { n <<= 1; lg++; }
  if (lg > two_adicity) return -1;
  const unsigned batch = kind ? 2 : 1;
  const int pub_comp = kind ? (party == 0 ? 0 : (party == 1 ? 1 : -1)) : 0;
  fe gen, shift; roots_of_unity(lg, &gen, &shift, fr, two_adicity);
  /* bit_reversed_coset_table (reduction.rs:45-60) */
  fe* table = (fe*)malloc(n * sizeof(fe));
  { fe* nat = twiddles(&shift, n, fr);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) table[bitrev((unsigned)i, lg)] = nat[i];
    free(nat); }
  fe* a = (fe*)malloc(n * batch * sizeof(fe));
  fe* b = (fe*)malloc(n * batch * sizeof(fe));
  fe* c = (fe*)malloc(n * sizeof(fe));
  spmv(a, d->a_row_ptr, d->a_col, (const fe*)d->a_coeff, (const fe*)pub_, ni, (const fe*)wit_, batch, pub_comp, nc, ni, n, fr);
  spmv(b, d->b_row_ptr, d->b_col, (const fe*)d->b_coeff, (const fe*)pub_, ni, (const fe*)wit_, batch, pub_comp, nc, 0, n, fr);
  local_mul(c, a, b, batch, kind ? (const fe*)m1 : NULL, NULL, n, fr);
  fe* vecs[3] = {a, b, c};
  unsigned bt[3] = {batch, batch, 1};
  for (int v = 0; v < 3; v++) {
    ifft_in_to_out(vecs[v], lg, bt[v], &gen, fr);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++)
      for (unsigned k = 0; k < bt[v]; k++) fe_mul(&vecs[v][(size_t)i * bt[v] + k], &vecs[v][(size_t)i * bt[v] + k], &table[i], fr);
    fft_out_to_in(vecs[v], lg, bt[v], &gen, fr);
  }
  local_mul((fe*)h_out, a, b, batch, kind ? (const fe*)m2 : NULL, c, n, fr);
  free(a); free(b); free(c); free(table);
  return 0;
}

/* Groth16::plain_prove with injected r, s (Montgomery).  pub includes the leading 1. */
int oracle_groth16_prove_plain(const key_desc* d, const u64* pub_, const u64* wit_, const u64* r_m, const u64* s_m,
                               u64* out_a, u64* out_b, u64* out_c) {
  const size_t nc = d->num_constraints, ni = d->num_instance_variables, nw = d->num_witness_variables;
  if (d->curve != 0) return -1;  /* G1/G2 here are BN254's (4-limb Fq) */
  size_t n = 1; while (n < nc + ni) n <<= 1;
  fe* h = (fe*)malloc(n * sizeof(fe));
  if (oracle_witness_map(d, 0, 0, pub_, wit_, NULL, NULL, (u64*)h)) { free(h); return -1; }
  u64* aux = canonical_scalars(wit_, 4, nw);
  u64* hs = canonical_scalars((const u64*)h, 4, n);
  u64* pubs = canonical_scalars(pub_, 4, ni);
  fe rc, sc, rs, rsc; fe_from_mont(&rc, (const fe*)r_m, &FR); fe_from_mont(&sc, (const fe*)s_m, &FR);
  fe_mul(&rs, (const fe*)r_m, (const fe*)s_m, &FR); fe_from_mont(&rsc, &rs, &FR);
  g1_xyzz A, B1, L, H, t, dl; g2_xyzz B2, t2, dl2;
  /* the five MSMs of rayon_join5! (groth16.rs:227-294) as ONE task pool; the G2 tasks (3x longer) go first */
  {
    const size_t want = (size_t)omp_get_max_threads() * 3;
    g1_job ja, jb1, jl, jh; g2_job jb2;
    g2_msm_plan(&jb2, (const g2_aff*)d->b_g2_query + ni, aux, 4, nw, want / 2);
    g1_msm_plan(&ja, (const g1_aff*)d->a_query + ni, aux, 4, nw, want / 6);
    g1_msm_plan(&jb1, (const g1_aff*)d->b_g1_query + ni, aux, 4, nw, want / 6);
    g1_msm_plan(&jl, (const g1_aff*)d->l_query, aux, 4, nw, want / 6);
    g1_msm_plan(&jh, (const g1_aff*)d->h_query, hs, 4, n, want / 6);
    long t2 = (long)g2_msm_ntasks(&jb2), ta = (long)g1_msm_ntasks(&ja), tb = (long)g1_msm_ntasks(&jb1),
         tl = (long)g1_msm_ntasks(&jl), th = (long)g1_msm_ntasks(&jh);
    long total = t2 + ta + tb + tl + th;
#pragma omp parallel for schedule(dynamic, 1)
    for (long t = 0; t < total; t++) {
      long k = t;
      if (k < t2) { g2_msm_task(&jb2, (size_t)k); continue; } k -= t2;
      if (k < ta) { g1_msm_task(&ja, (size_t)k); continue; } k -= ta;
      if (k < tb) { g1_msm_task(&jb1, (size_t)k); continue; } k -= tb;
      if (k < tl) { g1_msm_task(&jl, (size_t)k); continue; } k -= tl;
      g1_msm_task(&jh, (size_t)k);
    }
    g1_msm_finish(&ja, &A); g1_msm_finish(&jb1, &B1); g2_msm_finish(&jb2, &B2);
    g1_msm_finish(&jl, &L); g1_msm_finish(&jh, &H);
  }
  /* calculate_coeff (groth16.rs:179-203): + query[0] + vk_param + msm(query[1..=pub], inputs) + r*delta */
  g1_msm(&t, (const g1_aff*)d->a_query + 1, pubs + 4, 4, ni - 1); g1_padd(&A, &t);
  g1_from_aff(&t, (const g1_aff*)d->a_query); g1_padd(&A, &t);
  g1_from_aff(&t, (const g1_aff*)d->alpha_g1); g1_padd(&A, &t);
  g1_from_aff(&dl, (const g1_aff*)d->delta_g1); g1_mul(&t, &dl, rc.l); g1_padd(&A, &t);
  g1_msm(&t, (const g1_aff*)d->b_g1_query + 1, pubs + 4, 4, ni - 1); g1_padd(&B1, &t);
  g1_from_aff(&t, (const g1_aff*)d->b_g1_query); g1_padd(&B1, &t);
  g1_from_aff(&t, (const g1_aff*)d->beta_g1); g1_padd(&B1, &t);
  g1_mul(&t, &dl, sc.l); g1_padd(&B1, &t);
  g2_msm(&t2, (const g2_aff*)d->b_g2_query + 1, pubs + 4, 4, ni - 1); g2_padd(&B2, &t2);
  g2_from_aff(&t2, (const g2_aff*)d->b_g2_query); g2_padd(&B2, &t2);
  g2_from_aff(&t2, (const g2_aff*)d->beta_g2); g2_padd(&B2, &t2);
  g2_from_aff(&dl2, (const g2_aff*)d->delta_g2); g2_mul(&t2, &dl2, sc.l); g2_padd(&B2, &t2);
  /* C = s*A + r*B1 - rs*delta1 + L + H (groth16.rs:296-322) */
  g1_xyzz C; g1_mul(&C, &A, sc.l);
  g1_mul(&t, &B1, rc.l); g1_padd(&C, &t);
  g1_mul(&t, &dl, rsc.l); fe_neg(&t.y, &t.y, &FQ); g1_padd(&C, &t);
  g1_padd(&C, &L); g1_padd(&C, &H);
  g1_aff oa, oc; g2_aff ob;
  g1_to_aff(&oa, &A); g2_to_aff(&ob, &B2); g1_to_aff(&oc, &C);
  memcpy(out_a, &oa, sizeof(oa)); memcpy(out_b, &ob, sizeof(ob)); memcpy(out_c, &oc, sizeof(oc));
  free(h); free(aux); free(hs); free(pubs);
  return 0;
}

#include "plonk.inc"

int oracle_num_threads(void) { return omp_get_max_threads(); }
void oracle_set_threads(int n) { omp_set_num_threads(n); }
