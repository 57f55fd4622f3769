// Share-wise element kernels and the R1CS sparse matrix-vector product.
//
// Replaces, on n-sized vectors (n = domain size):
//  * `T::local_mul_vec` -> `rep3::arithmetic::local_mul_vec`
//    (mpc-core/src/protocols/rep3/arithmetic.rs:132-146; share product ops.rs:69-76):
//        z_i = a_i.a*b_i.a + a_i.a*b_i.b + a_i.b*b_i.a + mask_i          (Rep3)
//        z_i = a_i * b_i                                                  (plain / Shamir)
//  * `T::distribute_powers_and_mul_by_const` (co-groth16/src/mpc/rep3.rs:95-106, plain.rs:91-98)
//    and the inline c-scaling (reduction.rs:166-171):   x_i *= table_i   per share component
//  * the final `ab -= c` (reduction.rs:185-190)
//  * `evaluate_constraint` (co-groth16/src/mpc/rep3.rs:31-49, plain.rs:29-43; driver
//    reduction.rs:196-210) incl. the public rows re-inserted at reduction.rs:111-113
//  * the Rep3 -> Shamir bridge a*x + b*y (mpc-core/src/protocols/bridges/rep3_to_shamir.rs:43-63)
// All of these stream each operand once; they sit at the HBM/IMAD ridge (1-3 mulmods per 64-192 B).
#pragma once
#include "cs_common.cuh"
#include "cs_field.cuh"
#include "cs_ntt.cuh"  // ld_fr / st_fr

namespace cs {

enum VecOp { VEC_MUL = 0, VEC_ADD = 1, VEC_SUB = 2 };

// out = a (op) b, elementwise on n field elements
template <class FrP>
CS_GLOBAL void k_vec_binop(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                           uint32_t* __restrict__ out, size_t n, int op) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) {
    Fp<FrP> x = ld_fr<FrP>(a + i * FrP::N), y = ld_fr<FrP>(b + i * FrP::N), z;
    if (op == VEC_MUL) z = x * y;
    else if (op == VEC_ADD) z = x + y;
    else z = x - y;
    st_fr<FrP>(out + i * FrP::N, z);
  }
}

// x[i*batch + c] *= tab[i]     (distribute_powers_and_mul_by_const on plain values or shares)
template <class FrP>
CS_GLOBAL void k_vec_scale_table(uint32_t* __restrict__ x, const uint32_t* __restrict__ tab, size_t n,
                                 uint32_t batch) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n * batch; i += step) {
    size_t e = i / batch;
    Fp<FrP> v = ld_fr<FrP>(x + i * FrP::N) * ld_fr<FrP>(tab + e * FrP::N);
    st_fr<FrP>(x + i * FrP::N, v);
  }
}

// Rep3 local multiplication.  a, b: n shares {a,b} (2 x Fr each); mask: n Fr (nullable = 0);
// sub: n Fr (nullable) subtracted afterwards (fuses reduction.rs:182-190: ab = local_mul_vec(a,b) - c).
template <class FrP>
CS_GLOBAL void k_rep3_local_mul(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                                const uint32_t* __restrict__ mask, const uint32_t* __restrict__ sub,
                                uint32_t* __restrict__ out, size_t n) {
  constexpr int NW = FrP::N;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) {
    Fp<FrP> aa = ld_fr<FrP>(a + (2 * i) * NW), ab = ld_fr<FrP>(a + (2 * i + 1) * NW);
    Fp<FrP> ba = ld_fr<FrP>(b + (2 * i) * NW), bb = ld_fr<FrP>(b + (2 * i + 1) * NW);
    // a.a*b.a + a.a*b.b + a.b*b.a  ==  a.a*(b.a + b.b) + a.b*b.a   (exact in the field)
    Fp<FrP> z = Fp<FrP>::dot2(aa, ba + bb, ab, ba);  // one reduction for both products
    if (mask) z = z + ld_fr<FrP>(mask + i * NW);
    if (sub) z = z - ld_fr<FrP>(sub + i * NW);
    st_fr<FrP>(out + i * NW, z);
  }
}

// Plain / Shamir local multiplication with the same optional fused subtraction: out = a*b - sub
template <class FrP>
CS_GLOBAL void k_plain_mul_sub(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                               const uint32_t* __restrict__ sub, uint32_t* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) {
    Fp<FrP> z = ld_fr<FrP>(a + i * FrP::N) * ld_fr<FrP>(b + i * FrP::N);
    if (sub) z = z - ld_fr<FrP>(sub + i * FrP::N);
    st_fr<FrP>(out + i * FrP::N, z);
  }
}

// Rep3 -> Shamir(t=1) translation: out_i = ca * x_i.a + cb * x_i.b  (rep3_to_shamir.rs:43-63)
template <class FrP>
CS_GLOBAL void k_rep3_to_shamir(const uint32_t* __restrict__ x, const uint32_t* __restrict__ ca,
                                const uint32_t* __restrict__ cb, uint32_t* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  Fp<FrP> fa = ld_fr<FrP>(ca), fb = ld_fr<FrP>(cb);
  for (; i < n; i += step) {
    Fp<FrP> z = ld_fr<FrP>(x + 2 * i * FrP::N) * fa + ld_fr<FrP>(x + (2 * i + 1) * FrP::N) * fb;
    st_fr<FrP>(out + i * FrP::N, z);
  }
}

// Batched witness-extension VM operations on Rep3 share vectors (circom-mpc-vm/src/mpc/batched_rep3.rs:124-188,
// 322-337 -> rep3::arithmetic::{add, sub, add_public, sub_shared_by_public, sub_public_by_shared, mul_public,
// promote_to_trivial_share}, arithmetic.rs:36-100,321-327).  x: n shares {a, b}; y: n shares or n public values.
// The public operand enters party 0's `a` and party 1's `b` only (arithmetic.rs:41-48).
enum Rep3BatchOp {
  R3B_ADD = 0,            // shared + shared
  R3B_SUB = 1,            // shared - shared
  R3B_ADD_PUBLIC = 2,     // shared + public
  R3B_SUB_PUBLIC = 3,     // shared - public            (sub_shared_by_public)
  R3B_PUBLIC_SUB = 4,     // public - shared            (sub_public_by_shared)
  R3B_MUL_PUBLIC = 5,     // shared * public
  R3B_NEG = 6,            // -shared                     (y unused)
  R3B_PROMOTE = 7,        // public -> trivial share     (x unused)
  R3B_OPEN_FINISH = 8     // a + b + c, c = previous party's b (open_vec, arithmetic.rs:261-271): out = n public values
};
template <class FrP>
CS_GLOBAL void k_rep3_batch(int op, int party, const uint32_t* __restrict__ x, const uint32_t* __restrict__ y,
                            uint32_t* __restrict__ out, size_t n) {
  constexpr int NW = FrP::N;
  typedef Fp<FrP> F;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) {
    F xa = F::zero(), xb = F::zero();
    if (op != R3B_PROMOTE) { xa = ld_fr<FrP>(x + (2 * i) * NW); xb = ld_fr<FrP>(x + (2 * i + 1) * NW); }
    F ra, rb;
    if (op == R3B_ADD || op == R3B_SUB) {
      F ya = ld_fr<FrP>(y + (2 * i) * NW), yb = ld_fr<FrP>(y + (2 * i + 1) * NW);
      ra = op == R3B_ADD ? xa + ya : xa - ya;
      rb = op == R3B_ADD ? xb + yb : xb - yb;
    } else if (op == R3B_NEG) {
      ra = xa.neg(); rb = xb.neg();
    } else if (op == R3B_OPEN_FINISH) {
      st_fr<FrP>(out + i * NW, xa + xb + ld_fr<FrP>(y + i * NW));
      continue;
    } else {
      F p = ld_fr<FrP>(y + i * NW);
      if (op == R3B_MUL_PUBLIC) {
        ra = xa * p; rb = xb * p;
      } else {
        if (op == R3B_SUB_PUBLIC) p = p.neg();
        if (op == R3B_PUBLIC_SUB) { xa = xa.neg(); xb = xb.neg(); }
        ra = party == 0 ? xa + p : xa;
        rb = party == 1 ? xb + p : xb;
      }
    }
    st_fr<FrP>(out + (2 * i) * NW, ra);
    st_fr<FrP>(out + (2 * i + 1) * NW, rb);
  }
}
// open_vec, first half: b-components as a contiguous vector, optionally written straight into the NEXT party's
// receive buffer (peer memory) -- reshare_many(&b) (arithmetic.rs:269)
template <class FrP>
CS_GLOBAL void k_rep3_take_b(const uint32_t* __restrict__ x, uint32_t* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) st_fr<FrP>(out + i * FrP::N, ld_fr<FrP>(x + (2 * i + 1) * FrP::N));
}

// out_i = sum_j w_j * in_j[i], j < k <= LINCOMB_MAX.  Shamir's king-based degree reduction
// (mpc-core/src/protocols/shamir/network.rs:150-243): the "pair consumption" `inp += r_2t` / `share -= r_t`
// are k = 2 calls with weights (1, +-1); the king's Lagrange-weighted accumulation over the 2t+1 received
// vectors (:170-187) is one call with k = 2t+1; each party's fresh share `acc * c_id` (:196-214) is k = 1.
constexpr unsigned LINCOMB_MAX = 8;
struct LincombArgs {
  const uint32_t* in[LINCOMB_MAX];
  uint32_t w[LINCOMB_MAX][8];
};
template <class FrP>
CS_GLOBAL void k_vec_lincomb(LincombArgs args, uint32_t k, uint32_t* __restrict__ out, size_t n) {
  constexpr int NW = FrP::N;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) {
    Fp<FrP> acc = Fp<FrP>::zero();
    for (uint32_t j = 0; j < k; j++) {
      Fp<FrP> w;
      CS_UNROLL
      for (int l = 0; l < NW; l++) w.l[l] = args.w[j][l];
      acc = acc + ld_fr<FrP>(args.in[j] + i * NW) * w;
    }
    st_fr<FrP>(out + i * NW, acc);
  }
}

// eval_poly (mpc-core/src/protocols/rep3/poly.rs:42-68; plain: DensePolynomial::evaluate): the reference
// splits the coefficients into per-thread chunks, runs Horner on each, scales by point^(chunk start) and
// sums.  Same here: one thread per chunk of POLY_CHUNK coefficients, shared-memory tree per block; the
// per-block sums (`batch` components each) are added up by the caller.
constexpr unsigned POLY_CHUNK = 64;
template <class FrP>
CS_GLOBAL void k_poly_eval(const uint32_t* __restrict__ coeffs, size_t n, uint32_t batch,
                           const uint32_t* __restrict__ point, const uint32_t* __restrict__ point_chunk_pows,
                           uint32_t* __restrict__ block_sums) {
  constexpr int NW = FrP::N;
  CS_DYN_SMEM(uint32_t, sm);  // blockDim.x * batch elements
  typedef Fp<FrP> F;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t lo = t * POLY_CHUNK;
  F x = ld_fr<FrP>(point);
  F acc[2];
  acc[0] = F::zero();
  acc[1] = F::zero();
  if (lo < n) {
    size_t hi = lo + POLY_CHUNK < n ? lo + POLY_CHUNK : n;
    for (size_t k = hi; k-- > lo;) {
      acc[0] = acc[0] * x + ld_fr<FrP>(coeffs + (k * batch) * NW);
      if (batch == 2) acc[1] = acc[1] * x + ld_fr<FrP>(coeffs + (k * batch + 1) * NW);
    }
    // scale by point^lo = (point^POLY_CHUNK)^t, square-and-multiply over the table of squarings
    F pw = F::one();
    for (uint32_t j = 0; (t >> j) != 0; j++)
      if ((t >> j) & 1) pw = pw * ld_fr<FrP>(point_chunk_pows + (size_t)j * NW);
    acc[0] = acc[0] * pw;
    if (batch == 2) acc[1] = acc[1] * pw;
  }
  for (uint32_t c = 0; c < batch; c++) st_fr<FrP>(sm + ((size_t)threadIdx.x * batch + c) * NW, acc[c]);
  __syncthreads();
  for (uint32_t step = blockDim.x >> 1; step > 0; step >>= 1) {
    if (threadIdx.x < step)
      for (uint32_t c = 0; c < batch; c++) {
        uint32_t* mine = sm + ((size_t)threadIdx.x * batch + c) * NW;
        F v = ld_fr<FrP>(mine) + ld_fr<FrP>(sm + ((size_t)(threadIdx.x + step) * batch + c) * NW);
        st_fr<FrP>(mine, v);
      }
    __syncthreads();
  }
  if (threadIdx.x == 0)
    for (uint32_t c = 0; c < batch; c++)
      st_fr<FrP>(block_sums + ((size_t)blockIdx.x * batch + c) * NW, ld_fr<FrP>(sm + (size_t)c * NW));
}

// evaluate_constraint over CSR rows.  One thread per row.
//   wit: n_wit entries of `batch` components (1: plain value / half share; 2: Rep3 share {a,b})
//   pub: n_pub public inputs (pub[0] = 1).  Column index < n_pub selects a public input.
//   pub_comp: component that receives public terms (Rep3: 0 for party 0, 1 for party 1, -1 for
//             party 2; plain: 0)   -- arithmetic.rs:52-58
//   Rows [nrows, nrows + n_pubrows) get the promoted public inputs (reduction.rs:111-113) when
//   n_pubrows > 0; rows beyond that up to `domain` are zero-filled (reduction.rs:208).
//   grid.y = proofs of a batch: proof p reads pub + p n_pub and wit + p wpstride elements and writes `batch` columns
//   from column p batch of out's ocols-column rows (ocols = batch for one proof).
template <class FrP>
CS_GLOBAL void k_spmv(const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                      const uint32_t* __restrict__ coeff, const uint32_t* __restrict__ pub, uint32_t n_pub,
                      const uint32_t* __restrict__ wit, uint32_t batch, uint32_t wstride, int pub_comp, uint32_t nrows,
                      uint32_t n_pubrows, uint32_t domain, uint32_t wpstride, uint32_t ocols, uint32_t* __restrict__ out) {
  constexpr int NW = FrP::N;
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= domain) return;
  pub += (size_t)blockIdx.y * n_pub * NW;
  wit += (size_t)blockIdx.y * wpstride * NW;
  out += ((size_t)r * ocols + (size_t)blockIdx.y * batch) * NW;
  Fp<FrP> acc[2];
  acc[0] = Fp<FrP>::zero();
  acc[1] = Fp<FrP>::zero();
  if (r < nrows) {
    uint32_t beg = row_ptr[r], end = row_ptr[r + 1];
    for (uint32_t k = beg; k < end; k++) {
      uint32_t cidx = col[k];
      Fp<FrP> cf = ld_fr<FrP>(coeff + (size_t)k * NW);
      if (cidx < n_pub) {
        if (pub_comp >= 0) {
          Fp<FrP> t = cf * ld_fr<FrP>(pub + (size_t)cidx * NW);
          if (pub_comp == 0) acc[0] = acc[0] + t; else acc[1] = acc[1] + t;
        }
      } else {
        // wstride = elements per witness entry (2 for Rep3 shares); batch < wstride evaluates the `a`
        // component only: evaluate_constraint_half_share (mpc/rep3.rs:51-74)
        size_t wi = (size_t)(cidx - n_pub) * wstride;
        acc[0] = acc[0] + cf * ld_fr<FrP>(wit + wi * NW);
        if (batch == 2) acc[1] = acc[1] + cf * ld_fr<FrP>(wit + (wi + 1) * NW);
      }
    }
  } else if (r < nrows + n_pubrows) {
    if (pub_comp >= 0) {
      Fp<FrP> v = ld_fr<FrP>(pub + (size_t)(r - nrows) * NW);
      if (pub_comp == 0) acc[0] = v; else acc[1] = v;
    }
  }
  st_fr<FrP>(out, acc[0]);
  if (batch == 2) st_fr<FrP>(out + NW, acc[1]);
}

}  // namespace cs
