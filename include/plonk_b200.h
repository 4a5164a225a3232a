/* plonk_b200.h -- C ABI of libplonk_b200.so, the H100-native PLONK proving hot path.
 *
 * The reference (0xPARC/plonkathon) is pure Python and has no FFI of its own; these entry points are
 * what a binding for its hot path would call, one per reference callable (file:line cited per entry,
 * relative to the reference tree).  Plain pointers and sizes only; no torch types.
 *
 * Conventions
 *   - Fr element  : 32 bytes, little-endian integer in [0, r), r = BN254 group order (curve.py:11).
 *   - G1 affine   : 64 bytes, x || y, each a 32-byte little-endian integer in [0, q) (py_ecc FQ.n).
 *                   The identity (py_ecc Z1 == None) is reported through an `is_identity` flag.
 *   - "d_" pointers are device pointers on the context's device; "h_" pointers are host memory.
 *   - Vectors at the ABI are in canonical (non-Montgomery) form unless a parameter says otherwise.
 *   - Every call returns 0 on success, non-zero on error; pb200_last_error() describes the failure
 *     (thread-local).  The Python facade turns errors into exceptions/AssertionErrors matching the
 *     reference's behaviour.
 *   - Work is issued on the context's CUDA stream; calls that return host data synchronise it.
 *   - A context (and the SRS / prover objects created on it) is not thread-safe: one context per host thread
 *     and per GPU, like the reference's single-threaded call sequence.  Objects are freed by their _destroy
 *     call; the caller owns every h_ / d_ buffer it passes in.
 */
#ifndef PLONK_B200_H
#define PLONK_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pb200_ctx pb200_ctx;
typedef struct pb200_srs pb200_srs;
typedef struct pb200_prover pb200_prover;
typedef struct pb200_transcript pb200_transcript;

/* ---- context ------------------------------------------------------------------------------- */
const char* pb200_last_error(void);
const char* pb200_version(void);
/* cuda_stream may be NULL (the library creates its own non-blocking stream). */
int pb200_ctx_create(int device, void* cuda_stream, pb200_ctx** out);
void pb200_ctx_destroy(pb200_ctx* ctx);
int pb200_ctx_sync(pb200_ctx* ctx);
/* number of CUDA kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t pb200_ctx_launches(pb200_ctx* ctx);
/* per-kernel device timing with CUDA events on the launching stream (bench.py's roofline object).
 * enable != 0 clears the records and starts recording.  category 0: MSM bucket accumulation kernel,
 * 1: NTT pass kernel.  Returns the summed duration and the number of launches recorded. */
int pb200_ctx_timing(pb200_ctx* ctx, int enable);
int pb200_ctx_timing_read(pb200_ctx* ctx, int category, double* total_ms, uint64_t* count);
/* the context's CUDA stream (cudaStream_t) so callers can time with events on it */
void* pb200_ctx_stream(pb200_ctx* ctx);

/* ---- Fr vectors ---------------------------------------------------------------------------- */
/* canonical <-> Montgomery form, in place allowed */
int pb200_fr_to_mont(pb200_ctx* ctx, const void* d_in, void* d_out, uint64_t n);
int pb200_fr_from_mont(pb200_ctx* ctx, const void* d_in, void* d_out, uint64_t n);

/* poly.py:23-109  the ring operations of Polynomial on device-resident canonical vectors of n elements:
 *   op 0 a + b, 1 a - b, 2 a * b, 3 a / b (element-wise, py_ecc's inv(0) == 0);
 *   op 4 a + s, 5 a - s, 6 a * s for a Scalar s (h_scalar, canonical) on every element (LAGRANGE basis) --
 *   Polynomial / Scalar is op 6 with 1/s; op 7 / 8: + s / - s on element 0 only (MONOMIAL basis, poly.py:32-37);
 *   op 9 shift: out[i] = a[(i + shift) mod n] (poly.py:102-107; not in place).  d_out may alias d_a otherwise. */
int pb200_fr_vec_op(pb200_ctx* ctx, int op, const void* d_a, const void* d_b, const uint8_t* h_scalar, void* d_out,
                    uint64_t n, uint64_t shift);

/* poly.py:113-149  Polynomial.fft(inv) / ifft: natural order in and out, n = 2^log_n <= 2^28.
 * inverse != 0 uses the reversed roots and multiplies by n^-1.  d_out may alias d_in. */
int pb200_fr_ntt(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, int inverse);
int pb200_fr_ntt_host(pb200_ctx* ctx, const uint8_t* h_in, uint8_t* h_out, unsigned log_n, int inverse);

/* The local building block of the slab-sharded transform: the 2^log_m-point NTT of the strided sub-sequence
 * d_in[offset + stride * i] (rank h of G transforms x[h::G]). */
int pb200_fr_ntt_decimated(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_m, int inverse, uint64_t stride,
                           uint64_t offset);

/* poly.py:156-163  to_coset_extended_lagrange(offset): n Lagrange values -> 4n evaluations on
 * offset * <w_4n>.  h_offset: 32-byte canonical Fr. */
int pb200_fr_coset_extend(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, const uint8_t* h_offset);
int pb200_fr_coset_extend_host(pb200_ctx* ctx, const uint8_t* h_in, uint8_t* h_out, unsigned log_n,
                               const uint8_t* h_offset);
/* poly.py:169-177  coset_extended_lagrange_to_coeffs(offset): N values (N = 2^log_n, the extended size)
 * -> N coefficients. */
int pb200_fr_coset_to_coeffs(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, const uint8_t* h_offset);
int pb200_fr_coset_to_coeffs_host(pb200_ctx* ctx, const uint8_t* h_in, uint8_t* h_out, unsigned log_n,
                                  const uint8_t* h_offset);
/* poly.py:181-195  barycentric_eval(x) with py_ecc's inv(0) == 0 convention when x is on the domain. */
int pb200_fr_barycentric_eval(pb200_ctx* ctx, const void* d_vals, unsigned log_n, const uint8_t* h_x, uint8_t* h_out);
int pb200_fr_barycentric_eval_host(pb200_ctx* ctx, const uint8_t* h_vals, unsigned log_n, const uint8_t* h_x,
                                   uint8_t* h_out);

/* ---- G1 MSM -------------------------------------------------------------------------------- */
/* curve.py:38-44  ec_lincomb(pairs): sum_i scalars[i] * points[i].  Points must be on the curve and not
 * the identity (the facade drops None points); scalars already reduced mod r (curve.py:41).
 * n == 0 is an error (the reference raises ValueError from max(), curve.py:93). */
int pb200_g1_msm(pb200_ctx* ctx, const void* d_points, const void* d_scalars, uint64_t n, uint8_t* h_out_xy,
                 int* is_identity);
int pb200_g1_msm_host(pb200_ctx* ctx, const uint8_t* h_points, const uint8_t* h_scalars, uint64_t n,
                      uint8_t* h_out_xy, int* is_identity);

/* ---- SRS / Setup --------------------------------------------------------------------------- */
/* setup.py:16-22  Setup.powers_of_x.  h_points: n affine points (canonical).  precompute != 0 builds the
 * fixed-base window table in HBM (size ceil(256/c) * n * 64 bytes). */
int pb200_srs_create(pb200_ctx* ctx, const uint8_t* h_points, uint64_t n, int precompute, pb200_srs** out);
/* Ceremony SRS from a snarkjs .ptau, checked.  h_g1: `count` points exactly as section 2 (tauG1) stores them: x || y,
 * 32-byte little-endian Montgomery values (R = 2^256), 64 bytes per point -- the library's own device form, so the
 * bytes go to the device unconverted, in chunks through pinned staging.  h_tau_g2: [tau]_2 as section 3 stores its
 * second point (x.c0 x.c1 y.c0 y.c1, Montgomery, 128 bytes).  precompute as for pb200_srs_create.  Refused (an error;
 * nothing is kept and the context stays usable) unless every coordinate is below q (the error names the lowest bad
 * point), every point is on y^2 = x^3 + 3 and none is the identity (ditto), point 0 is the generator (1, 2), [tau]_2
 * is on the twist and r [tau]_2 = O, and e(sum r_i G_(i+1), G2) = e(sum r_i G_i, [tau]_2) for fresh 128-bit r_i from
 * getrandom(2) -- one two-vector MSM over the loaded points and one pairing product, which with the generator check
 * makes G_i = [tau^i]G for the tau of [tau]_2 except with probability about 2^-128.  Messages start "ptau: ". */
int pb200_srs_create_ptau(pb200_ctx* ctx, const uint8_t* h_g1, uint64_t count, const uint8_t* h_tau_g2, int precompute,
                          pb200_srs** out);
/* The Lagrange block of the size-n domain (n a power of two) as section 12 stores it (points n - 1 .. 2n - 2 of the
 * section, same encoding), checked like the points above and against srs_monomial (at least n powers): for random
 * values v, sum_i v_i [L_i] must equal the commitment of iNTT(v) to the monomial powers. */
int pb200_srs_create_ptau_lagrange(pb200_ctx* ctx, const uint8_t* h_block, uint64_t n, pb200_srs* srs_monomial,
                                   int precompute, pb200_srs** out);
/* Stage times (ms) of the calling thread's last pb200_srs_create_ptau / _lagrange, in this order: host-to-device copy,
 * check kernel (CUDA events), window table, random scalars, consistency MSM, pairing, [tau]_2 checks.  Stages a call
 * did not reach read 0. */
void pb200_srs_ptau_stages(double* ms, int count);
/* Structured test SRS generated on the device: points [tau^i]G, i < n, for a known (toxic) tau --
 * the 2^20 / 2^22 configurations need more powers than the reference's shipped .ptau holds
 * (setup.py:27 reads 2^11).  h_tau: canonical 32-byte Fr.  tau == 0 is refused (an error, before any device
 * work; the context stays usable): every point after the first would be the identity. */
int pb200_srs_generate(pb200_ctx* ctx, const uint8_t* h_tau, uint64_t n, int precompute, pb200_srs** out);
/* SURVEY.md 8(f) N4: the same for the Lagrange basis of the size-n domain (n a power of two): points
 * [L_i(tau)]G, i < n -- what section 12 of a snarkjs .ptau holds for the ceremony's tau.  Against such an SRS
 * Setup.commit(values) (setup.py:66-72) is ONE MSM over the values, with no inverse transform:
 * pb200_srs_commit_coeffs / _host with the LAGRANGE values in place of coefficients.  A tau with tau^n == 1 (a
 * point of the domain) is refused like tau == 0 above: L_i(tau) would be 0 for every i but one. */
int pb200_srs_generate_lagrange(pb200_ctx* ctx, const uint8_t* h_tau, uint64_t n, int precompute, pb200_srs** out);
/* copy `count` points starting at `first` back to the host (canonical x||y) */
int pb200_srs_export(pb200_ctx* ctx, pb200_srs* srs, uint8_t* h_points, uint64_t first, uint64_t count);
void pb200_srs_destroy(pb200_srs* srs);
uint64_t pb200_srs_size(pb200_srs* srs);
/* setup.py:66-72  Setup.commit(values): values in the LAGRANGE basis -> ifft -> MSM with powers_of_x.
 * n = 2^log_n must be <= srs size. */
int pb200_srs_commit_lagrange(pb200_ctx* ctx, pb200_srs* srs, const void* d_values, unsigned log_n,
                              uint8_t* h_out_xy, int* is_identity);
int pb200_srs_commit_lagrange_host(pb200_ctx* ctx, pb200_srs* srs, const uint8_t* h_values, unsigned log_n,
                                   uint8_t* h_out_xy, int* is_identity);
/* MSM of m coefficients (monomial basis) with the first m powers. */
int pb200_srs_commit_coeffs(pb200_ctx* ctx, pb200_srs* srs, const void* d_coeffs, uint64_t m, int coeffs_montgomery,
                            uint8_t* h_out_xy, int* is_identity);
/* same from host memory (canonical scalars) */
int pb200_srs_commit_coeffs_host(pb200_ctx* ctx, pb200_srs* srs, const uint8_t* h_coeffs, uint64_t m,
                                 uint8_t* h_out_xy, int* is_identity);

/* ---- Circuit preprocessing ------------------------------------------------------------------ */
/* The copy-constraint permutation of a wiring (compiler/program.py:70-113): h_ids holds 3n variable ids, row-major
 * (L, R, O of row 0, then of row 1, ...), -1 for "no variable", each in [-1, 2^32 - 2].  Every cell stores the label
 * omega^row' (col' + 1) of the previous cell carrying its id, in cell order and cyclically; all -1 cells form one more
 * cycle.  Writes S1, S2, S3 (n canonical 32-byte little-endian values each, one after the other) to h_S, exactly the
 * "S1".."S3" columns of a proving key.  Runs on the context's stream and frees its device memory before returning.
 * Refuses, before any device work, log_n outside 1..26, an id out of range (naming its cell) and more device memory
 * than is free (naming the bytes needed: 176 n bytes + the sort's temporary storage). */
int pb200_permutation(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint8_t* h_S);

/* The wire values A, B, C of a circuit from the values of its input variables, the way the reference runs a program
 * (compiler/program.py:161-192).  h_ids: 3n variable ids as pb200_permutation takes them; rows from n_constraints on
 * are unused (their ids are not read).  h_sel: QL, QR, QM, QO, QC (n canonical 32-byte little-endian values each);
 * n_custom custom gate terms as six exponents each (i, j, l, i', j', l') in h_exps, their selectors in h_custom.
 * n_inputs variables with given values: ids in h_input_ids, canonical values in h_input_values (32 bytes each).
 * A row r < n_constraints defines its O variable v when v is not -1, QO[r] != 0, no term whose selector is non-zero at
 * r reads c or the next row, v is no input and no earlier row defines v; it sets
 * c = -(QL a + QR b + QM a b + QC + sum_k Q_k a^i b^j) / QO.  Unused cells get 0.
 * h_counts[2]: the exact number of
 *   unset  cells whose variable is neither an input nor defined by a row,
 *   order  L or R cells of a defining row whose variable that row or a later row defines;
 * h_lists (3 limit uint32): the lowest `limit` unset cells (3 row + col), then `limit` (cell, defining row) pairs of
 * order cells, ascending, unused entries 0xffffffff.  With either count non-zero nothing is written to `out`;
 * otherwise out[0..2] get A, B, C (n canonical values each): device buffers when out_on_device, else host buffers.
 * Runs on the context's stream and frees its device memory before returning.  Refuses, before any device work, log_n
 * outside 1..26, an id out of range (naming its cell), an input id out of range, two inputs naming one variable, an
 * input value not reduced below r and more device memory than is free or than PB200_SOLVE_MAX_BYTES allows (naming the
 * bytes needed); afterwards, a selector value not reduced below r. */
int pb200_solve_wires(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint64_t n_constraints,
                      const uint8_t* const* h_sel, unsigned n_custom, const uint8_t* h_exps,
                      const uint8_t* const* h_custom, uint64_t n_inputs, const int64_t* h_input_ids,
                      const uint8_t* h_input_values, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists,
                      void* const* out, int out_on_device);
/* pb200_solve_wires for a circuit with lookups: rows that read a table also define their O variable from it.
 * h_qk (n x 32 bytes, 0 or 1), and the table h_t1..h_t3 (table_rows x 32 bytes each, canonical) as
 * pb200_prover_set_lookup takes them; for several tables h_qtag (Q_T) and h_t4 as pb200_prover_set_lookup_tagged takes
 * them, else both NULL.  The gate rule is unchanged.  In addition a row r < n_constraints defines its O variable v from
 * its table when q_K[r] != 0, QO[r] = 0, v is not -1, no input and not defined by an earlier row (of either kind): it
 * sets c = t3 of the table rows whose (t1, t2[, t4]) equal (a, b[, Q_T[r]]).  h_counts[4]: unset and order as
 * pb200_solve_wires counts them, then
 *   miss       rows that define from their table and whose key matches no table row,
 *   ambiguous  rows that define from their table and whose key matches table rows with different t3;
 * these two are found while the rows are evaluated, so they are counted only when unset and order are both 0.
 * h_lists (5 limit uint32): pb200_solve_wires' 3 limit entries, then the lowest `limit` miss rows and the lowest
 * `limit` ambiguous rows, unused entries 0xffffffff.  h_operands (4 limit x 32 bytes, or NULL): a and b (canonical)
 * of each listed miss row, then of each listed ambiguous row, at 64 limit bytes.  With any count non-zero nothing is
 * written to `out`.  Refuses what pb200_solve_wires refuses and, before any device work, what
 * pb200_prover_set_lookup(_tagged) refuses: q_K not 0/1, Q_T not canonical or not 0 where q_K = 0, a table value not
 * reduced below r, an empty table, more table rows than n.  The table index (about 174 bytes a table row, plus 66 bytes
 * a row for q_K, Q_T and the error flags) is counted against free memory and PB200_SOLVE_MAX_BYTES and freed before
 * the call returns. */
int pb200_solve_wires_lookup(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint64_t n_constraints,
                             const uint8_t* const* h_sel, unsigned n_custom, const uint8_t* h_exps,
                             const uint8_t* const* h_custom, uint64_t n_inputs, const int64_t* h_input_ids,
                             const uint8_t* h_input_values, const uint8_t* h_qk, const uint8_t* h_qtag,
                             const uint8_t* h_t1, const uint8_t* h_t2, const uint8_t* h_t3, const uint8_t* h_t4,
                             uint64_t table_rows, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists,
                             uint8_t* h_operands, void* const* out, int out_on_device);
/* pb200_solve_wires for a circuit with a shuffle: the out-rows get the in-rows' tuples, sorted.  h_qin, h_qout (n x 32
 * bytes, 0 or 1) as pb200_prover_set_shuffle takes them.  In-rows have q_in = 1 and q_out = 0, out-rows q_out = 1 and
 * q_in = 0 (a row with both is an ordinary row); p is the first out-row.  Out-rows define nothing by the gate rule.
 * The shuffle defines every variable on an out-row cell at row p: once every row below p is evaluated, the out-rows,
 * ascending, take the in-rows' tuples in ascending lexicographic order of (a, b, c) as canonical integers.  To unset
 * and order, out-row variables are defined at row p: a defining row at or below p that reads one is an order error
 * naming row p.  h_counts[4]: unset and order as pb200_solve_wires counts them, then
 *   late   in-row cells whose variable is defined at or after p (by the shuffle or by a row above p), not before it,
 *   clash  out-row cells that cannot take the shuffled value;
 * found before any row is evaluated.  h_lists (8 limit uint32): pb200_solve_wires' 3 limit entries, then `limit`
 * (cell, defining row) pairs of late cells, then `limit` (cell, reason, row) triples of clash cells, ascending, unused
 * entries 0xffffffff.  Reasons: 0 the cell has no variable (-1), 1 its variable is an input, 2 a row below p defines
 * it (that row is the third entry, else 0xffffffff), 3 it is on another out-row cell too.  With any count non-zero
 * nothing is written to `out`.  Without out-rows the call solves as pb200_solve_wires.  Refuses what pb200_solve_wires
 * refuses and, before any device work, a null h_qin or h_qout, a value other than 0 or 1, and unequal numbers of ones.
 * The shuffle's memory (3 bytes a row, 6 a cell, 128 an in-row) is counted against free memory and
 * PB200_SOLVE_MAX_BYTES and freed before the call returns. */
int pb200_solve_wires_shuffle(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint64_t n_constraints,
                              const uint8_t* const* h_sel, unsigned n_custom, const uint8_t* h_exps,
                              const uint8_t* const* h_custom, uint64_t n_inputs, const int64_t* h_input_ids,
                              const uint8_t* h_input_values, const uint8_t* h_qin, const uint8_t* h_qout,
                              uint32_t limit, uint64_t* h_counts, uint32_t* h_lists, void* const* out,
                              int out_on_device);
/* the last pb200_solve_wires_shuffle call on this thread that evaluated its rows: milliseconds of phase 1 (the
 * defining rows below p), the shuffle step and phase 2 (the rest), from device events; count <= 3 */
void pb200_solve_shuffle_stages(double* ms, int count);

/* ---- Prover (prover.py:39-306) ---------------------------------------------------------------- */
/* Proof layout.  A prover's proof is the plain 15 fields, then the fields of the blocks it has (next-row custom gate
 * terms, a shuffle, a lookup argument), in this order; a point is 64 bytes (x||y), a scalar 32, big-endian in a proof
 * and little-endian from the round entry points.  Within each transcript step the fields are absorbed in the same
 * order (plonkathon_b200/transcript.py holds the table).
 *
 *   kind                   bytes  fields after the plain 15, in byte order
 *   plain                    768  none
 *   next-row                 864  a_shifted_eval b_shifted_eval c_shifted_eval
 *   shuffle                  896  z3_1 qin_eval z3_shifted_eval
 *   next-row shuffle         992  the next-row three, then the shuffle three
 *   lookup (one or tagged)  1216  f_1 h1_1 h2_1 z2_1 f_eval t_eval t_shifted_eval h2_eval h1_shifted_eval z2_shifted_eval
 *
 * Each kind has its own prove and serialize entry points, and round 2 / round 4 entry points where its fields of that
 * step differ from the plain ones; each round entry point returns its step's fields in this order.  An entry point of
 * another kind returns an error naming the prover's proof size and its own entry point. */
/* prover.py:45-49  Prover(setup, program): h_pk = 8 pointers, in the order of CommonPreprocessedInput
 * (compiler/program.py:10-30): QM QL QR QO QC S1 S2 S3, each 2^log_n Lagrange values (canonical).
 * Converts them to coefficients and to a cached 4n coset extension in HBM. */
int pb200_prover_create(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                        pb200_prover** out);
/* Custom gates: the gate constraint gains  sum_k Q_k * a^i_k * b^j_k * c^l_k.  n_custom <= 4 terms; h_exps = 3 bytes
 * (i, j, l) per term, total degree 2 or 3, never (1, 1, 0) (QM's term), no triple twice; h_custom = n_custom pointers
 * to the selector columns Q_k (2^log_n Lagrange values, canonical).  The proof keeps its 768-byte form; the
 * verification key gains one commitment per term.  n_custom = 0 is pb200_prover_create. */
int pb200_prover_create_custom(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                               unsigned n_custom, const uint8_t* h_exps, const uint8_t* const* h_custom,
                               pb200_prover** out);
void pb200_prover_destroy(pb200_prover* p);
/* *out = 1 when the prover is sliced, else 0.  A one-GPU prover whose cache on the 4n coset (selector extensions, L0,
 * coset points, the per-proof extensions and quotient, the 4n NTT plans) does not fit the free device memory at
 * creation evaluates the quotient one n-point slice of the coset at a time instead: the same proofs, with the selector
 * extensions recomputed in every proof.  PB200_SLICED=1 in the environment forces it (it cannot prevent it).  A sliced
 * prover proves plain circuits and same-row custom terms; pb200_prover_set_zk(p, 1, ...), set_zk_lookup,
 * set_zk_shuffle, set_lookup(_tagged) and set_shuffle return an error on it and leave it usable, and
 * pb200_prover_create_custom_next_row fails rather than slice.  When neither layout fits, creation fails with the
 * bytes both need and the bytes free.  The sharded prover is never sliced. */
int pb200_prover_sliced(pb200_prover* p, int* out);
/* prover.py:51-84  prove(witness): h_A/h_B/h_C = wire values per row (prover.py:97-103), h_public = the
 * public input values in order (prover.py:57-62; the library negates them).  Writes the canonical 768-byte
 * proof: Proof.flatten() order (prover.py:18-35), G1 as x||y, 32-byte big-endian integers.
 * Fails (error string starts with "AssertionError") where the reference's asserts would. */
int pb200_prover_prove(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                       const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof768);
/* same, with the wire values already resident in HBM (canonical form, n x 32 bytes each) */
int pb200_prover_prove_device(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                              const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof768);
/* the individual rounds, challenges supplied by the caller's transcript; outputs little-endian */
int pb200_prover_round1(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                        const uint8_t* h_public, uint64_t n_public, uint8_t* h_abc_xy /*3*64*/);   /* prover.py:86 */
int pb200_prover_round2(pb200_prover* p, const uint8_t* beta, const uint8_t* gamma, uint8_t* h_z_xy);  /* :121 */
int pb200_prover_round3(pb200_prover* p, const uint8_t* alpha, const uint8_t* fft_cofactor,
                        uint8_t* h_t_xy /*3*64*/);                                                   /* :154 */
int pb200_prover_round4(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals /*6*32*/);             /* :228 */
int pb200_prover_round5(pb200_prover* p, const uint8_t* v, uint8_t* h_w_xy /*2*64*/);                 /* :241 */

/* The round state the reference keeps on `self` (read by its own sanity asserts, prover.py:108-116, 137-145,
 * 215-219), copied out in canonical form to a device buffer of 2^log_n elements: which = 0 A, 1 B, 2 C, 3 Z, 4 PI
 * (Lagrange values), 5 T1, 6 T2, 7 T3 (coefficients).  Valid after the round that produces them.  In zero-knowledge
 * mode which = 5..7 is an error (the blinded pieces have more than 2^log_n coefficients); 0..4 are unchanged. */
int pb200_prover_read_vector(pb200_prover* p, int which, void* d_out);
/* Zero-knowledge mode for every later proof of this prover: enable != 0 blinds per PLONK paper (11 scalars; 14 on a
 * next-row prover, see pb200_prover_create_custom_next_row).
 * h_blinders == NULL: fresh scalars from the OS CSPRNG for every proof; otherwise 11 (14) x 32-byte canonical Fr used
 * for every proof (reproducible tests).  Errors: SRS shorter than n + 6, n < 8, a sharded prover, unreduced blinders;
 * on a next-row prover an SRS shorter than n + 9 and n < 16. */
int pb200_prover_set_zk(pb200_prover* p, int enable, const uint8_t* h_blinders);
/* canonical 768-byte proof of the last rounds run on this prover (Proof.flatten() order, prover.py:18-35) */
int pb200_prover_serialize(pb200_prover* p, uint8_t* h_proof768);

/* Lookups: a plookup argument over one fixed table of three columns.  Called once, before the first proof.
 * h_qk: n x 32 bytes, q_K in {0, 1} per row; h_t1..h_t3: table_rows x 32 bytes each (canonical LE), 1 <= table_rows
 * <= n, padded to n by repeating the last row.  A row with q_K = 1 claims that (a, b, c) is a row of the table.
 * Errors: malformed input, a sharded prover, a prover in zero-knowledge mode (set the table first, then
 * pb200_prover_set_zk_lookup), a second call.
 * On a lookup prover pb200_prover_prove, _prove_device, _serialize, _round2 and _round4 return an error: a proof has
 * 13 points and 12 scalars (1216 bytes) and is made by the entry points below.  Round 1, 3 and 5 are unchanged. */
int pb200_prover_set_lookup(pb200_prover* p, const uint8_t* h_qk, const uint8_t* h_t1, const uint8_t* h_t2,
                            const uint8_t* h_t3, uint64_t table_rows);
/* Lookups over several tables, told apart by a table tag (PlonKup).  The tables are concatenated into h_t1..h_t3 and
 * h_t4 holds each table row's table id (table_rows x 32 bytes, canonical LE).  h_qtag: n x 32 bytes, Q_T = the id of
 * the table each lookup row reads, canonical and 0 wherever q_K = 0.  A row with q_K = 1 claims that (a, b, c, Q_T)
 * is a row of (t1, t2, t3, t4).  The same refusals as pb200_prover_set_lookup; proofs are made by the same entry
 * points and have the same 1216 bytes.  With t4 = Q_T = 0 the proof equals pb200_prover_set_lookup's. */
int pb200_prover_set_lookup_tagged(pb200_prover* p, const uint8_t* h_qk, const uint8_t* h_qtag, const uint8_t* h_t1,
                                   const uint8_t* h_t2, const uint8_t* h_t3, const uint8_t* h_t4, uint64_t table_rows);
/* step 1L, after round 1 and the challenge eta: commitments f_1 h1_1 h2_1 */
int pb200_prover_round_lookup(pb200_prover* p, const uint8_t* eta, uint8_t* h_fh_xy /*3*64*/);
/* round 2 with the lookup challenges: commitments z_1 z2_1 */
int pb200_prover_round2_lookup(pb200_prover* p, const uint8_t* beta, const uint8_t* gamma, const uint8_t* delta,
                               const uint8_t* epsilon, uint8_t* h_zz2_xy /*2*64*/);
/* round 4: the 6 plain evaluations, then the six lookup evaluations (Proof layout) */
int pb200_prover_round4_lookup(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals /*12*32*/);
/* the whole proof (1216 bytes, Proof layout) */
int pb200_prover_prove_lookup(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                              const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof1216);
/* same, with the wire values already resident in HBM (canonical form, n x 32 bytes each) */
int pb200_prover_prove_device_lookup(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                     const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof1216);
int pb200_prover_serialize_lookup(pb200_prover* p, uint8_t* h_proof1216);
/* Zero-knowledge lookup proofs for every later proof of a lookup prover (one table or several): enable != 0 blinds A,
 * B, C, Z and the quotient pieces as pb200_prover_set_zk does, and F, H1, H2, Z2 with 10 more scalars (21 in all,
 * DESIGN.md section 1).  h_blinders == NULL: fresh scalars from the OS CSPRNG for every proof; otherwise 21 x 32-byte
 * canonical Fr used for every proof (reproducible tests).  The proofs keep their 1216 bytes and entry points
 * (_prove_lookup, _round_lookup, _round2_lookup, _round4_lookup, _serialize_lookup) and the verifier does not change.
 * enable == 0, or pb200_prover_set_zk(p, 0, NULL), returns to plain lookup proofs.  Errors: a prover without a table,
 * a sharded prover, n < 8, an SRS shorter than n + 6, unreduced blinders; a refused call leaves the prover as it was.
 * pb200_prover_set_zk(p, 1, ...) on a lookup prover stays an error. */
int pb200_prover_set_zk_lookup(pb200_prover* p, int enable, const uint8_t* h_blinders);

/* Custom gates over the next row (TurboPLONK): h_exps = 6 bytes (i, j, l, i', j', l') per term, the term
 * Q_k * a^i b^j c^l * a(wX)^i' b(wX)^j' c(wX)^l'.  Rows are cyclic: row n - 1 reads row 0.  A term without next-row
 * exponents keeps the rules of pb200_prover_create_custom; a term with one has total degree 1, 2 or 3.  At most 4 terms,
 * none twice.  With at least one next-row term the prover is a next-row prover: round 4 also evaluates A, B, C at
 * zeta w, the zeta w opening batches them with Z, and a proof has 864 bytes.  Otherwise it is the prover
 * pb200_prover_create_custom makes.  One GPU only: there is no sharded form.
 * On a next-row prover pb200_prover_prove, _prove_device, _serialize and _round4 return an error, and so do
 * pb200_prover_set_lookup and _set_lookup_tagged (lookups do not combine with next-row terms).  Rounds 1, 2, 3 and 5
 * are the plain entry points.  pb200_prover_set_zk takes 14 blinders on a next-row prover (b12..b14 give A, B, C a
 * third blinder each) and needs n >= 16 and an SRS of n + 9 powers. */
int pb200_prover_create_custom_next_row(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                                        unsigned n_custom, const uint8_t* h_exps, const uint8_t* const* h_custom,
                                        pb200_prover** out);
/* round 4 of a next-row prover: the 6 plain evaluations, then a(zeta w), b(zeta w), c(zeta w) */
int pb200_prover_round4_next_row(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals /*9*32*/);
/* the whole proof (864 bytes, Proof layout) */
int pb200_prover_prove_next_row(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                                const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof864);
/* same, with the wire values already resident in HBM (canonical form, n x 32 bytes each) */
int pb200_prover_prove_device_next_row(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                       const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof864);
int pb200_prover_serialize_next_row(pb200_prover* p, uint8_t* h_proof864);

/* Shuffle argument: two fixed boolean selectors q_in, q_out (n x 32-byte canonical Fr, 0 or 1 on every row, as many
 * ones in each) claim that the multiset {(a_i, b_i, c_i) : q_in[i] = 1} equals {(a_i, b_i, c_i) : q_out[i] = 1}, with
 * no copy constraint between the two sides.  Set once, before the first proof.  Round 1 is unchanged; the transcript
 * then draws theta and kappa after beta and gamma, round 2 commits the grand product Z3 beside Z, round 4 adds
 * q_in(zeta) and Z3(zeta w).  A proof has 896 bytes, 992 on a next-row prover (Proof layout).  A witness whose two
 * sides differ fails round 2 with
 * "AssertionError: shuffle: the q_in rows and the q_out rows are not permutations of each other".
 * Errors, the prover left as it was: the sharded prover, a lookup table, zero-knowledge mode (set the shuffle first,
 * then pb200_prover_set_zk_shuffle), selectors already set, a selector value other than 0 / 1, unequal numbers of
 * ones.  On a shuffle prover pb200_prover_set_lookup(_tagged) and pb200_prover_set_zk(p, 1, ...) are errors, and so
 * are every prove / serialize / round 4 entry point of another proof size and the plain pb200_prover_round2.  Rounds 1,
 * 3 and 5 are the plain entry points. */
int pb200_prover_set_shuffle(pb200_prover* p, const uint8_t* h_qin, const uint8_t* h_qout);
/* Zero-knowledge shuffle proofs for every later proof of a shuffle prover: enable != 0 blinds A, B, C, Z and the
 * quotient pieces as pb200_prover_set_zk does, and Z3 with 3 more scalars, the last three: 14 in all, 17 on a
 * next-row prover (DESIGN.md section 1).  h_blinders == NULL: fresh scalars from the OS CSPRNG for every proof;
 * otherwise 14 (17) x 32-byte canonical Fr used for every proof (reproducible tests).  The proofs keep their 896 (992)
 * bytes and entry points, and the verifier does not change.  enable == 0, or pb200_prover_set_zk(p, 0, NULL), returns
 * to plain shuffle proofs.  Errors: a prover without a shuffle, a sharded prover, n < 8 and an SRS shorter than n + 6
 * (n < 16 and n + 9 on a next-row prover), unreduced blinders; a refused call leaves the prover as it was. */
int pb200_prover_set_zk_shuffle(pb200_prover* p, int enable, const uint8_t* h_blinders);
/* round 2 of a shuffle prover: z_1 then z3_1 */
int pb200_prover_round2_shuffle(pb200_prover* p, const uint8_t* beta, const uint8_t* gamma, const uint8_t* theta,
                                const uint8_t* kappa, uint8_t* h_zz3_xy /*2*64*/);
/* round 4: the plain evaluations, then the next-row (for the _next_row_shuffle form) and shuffle ones (Proof layout) */
int pb200_prover_round4_shuffle(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals /*8*32*/);
int pb200_prover_round4_next_row_shuffle(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals /*11*32*/);
int pb200_prover_prove_shuffle(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                               const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof896);
/* same, with the wire values already resident in HBM (canonical form, n x 32 bytes each) */
int pb200_prover_prove_device_shuffle(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                      const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof896);
int pb200_prover_serialize_shuffle(pb200_prover* p, uint8_t* h_proof896);
int pb200_prover_prove_next_row_shuffle(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                                        const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof992);
/* same, with the wire values already resident in HBM (canonical form, n x 32 bytes each) */
int pb200_prover_prove_device_next_row_shuffle(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                               const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof992);
int pb200_prover_serialize_next_row_shuffle(pb200_prover* p, uint8_t* h_proof992);

/* ---- Witness check: every failing constraint, without proving -------------------------------------------------------
 * Checks a witness (A, B, C per row, canonical, and the public inputs as for pb200_prover_prove) against the prover's
 * own key and reports five categories, each as an exact count and its lowest `limit` locations in ascending order:
 *   gate     rows whose gate constraint (custom and next-row terms included, PI_i = -public_i) is not 0;
 *   copy     cells c = 3 row + col whose value differs from that of sigma(c), the cell whose label omega^row' (col' + 1)
 *            is S_col[row] -- the previous cell of its cycle;
 *   key      cells whose S entry is no cell label, or repeats the label of a lower cell: S is not a permutation and no
 *            witness can prove;
 *   lookup   lookup provers: rows with q_K = 1 whose (a, b, c), or (a, b, c, Q_T) tagged, is not a row of the table;
 *   shuffle  shuffle provers: rows with q_in = 1 or q_out = 1 whose (a, b, c) occurs a different number of times among
 *            the q_in rows than among the q_out rows (a row with both selectors counts on both sides).
 * counts[5]: gate, copy, key, lookup, shuffle.  lists: gate rows (limit), copy pairs (2*limit: c, sigma(c)),
 * key cells (limit), lookup rows (limit), shuffle rows (limit) -- 6*limit uint32, ascending, unused entries 0xffffffff.
 * Equality is decided on full field elements, so for a key that is a permutation all counts are 0 iff rounds 1 and 2 of
 * a proof pass their checks (up to the proof's own soundness error).  Draws no blinders and leaves the round state and
 * every later proof unchanged.  The first call builds sigma on the device and keeps it with the prover (12n bytes);
 * every other buffer is freed before the call returns.  Refused, with the prover and the context usable afterwards: the
 * sharded prover, a null h_public with n_public > 0, more public inputs than rows, limit > 3n, values not reduced below
 * r (the prove messages), and more device memory than is free, or than PB200_CHECK_MAX_BYTES if set (naming the bytes). */
int pb200_prover_check(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                       const uint8_t* h_public, uint64_t n_public, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists);
/* same, with the wire values already resident in HBM (canonical form, n x 32 bytes each), read on the context's stream:
 * writes to them on another stream must be finished or ordered before the call */
int pb200_prover_check_device(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                              const uint8_t* h_public, uint64_t n_public, uint32_t limit, uint64_t* h_counts,
                              uint32_t* h_lists);

/* ---- multi-GPU: one process per GPU, one communicator per context (SURVEY.md 8(e)) -------------------------
 * The library issues its data-path collectives itself, on the context's stream, through NCCL (bound at run time
 * from the libnccl.so.2 the process has loaded; the single-GPU entry points work without it).  Rendezvous stays
 * with the caller: one rank draws pb200_comm_unique_id, distributes the 128 bytes (torch.distributed in
 * plonkathon_b200/parallel.py), every rank calls pb200_comm_init.  2, 4 or 8 ranks of one box. */
int pb200_comm_unique_id(uint8_t* out128);
int pb200_comm_init(pb200_ctx* ctx, const uint8_t* id128, int rank, int world);
/* rank / world of the context (0 / 1 without a communicator), data-path collectives issued so far and the bytes
 * this rank received in them */
int pb200_comm_info(pb200_ctx* ctx, int* rank, int* world, uint64_t* collectives, uint64_t* bytes_received);
/* poly.py:113-149 slab-sharded across the ranks: d_in (2^log_n elements, present on every rank; rank h reads only
 * x[h::G]) -> d_out (the full transform, on every rank).  Local 2^log_n / G-point transforms with the join twiddle
 * fused into the store, ONE allgather, then a G-point DFT per element (csrc/ntt_shard.cuh). */
int pb200_fr_ntt_sharded(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, int inverse);
/* setup.py:66-72's MSM with the 2^(c-1) signed-digit buckets split evenly over the ranks (every rank holds the
 * coefficients and an SRS replica, walks all digits, but sorts / accumulates / reduces only its buckets); ONE
 * allgather of 256 bytes per rank at the join; the same affine result on every rank. */
int pb200_srs_commit_coeffs_sharded(pb200_ctx* ctx, pb200_srs* srs, const void* d_coeffs, uint64_t m,
                                    int coeffs_montgomery, uint8_t* h_out_xy, int* is_identity);
/* prover.py:45-49 for one proof across the ranks: as pb200_prover_create, but rank r caches and works on every
 * G-th point of the 4n coset (coset extensions, selector cache and quotient divide by G), interpolations are
 * slab-sharded, commitments bucket-sharded.  Every rank calls the prove / round entry points with the same
 * inputs and gets the same 768 bytes.  A failing check (the reference's asserts) fails on every rank alike. */
int pb200_prover_create_sharded(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                                pb200_prover** out);
/* pb200_prover_create_custom for one proof across the ranks */
int pb200_prover_create_custom_sharded(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                                       unsigned n_custom, const uint8_t* h_exps, const uint8_t* const* h_custom,
                                       pb200_prover** out);
/* Operator-level shards with a caller-side join (tests, other transports): the partial sum over the SRS powers
 * [first, first+count) and the bucket magnitudes [bucket_lo, bucket_hi) of pb200_srs_bucket_count's range, as one
 * XYZZ point (128 bytes, Montgomery limbs); pb200_g1_combine_partials_host adds such partials. */
int pb200_srs_commit_partial(pb200_ctx* ctx, pb200_srs* srs, const void* d_coeffs, uint64_t first, uint64_t count,
                             uint32_t bucket_lo, uint32_t bucket_hi, int coeffs_montgomery, uint8_t* h_xyzz128);
int pb200_srs_bucket_count(pb200_srs* srs, uint32_t* out);
int pb200_g1_combine_partials_host(const uint8_t* h_xyzz, unsigned count, uint8_t* h_out_xy, int* is_identity);
/* the host half of the sharded commitment's join: h_sr = [world][sets] pairs (S = sum of the rank's buckets,
 * R = sum_j (j+1) B_j over them, j the rank's local bucket index; 2 x 128 bytes XYZZ).  nloc > 0: rank rho owns the
 * contiguous buckets [rho * nloc, (rho+1) * nloc); nloc == 0: strided ownership, rank rho owns the buckets
 * world * k + rho (what pb200_srs_commit_coeffs_sharded uses: skewed digits spread over all ranks). */
int pb200_g1_join_bucket_shards_host(const uint8_t* h_sr, unsigned world, unsigned sets, uint32_t nloc, uint8_t* h_out_xy,
                                     int* is_identity);

/* ---- Transcript (transcript.py:58-123; host code) ---------------------------------------------- */
int pb200_transcript_create(const uint8_t* label, size_t label_len, pb200_transcript** out);
void pb200_transcript_destroy(pb200_transcript* t);
int pb200_transcript_append_message(pb200_transcript* t, const uint8_t* label, size_t label_len,
                                    const uint8_t* msg, size_t msg_len);
int pb200_transcript_challenge_bytes(pb200_transcript* t, const uint8_t* label, size_t label_len, uint8_t* out,
                                     size_t n);
/* transcript.py:69-75: challenge as a canonical little-endian Fr (never zero) */
int pb200_transcript_get_and_append_challenge(pb200_transcript* t, const uint8_t* label, size_t label_len,
                                              uint8_t* out_le32);

/* ---- Pairing and G2 (host code; SURVEY.md 8(f) N3) ------------------------------------------------
 * Replaces py_ecc's `b.pairing`, `b.add`/`b.multiply` on G2 as the reference's verifier calls them
 * (TESTING_verifier_DO_NOT_OPEN.py:148-151, 237-262) and `b.is_on_curve(X2, b.b2)` (setup.py:59).
 * G1 points: 64 B x||y, G2 points: 128 B x.c0||x.c1||y.c0||y.c1 (the .ptau order, setup.py:53-58), every
 * coordinate 32-byte little-endian canonical; identity flags are one byte per point (NULL = none).
 * Points off their curve are an error; membership of the order-r subgroup of G2 is NOT checked. */
/* *ok = 1 iff  prod_i e(g1_i, g2_i) == 1  in GT */
int pb200_pairing_check(const uint8_t* h_g1, const uint8_t* h_g1_identity, const uint8_t* h_g2,
                        const uint8_t* h_g2_identity, unsigned count, int* ok);
int pb200_g2_mul(const uint8_t* h_point, const uint8_t* h_scalar_le32, uint8_t* h_out, int* is_identity);
int pb200_g2_add(const uint8_t* h_p, int p_identity, const uint8_t* h_q, int q_identity, uint8_t* h_out,
                 int* is_identity);

/* ---- micro-benchmarks (bench.py / profiles only) --------------------------------------------- */
/* runs `iters` dependent Montgomery products per thread over `threads` threads; returns elapsed ms */
int pb200_bench_modmul(pb200_ctx* ctx, int field /*0 Fr, 1 Fq*/, uint64_t threads, uint32_t iters, float* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* PLONK_B200_H */
