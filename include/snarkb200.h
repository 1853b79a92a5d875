/* snarkb200.h — C ABI of libsnarkb200.so, the H100 (sm_90a) backend for snarkjs' bulk curve operations.
 *
 * Every entry point replaces one async method of the ffjavascript `curve` object that snarkjs' provers call
 * (SURVEY.md §8b).  Citations are into snarkjs' build/snarkjs.js (first bundled copy of
 * ffjavascript@0.3.1) unless a src/ path is given.  INTEGRATION.md shows the N-API shim that binds them.
 *
 * Conventions
 *   - all pointers are HOST memory unless the name ends in _dev; buffers are little-endian;
 *   - field elements are 32 bytes (Fr, BN254 Fq) or 48 bytes (BLS12-381 Fq);
 *     "Montgomery" = x*2^(8*n8) mod p, fully reduced (reference 2873-2874, 3263-3272);
 *   - G1 affine = x||y (2*n8q), G2 affine = x.c0||x.c1||y.c0||y.c1 (4*n8q), infinity = all-zero bytes;
 *   - MSM output = Jacobian X||Y||Z Montgomery (3*n8q / 6*n8q), normalised to Z = 1 (infinity = (0,1,0));
 *     the reference returns an arbitrary projective representative, only its toAffine() is defined (§3.3);
 *   - return 0 on success, negative on error; sb_last_error(ctx) gives the message — the JS shim throws
 *     `new Error(msg)` so that error strings match the reference's;
 *   - the callee never retains caller memory (reference: inputs are sliced/copied, 14645-14646, 14739);
 *   - a context is bound to one CUDA device.  Every call locks its context for its duration, so overlapping calls on
 *     one context from several threads are safe and run one after the other (the reference awaits several bulk calls at
 *     once, 14653 / 14929-14932; an N-API shim runs them as AsyncWorkers on libuv threads).  For concurrency use one
 *     context per thread / per GPU.  sb_last_error returns the message of the calling thread's last failed call.
 */
#ifndef SNARKB200_H
#define SNARKB200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sb_ctx sb_ctx;
enum { SB_BN254 = 0, SB_BLS12_381 = 1 };
enum { SB_G1 = 1, SB_G2 = 2 };
enum {
    SB_OK = 0,
    SB_ERR_ARG = -1,        /* bad argument (message mirrors the reference's Error text) */
    SB_ERR_CUDA = -2,       /* CUDA runtime error */
    SB_ERR_NOMEM = -3,
    SB_ERR_FORMAT = -4,     /* malformed zkey / wtns */
    SB_ERR_NODEVICE = -5    /* no CUDA device: the library never falls back to the CPU */
};

/* buildBn128 / buildBls12381 + buildEngine (16413-16523, 15433-15490): one context per curve and device. */
int  sb_create(int curve, int device_id, sb_ctx** out);
void sb_destroy(sb_ctx* ctx);                       /* curve.terminate() 14259-14264 */
const char* sb_last_error(sb_ctx* ctx);
const char* sb_version(void);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t sb_launch_count(sb_ctx* ctx);

/* G1.multiExpAffine / G2.multiExpAffine (14666-14668 -> _multiExp 14605-14661).
 * n = number of points; scalar_bytes = bytes per scalar (the reference infers it as byteLength/n and throws
 * "Scalar size does not match" when not integral, 14562-14565 — the shim performs that check).
 * n == 0 -> zero point (14561, 14627). */
int sb_msm_g1_affine(sb_ctx* ctx, const uint8_t* bases, const uint8_t* scalars, uint32_t scalar_bytes, uint64_t n, uint8_t* out);
int sb_msm_g2_affine(sb_ctx* ctx, const uint8_t* bases, const uint8_t* scalars, uint32_t scalar_bytes, uint64_t n, uint8_t* out);

/* Read-only base sets (zkey sections 5-9, PLONK/fflonk PTau) registered once and kept in HBM across proofs. */
int sb_bases_register(sb_ctx* ctx, int group, const uint8_t* bases, uint64_t n, uint64_t* handle);
int sb_bases_release(sb_ctx* ctx, uint64_t handle);
/* MSM over registered bases [first, first+n) with host scalars. */
int sb_msm_registered(sb_ctx* ctx, uint64_t handle, uint64_t first, const uint8_t* scalars, uint32_t scalar_bytes, uint64_t n, uint8_t* out);
/* Same, additionally returning the un-normalised extended-Jacobian partial (X,Y,ZZ,ZZZ; 4 or 8 coordinates) that
 * sb_msm_sum_partials combines — the exchange unit of the multi-GPU MSM (one rank per GPU, SURVEY.md §8e). */
int sb_msm_registered_partial(sb_ctx* ctx, uint64_t handle, uint64_t first, const uint8_t* scalars, uint32_t scalar_bytes, uint64_t n, uint8_t* partial_out);
/* count MSMs over the same registered bases [first, first+n): scalars = count * n * scalar_bytes; out = count normalised Jacobian
 * points.  Result k equals sb_msm_registered on row k; the rows are sorted and reduced together (sub-batches sized from free
 * device memory, sb_set_tuning(14) caps them).  count == 0 writes nothing. */
int sb_msm_registered_batch(sb_ctx* ctx, uint64_t handle, uint64_t first, const uint8_t* scalars, uint32_t scalar_bytes,
                            uint64_t n, uint32_t count, uint8_t* out);
int sb_msm_sum_partials(sb_ctx* ctx, int group, const uint8_t* partials, int count, uint8_t* out);
uint32_t sb_msm_partial_bytes(sb_ctx* ctx, int group);

/* Fr.fft / Fr.ifft (15101-15107 -> _fft 14675-14918).  n must be a power of two ("fft must be multiple of 2",
 * 14745-14747) with log2(n) <= Fr.s (28 / 32).  Natural order in and out; inverse != 0 scales by 1/n. */
int sb_ntt_fr(sb_ctx* ctx, const uint8_t* in, uint64_t n, int inverse, uint8_t* out);
/* Fr.batchApplyKey (14273-14384 / frm_batchApplyKey 9458): out[i] = in[i] * first * inc^i. */
int sb_fr_batch_apply_key(sb_ctx* ctx, const uint8_t* in, uint64_t n, const uint8_t first[32], const uint8_t inc[32], uint8_t* out);
/* Fr.batchToMontgomery / Fr.batchFromMontgomery (12895-12896 -> 12780-12830). */
int sb_fr_batch_to_montgomery(sb_ctx* ctx, const uint8_t* in, uint64_t n, uint8_t* out);
int sb_fr_batch_from_montgomery(sb_ctx* ctx, const uint8_t* in, uint64_t n, uint8_t* out);
/* tm.queueAction([qap_joinABC, frm_batchFromMontgomery]) as used by joinABC, src/groth16_prove.js:320-374:
 * out[i] = fromMontgomery(a[i]*b[i] - c[i]). */
int sb_qap_join_abc(sb_ctx* ctx, const uint8_t* a, const uint8_t* b, const uint8_t* c, uint64_t n, uint8_t* out_plain);
/* Fr constants the JS side reads from the curve object: what = -1 -> Fr.shift (nqr^2), -2 -> Fr.nqr,
 * 0..s -> Fr.w[what] (12866-12889).  Returns s. */
int sb_fr_root(sb_ctx* ctx, int what, uint8_t out[32]);
/* G1/G2.fft and G1/G2.ifft (15101-15107 -> _fft 14675-14918): n points in natural order, affine (in_jacobian = 0, infinity =
 * all-zero bytes) or Jacobian (Z = 0 is infinity); out as affine or as Jacobian normalised to Z = 1 (infinity (0,1,0)),
 * the MSM output convention.  inverse != 0 gives x[k] = n^-1 X[(n-k) mod n].  n must be a power of two ("fft must be
 * multiple of 2") with log2(n) <= Fr.s; the reference's fftExt path (log2(n) = Fr.s + 1) is refused with SB_ERR_ARG.
 * Every butterfly is one variable-base scalar multiplication on the GPU.  sb_last_ms: 0 total, 1 upload, 2 compute,
 * 3 download.  G.lagrangeEvaluations (15109-15176) is the inverse transform for log2(n) <= Fr.s. */
int sb_group_fft(sb_ctx* ctx, int group, const uint8_t* in, int in_jacobian, uint64_t n, int inverse,
                 int out_jacobian, uint8_t* out);
/* G1/G2.batchApplyKey (14268-14385): out[i] = in[i] * first * inc^i (first, inc Montgomery Fr); same point formats as
 * sb_group_fft; n = 0 writes nothing. */
int sb_group_batch_apply_key(sb_ctx* ctx, int group, const uint8_t* in, int in_jacobian, uint64_t n,
                             const uint8_t first[32], const uint8_t inc[32], int out_jacobian, uint8_t* out);

/* Fused Groth16 prover (src/groth16_prove.js:28-144) with every intermediate resident in HBM.
 * sb_groth16_load parses a Groth16 .zkey image (src/zkey_utils.js:229-259 + sections 4-9), uploads the five base
 * sets and a CSR form of the coefficient section once.  sb_groth16_prove takes the witness section payload
 * (n_witness * 32 bytes, plain LE, src/wtns_utils.js:25-37) and (r, s) as 32-byte Montgomery Fr elements (the
 * reference draws them with Fr.random(), :103-104), and writes the affine proof pi_a (2*n8q) || pi_b (4*n8q) ||
 * pi_c (2*n8q), Montgomery.  public signals are witness[1..nPublic]. */
int sb_groth16_load(sb_ctx* ctx, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handle);
int sb_groth16_load_file(sb_ctx* ctx, const char* zkey_path, uint64_t* handle);
/* multi-GPU variant: this rank keeps (and builds window tables for) only its point-range shard of the five base sets;
 * the handle then serves sb_groth16_prove_shard(shard, n_shards) only. */
int sb_groth16_load_sharded(sb_ctx* ctx, const uint8_t* zkey, uint64_t zkey_len, int shard, int n_shards, uint64_t* handle);
int sb_groth16_info(sb_ctx* ctx, uint64_t handle, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_size);
int sb_groth16_prove(sb_ctx* ctx, uint64_t handle, const uint8_t* witness, uint64_t n_witness,
                     const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out);
/* full file-to-proof convenience: reads the .wtns container, checks curve and length like the reference (:44-50). */
int sb_groth16_prove_wtns(sb_ctx* ctx, uint64_t handle, const uint8_t* wtns, uint64_t wtns_len,
                          const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out);
/* same proof with the witness uploaded by the previous sb_groth16_prove on this handle still resident in HBM
 * (no host->device copy): the device-resident timing bench.py reports as `value`. */
int sb_groth16_prove_resident(sb_ctx* ctx, uint64_t handle, const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out);
/* count proofs against one loaded (unsharded) Groth16 key.  witnesses = count * n_witness * 32 bytes (section-2 payloads,
 * back to back); r, s = count * 32 bytes (Montgomery Fr); proofs_out = count * 8*n8q bytes, each laid out as sb_groth16_prove's.
 * Proof k is byte-identical to sb_groth16_prove(witness k, r k, s k).  The proofs run in sub-batches sized from free device
 * memory (sb_set_tuning(14) caps them); each sub-batch runs the QAP, NTT and MSM kernels once over all its proofs.  The
 * resident witness of sb_groth16_prove_resident is left as it was.  count == 0 writes nothing; a wrong n_witness gives
 * "Invalid witness length. Circuit: N, witness: M"; a sharded key is refused.  sb_last_ms(0) = the whole call. */
int sb_groth16_prove_batch(sb_ctx* ctx, uint64_t handle, const uint8_t* witnesses, uint64_t n_witness, uint32_t count,
                           const uint8_t* r, const uint8_t* s, uint8_t* proofs_out);
int sb_groth16_release(sb_ctx* ctx, uint64_t handle);
/* groth16Verify (src/groth16_verify.js:26-87) for count proofs against one verification key.
 * vk = alpha1 (G1) || beta2 (G2) || gamma2 (G2) || delta2 (G2) || IC[0..n_public] (G1): affine Montgomery, all-zero =
 *   infinity, i.e. the zkey's header points and section 3; vk_len must be (14 + 2 (n_public + 1)) * n8q; a vk point off its
 *   curve or a coordinate >= q: SB_ERR_ARG.
 * publics = count * n_public * 32 bytes, plain LE; proofs = count * 8*n8q bytes laid out as sb_groth16_prove writes them
 *   (a coordinate >= q counts as not on the curve).
 * status_out[k]: 0 verifies, 1 "Invalid proof", 2 "Public inputs are not valid.", 3 "Proof commitments are not valid."
 *   (checked in that reference order: 2, then 3, then 1).  As in the reference, points are checked to be on their curves
 *   (infinity included) and not for subgroup membership.  The proofs run in sub-batches of at most 2^15 (fewer for many
 *   public inputs; sb_set_tuning(14) caps them).  count == 0 writes nothing.  sb_last_ms(0) = the whole call. */
int sb_groth16_verify_batch(sb_ctx* ctx, const uint8_t* vk, uint64_t vk_len, uint32_t n_public,
                            const uint8_t* publics, const uint8_t* proofs, uint32_t count, int32_t* status_out);
/* plonkVerify (src/plonk_verify.js:29-421) / fflonkVerify (src/fflonk_verify.js:28-597) for count proofs against one
 * verification key of a circuit with n_public public signals and domain size 2^power.
 * vk (affine Montgomery points, all-zero = infinity; Fr values Montgomery, 32 bytes each):
 *   PLONK:  Qm Ql Qr Qo Qc S1 S2 S3 (G1) || X_2 (G2) || k1 || k2 (Fr): 20 n8q + 64 bytes
 *   fflonk: C0 (G1) || X_2 (G2) || k1 k2 w w3 w4 w8 wr (Fr): 6 n8q + 224 bytes; BN254 only
 * publics = count * n_public * 32 bytes, plain LE; proofs = count * sb_plonk_proof_bytes / sb_fflonk_proof_bytes, laid out as
 *   the provers write them (fflonk's inv evaluation is carried but not read).
 * status_out[k]: 0 verifies, 1 "Invalid Proof", 2 "Public inputs are not valid." (a signal >= r), 3 proof commitments not
 *   valid (a point off its curve or a coordinate >= q; no subgroup check), 4 proof evaluations not valid (a Montgomery
 *   evaluation >= r), checked in the order 3, 4, 2, then the pairing.  SB_ERR_ARG: a wrong vk_len, a null buffer, a vk point
 *   off its curve or with a coordinate >= q, power above the 2-adicity of Fr, fflonk on a BLS12-381 context.  Sub-batches,
 *   sb_set_tuning(14), count == 0 and sb_last_ms(0) as sb_groth16_verify_batch. */
int sb_plonk_verify_batch(sb_ctx* ctx, const uint8_t* vk, uint64_t vk_len, uint32_t n_public, uint32_t power,
                          const uint8_t* publics, const uint8_t* proofs, uint32_t count, int32_t* status_out);
int sb_fflonk_verify_batch(sb_ctx* ctx, const uint8_t* vk, uint64_t vk_len, uint32_t n_public, uint32_t power,
                           const uint8_t* publics, const uint8_t* proofs, uint32_t count, int32_t* status_out);
/* test hook, the device pairing (csrc/pairing.cuh) on the context's curve over n records: op 0 Fq12 mul (a, b), 1 Fq12 square,
 * 2 cyclotomic square, 3 inverse, 4 Frobenius (a -> a^q, a^(q^2), a^(q^3): three outputs), 5 Miller loop of one (G1, G2)
 * pair, 6 final exponentiation, 7 full pairing.  Tower elements are 12 Montgomery Fq coefficients in ffjavascript's order
 * (Fq12 = Fq6[w]/(w^2 - v), Fq6 = Fq2[v]/(v^3 - xi)); a pair is G1 x, y || G2 x.c0, x.c1, y.c0, y.c1, affine Montgomery, all
 * zero = infinity.  The final exponentiation raises to c (q^12 - 1)/r with c = 2x(6x^2 + 3x + 1) on BN254, 3 on BLS12-381.
 * Other ops: SB_ERR_ARG. */
int sb_pairing_eval(sb_ctx* ctx, int op, const uint8_t* in, uint64_t n, uint8_t* out);
/* ---- PLONK (src/plonk_prove.js:47-889), next-tier path per SURVEY §8f rank 3 ----------------------------------
 * sb_plonk_load: a PLONK zkey (protocol id 2, sections 2-14: src/zkey_utils.js:261-299, src/plonk_constants.js) goes to
 *   HBM once: selector / sigma / Lagrange polynomials in coefficient and 4n-evaluation form, wire maps, additions, and the
 *   PTau bases (section 14) with their MSM window tables.  Error "zkey file is not plonk" as plonk_prove.js:58-60.
 * sb_plonk_prove: witness = section 2 of the .wtns file (plain LE, nVars - nAdditions elements, plonk_prove.js:66-68);
 *   blinders = b_1..b_11 as 11 Montgomery field elements (the reference draws them with Fr.random(), :246-249);
 *   proof_out = A B C Z T1 T2 T3 Wxi Wxiw (affine Montgomery, 2*n8q bytes each) then eval_a eval_b eval_c eval_s1
 *   eval_s2 eval_zw (Montgomery, 32 bytes each): sb_plonk_proof_bytes().  Errors carry the reference's texts:
 *   "Invalid witness length. Circuit: N, witness: M, A", "Copy constraints does not match" (:436-438),
 *   "Polynomial is not divisible" (polynomial.js:608, 653), "T Polynomial is not well calculated" (:648-650), and for a key
 *   with nPublic = 0, "Evaluations.getEvaluation() out of bounds" (round 3, :613-617, where the reference reads L1 from an
 *   empty Lagrange buffer).  A witness refused at round 2 or later stays resident, so sb_plonk_prove_resident refuses it
 *   with the same text. */
int sb_plonk_load(sb_ctx* ctx, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handle);
/* same from a file: the .zkey is mapped read-only and streamed to HBM section by section (SURVEY §8f rank 2) */
int sb_plonk_load_file(sb_ctx* ctx, const char* zkey_path, uint64_t* handle);
int sb_plonk_info(sb_ctx* ctx, uint64_t handle, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_size, uint32_t* n_additions);
uint32_t sb_plonk_proof_bytes(sb_ctx* ctx);
/* the same proof from the witness the previous sb_plonk_prove on this key left in HBM (device-resident timing, and
 * re-proving with fresh blinders without a second upload) */
int sb_plonk_prove_resident(sb_ctx* ctx, uint64_t handle, const uint8_t* blinders, uint8_t* proof_out);
int sb_plonk_prove(sb_ctx* ctx, uint64_t handle, const uint8_t* witness, uint64_t n_witness, const uint8_t* blinders,
                   uint8_t* proof_out);
/* count PLONK proofs against one loaded key.  witnesses = count * n_witness * 32 bytes (wtns section-2 payloads, back to
 * back, n_witness = nVars - nAdditions); blinders = count * 11 * 32 bytes (b_1..b_11 per proof, Montgomery);
 * proofs_out = count * sb_plonk_proof_bytes(); status_out = count int32 (may be NULL).
 * Proof k is byte-identical to sb_plonk_prove(witness k, blinders k).  The proofs run in lockstep in sub-batches sized from
 * free device memory (sb_set_tuning(14) caps them): each round's kernels, NTTs and commitments run once over a sub-batch.
 * - Argument errors come before any device work: a wrong n_witness gives "Invalid witness length. Circuit: N, witness: M, A";
 *   an invalid handle or a null pointer gives SB_ERR_ARG; count == 0 writes nothing and returns SB_OK.
 * - A proof the reference would reject does not stop the others.  Its slot is zero-filled and status_out[k] holds the code of
 *   its first error: 3 "Copy constraints does not match", 4 "Polynomial is not divisible", 5 "T Polynomial is not well
 *   calculated", 6 "Evaluations.getEvaluation() out of bounds" (every proof not refused earlier, on a key with nPublic = 0);
 *   0 for a good proof.  The call then returns SB_ERR_ARG, and sb_last_error holds the text of the
 *   lowest-index failing proof.
 * - The batch's device buffers grow with the largest sub-batch and belong to the key (sb_plonk_release frees them).  When
 *   not even one proof fits, the call fails with SB_ERR_NOMEM.
 * - The resident witness of sb_plonk_prove_resident is left as it was.  sb_last_ms(0) = the whole call. */
int sb_plonk_prove_batch(sb_ctx* ctx, uint64_t handle, const uint8_t* witnesses, uint64_t n_witness, uint32_t count,
                         const uint8_t* blinders, uint8_t* proofs_out, int32_t* status_out);
int sb_plonk_release(sb_ctx* ctx, uint64_t handle);
/* ---- fflonk (src/fflonk_prove.js:51-1286), BN254 only like the reference's setup constants ----------------------
 * sb_fflonk_load: an fflonk zkey (protocol id 10, sections 2-17: src/zkey_utils.js:301-339, src/fflonk_constants.js).
 * sb_fflonk_prove: witness as for sb_plonk_prove; blinders = b_1..b_9 as 9 Montgomery field elements (:321-324);
 *   proof_out = C1 C2 W1 W2 (affine Montgomery) then the 16 evaluations ql qr qm qo qc s1 s2 s3 a b c z zw t1w t2w inv
 *   (Montgomery, 32 bytes each): sb_fflonk_proof_bytes().  Errors: "zkey file is not fflonk" (:71-73), "Invalid witness
 *   length. Circuit: N, witness: M, A" (:79-81), "Copy constraints does not match" (:649-651), "Polynomial is not
 *   divisible", "T0/T1/T2 Polynomial is not well calculated". */
int sb_fflonk_load(sb_ctx* ctx, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handle);
int sb_fflonk_load_file(sb_ctx* ctx, const char* zkey_path, uint64_t* handle);
int sb_fflonk_info(sb_ctx* ctx, uint64_t handle, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_size, uint32_t* n_additions);
uint32_t sb_fflonk_proof_bytes(sb_ctx* ctx);
int sb_fflonk_prove_resident(sb_ctx* ctx, uint64_t handle, const uint8_t* blinders, uint8_t* proof_out);
int sb_fflonk_prove(sb_ctx* ctx, uint64_t handle, const uint8_t* witness, uint64_t n_witness, const uint8_t* blinders,
                    uint8_t* proof_out);
/* count fflonk proofs against one loaded key, with the contract of sb_plonk_prove_batch: witnesses = count * n_witness * 32
 * bytes; blinders = count * 9 * 32 bytes (b_1..b_9 per proof, Montgomery); proofs_out = count * sb_fflonk_proof_bytes();
 * status_out = count int32 (may be NULL).  Proof k is byte-identical to sb_fflonk_prove(witness k, blinders k).  The proofs
 * run in lockstep in sub-batches sized from free device memory (sb_set_tuning(14) caps them).
 * - Argument errors come before any device work, as for sb_plonk_prove_batch.
 * - A proof the reference would reject does not stop the others.  Its slot is zero-filled and status_out[k] holds the code of
 *   its first error: 3 "Copy constraints does not match", 4 "Polynomial is not divisible", 5 "T0 Polynomial is not well
 *   calculated", 6 "T1 ...", 7 "T2 ...", 8 "Degree of L(X)/(ZTS2(y)(X-y)) remainder should be 0"; 0 for a good proof.  The call
 *   then returns SB_ERR_ARG, and sb_last_error holds the text of the lowest-index failing proof.  Keys with nPublic = 0
 *   prove, as with sb_fflonk_prove.
 * - The batch's device buffers grow with the largest sub-batch and belong to the key (sb_fflonk_release frees them).  When
 *   not even one proof fits, the call fails with SB_ERR_NOMEM and says how much one proof needs.
 * - The resident witness of sb_fflonk_prove_resident is left as it was.  sb_last_ms(0) = the whole call. */
int sb_fflonk_prove_batch(sb_ctx* ctx, uint64_t handle, const uint8_t* witnesses, uint64_t n_witness, uint32_t count,
                          const uint8_t* blinders, uint8_t* proofs_out, int32_t* status_out);
int sb_fflonk_release(sb_ctx* ctx, uint64_t handle);
/* ---- one PLONK / fflonk proof on several devices, each commitment sharded over the PTau point range -------------------
 * The rounds stay serial (the transcript needs every commitment before the next round), so rank 0 = ctxs[0] runs the whole
 * single-device proof (kernels, NTTs, transcript, evaluations) and only the commitments are split: the P PTau points
 * (P = n + 6 for PLONK, 9n + 18 for fflonk) go to the n contexts in the contiguous ranges sb_shard_range(P, i, n), and each
 * commitment over `len` points is the sum of one MSM partial per rank over the part of [0, len) inside its range.  Rank 0's
 * scalars reach the other ranks by CUDA peer copy (no NCCL; contexts from sb_create or sb_create_multi, several of them may
 * share one device), the partials come back to the host, and the sum is normalised there: the proof is byte-identical to
 * sb_plonk_prove / sb_fflonk_prove with the same witness and blinders.
 * sb_*_load_multi: n in 1..64 distinct contexts; the n loads run on parallel host threads.  Rank 0 holds everything
 *   sb_*_load holds except the PTau points outside its range; ranks i > 0 hold only their PTau range (with its window table
 *   when the range is large enough for one) and a receive buffer of range x 32 bytes.  Ranks on different devices get peer
 *   access to rank 0's device where the devices allow it.  If a rank fails, the handles already made are released and the
 *   call returns that rank's code, with its message on ctxs[0].  With n = 1 the call is sb_*_load.
 * Each handle is freed with sb_*_release(ctxs[i], handles[i]), and sb_*_info works on it.  sb_*_prove, sb_*_prove_resident
 *   and sb_*_prove_batch refuse every handle of a multi load with n > 1 (SB_ERR_ARG): no rank holds the whole PTau.
 * sb_*_prove_multi: handles[i] = handles_out[i] of one sb_*_load_multi call with the same contexts in the same order;
 *   witness and blinders as for sb_*_prove.  Null pointers, n outside 1..64, a context given twice, contexts of different
 *   curves and handles of another load, rank or order give SB_ERR_ARG before any device work; every other refusal has the
 *   single path's code and text (witness length, copy constraints, divisibility, T checks, PLONK keys with nPublic = 0).
 *   The call holds every context's lock for its duration.  A CUDA error on any rank is reported on ctxs[0]
 *   (sb_last_error), and sb_last_ms(ctxs[0], 0..5) mean what they mean for sb_*_prove.  With n = 1 the call is sb_*_prove. */
int sb_plonk_load_multi(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles_out);
int sb_plonk_prove_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witness, uint64_t n_witness,
                         const uint8_t* blinders, uint8_t* proof_out);
int sb_fflonk_load_multi(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles_out);
int sb_fflonk_prove_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witness, uint64_t n_witness,
                          const uint8_t* blinders, uint8_t* proof_out);
/* ---- a batch of proofs of one key on several devices --------------------------------------------------------------------
 * sb_*_load_replicas: the whole key is loaded on each of n in 1..64 distinct contexts, as sb_*_load would, on parallel host
 *   threads (each under its context's lock).  If a context fails, the handles already made are released and the call returns
 *   that context's code, with its message on ctxs[0].  Each handle is a complete key: sb_*_prove, sb_*_prove_resident,
 *   sb_*_prove_batch and sb_*_info take it on its own context, and sb_*_release(ctxs[i], handles[i]) frees it alone.
 *   sb_*_prove_multi with n > 1 refuses it (SB_ERR_ARG).
 * sb_*_prove_batch_multi: handles[i] = handles_out[i] of one sb_*_load_replicas call with the same contexts in the same
 *   order; witnesses, r / s or blinders, proofs_out and status_out (may be NULL) as for sb_*_prove_batch.
 * - Null pointers, n outside 1..64, a context given twice, contexts of different curves, and handles of another load (plain,
 *   sharded, another replicas call) or in another order give SB_ERR_ARG before any device work.  A wrong n_witness gives
 *   the single batch's "Invalid witness length..." text; count == 0 then writes nothing and returns SB_OK.
 * - The call holds every context's lock for its duration.  Rank i proves the contiguous range sb_shard_range(count, i, n) of
 *   the proofs with sb_*_prove_batch's device path on a host thread of its own (its sub-batches sized from its own device's
 *   free memory and sb_set_tuning(14)); a Groth16 rank's host work runs on max(1, cores / n) threads.  Contexts may share
 *   one device: they run on their own streams.
 * - Proof k is byte-identical to sb_*_prove_batch on one context with the same inputs.  PLONK / fflonk: a refused proof's
 *   slot is zero-filled and its status set as in sb_*_prove_batch; the call then returns SB_ERR_ARG and sb_last_error(ctxs[0])
 *   holds the text of the lowest-index refused proof.  Any other failure of a rank (a CUDA error, SB_ERR_NOMEM) is returned
 *   with that rank's message on ctxs[0], the lowest rank first, and status_out is not written.
 * - The resident witness of every context is left as it was.  sb_last_ms(ctxs[0], 0) = the host wall clock of the whole
 *   call; sb_last_ms(ctxs[i], 0), i > 0 = rank i's own batch time (0 for an empty range).  With n = 1 the call is
 *   sb_*_prove_batch. */
int sb_groth16_load_replicas(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles_out);
int sb_plonk_load_replicas(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles_out);
int sb_fflonk_load_replicas(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles_out);
int sb_groth16_prove_batch_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witnesses,
                                 uint64_t n_witness, uint32_t count, const uint8_t* r, const uint8_t* s, uint8_t* proofs_out);
int sb_plonk_prove_batch_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witnesses,
                               uint64_t n_witness, uint32_t count, const uint8_t* blinders, uint8_t* proofs_out, int32_t* status_out);
int sb_fflonk_prove_batch_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witnesses,
                                uint64_t n_witness, uint32_t count, const uint8_t* blinders, uint8_t* proofs_out, int32_t* status_out);
/* multi-GPU: this rank proves with its shard [shard, n_shards) of every MSM and returns the five un-normalised
 * MSM partials (A, B1, C, H in G1; B2 in G2) instead of a proof; the ranks exchange them (NCCL all-gather) and any
 * rank finishes with sb_groth16_finish. */
int sb_groth16_prove_shard(sb_ctx* ctx, uint64_t handle, const uint8_t* witness, uint64_t n_witness,
                           int shard, int n_shards, uint8_t* partials_out);
uint32_t sb_groth16_partials_bytes(sb_ctx* ctx);
int sb_groth16_finish(sb_ctx* ctx, uint64_t handle, const uint8_t* partials_all_ranks, int n_shards,
                      const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out);

/* ---- multi-GPU inside the library (SURVEY §8b "NCCL comm built here", §8e) -------------------------------------------
 * One context per GPU, one NCCL rank per context.  libnccl.so.2 is dlopen'ed on first use (a copy already loaded in the
 * process, e.g. torch's, is reused), so single-GPU hosts need no NCCL.
 *   multi-process (one process per GPU, torchrun / a Node cluster): rank 0 calls sb_comm_unique_id and hands the 128 bytes
 *     to the other processes over any channel; every rank calls sb_comm_init_rank, loads its key shard with
 *     sb_groth16_load_sharded(rank, world) and then sb_groth16_prove_dist per proof (a collective call).
 *   single process: sb_create_multi / sb_groth16_load_multi / sb_groth16_prove_multi do the same with one host thread per
 *     device — the _multiExp chunk fan-out (14636-14658) and the worker pool (14064-14232) replaced by GPUs.
 * What a distributed proof exchanges: each rank uploads 1/world of the witness and an all-gather over NVLink completes it;
 * the iNTT -> coset-NTT chains of A, B, C run on ranks sb_dist_chain_owner(0..2) and their evaluations are sent to the rank
 * that owns each H range; every rank multiplies its point range of the five base sets; one all-gather of the (A, C', B2)
 * partials (a few hundred bytes) ends the proof.  Proof bytes equal the single-GPU ones. */
int sb_comm_unique_id(uint8_t out[128]);
int sb_comm_init_rank(sb_ctx* ctx, int world, int rank, const uint8_t id[128]);
int sb_comm_info(sb_ctx* ctx, int* rank, int* world);      /* world = 0 when the context has no communicator */
int sb_comm_destroy(sb_ctx* ctx);
int sb_dist_chain_owner(int chain, int world);
int sb_groth16_prove_dist(sb_ctx* ctx, uint64_t handle, const uint8_t* witness, uint64_t n_witness,
                          const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out_or_null);
int sb_create_multi(int curve, const int* device_ids, int n_devices, sb_ctx** out_contexts);
int sb_groth16_load_multi(sb_ctx* const* ctxs, int n, const uint8_t* zkey, uint64_t zkey_len, uint64_t* handles_out);
int sb_groth16_prove_multi(sb_ctx* const* ctxs, const uint64_t* handles, int n, const uint8_t* witness, uint64_t n_witness,
                           const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out);

/* Host-only halves of the multi-GPU path (no context, no device needed): combine partials gathered from the ranks and
 * assemble the proof (src/groth16_prove.js:103-132).  partial = extended-Jacobian X,Y,ZZ,ZZZ Montgomery bytes;
 * Groth16 partial block = A | B1 | C | H (G1) | B2 (G2). */
int sb_host_sum_partials(int curve, int group, const uint8_t* partials, int count, uint8_t* out_jacobian);
int sb_host_partial_from_affine(int curve, int group, const uint8_t* affine, uint8_t* partial_out);
uint32_t sb_host_partial_bytes(int curve, int group);
int sb_host_groth16_finish(int curve, const uint8_t* vk_alpha1, const uint8_t* vk_beta1, const uint8_t* vk_beta2,
                           const uint8_t* vk_delta1, const uint8_t* vk_delta2, const uint8_t* partials_all_ranks, int n_shards,
                           const uint8_t r[32], const uint8_t s[32], uint8_t* proof_affine_out);
void sb_shard_range(uint64_t total, int shard, int n_shards, uint64_t* first, uint64_t* count);

/* Device-resident variants (inputs already in HBM): what bench.py's `value` times.  Pointers are device pointers
 * in this context's device; out is host memory. */
int sb_msm_dev(sb_ctx* ctx, int group, const void* bases_dev, const void* scalars_dev, uint32_t scalar_bytes, uint64_t n, uint8_t* out);
int sb_ntt_fr_dev(sb_ctx* ctx, void* data_dev, void* scratch_dev, uint64_t n, int inverse, void** result_dev);
void* sb_dev_alloc(sb_ctx* ctx, uint64_t bytes);
int sb_dev_free(sb_ctx* ctx, void* p);
int sb_dev_upload(sb_ctx* ctx, void* dst_dev, const uint8_t* src, uint64_t bytes);
int sb_dev_download(sb_ctx* ctx, uint8_t* dst, const void* src_dev, uint64_t bytes);
/* timing of the last call on this context, measured with CUDA events on the context's stream (ms):
 * which = 0 total device time of the call, 1.. = per-stage breakdown where the call defines one.
 * sb_plonk_prove / sb_fflonk_prove: 1..5 = host wall clock of rounds 1..5 (each round ends on a synchronising commit). */
float sb_last_ms(sb_ctx* ctx, int which);
/* counters of the last MSM / prove call: 0/1 = summed device time (ms) of the G1 / G2 bucket-accumulation kernel
 * launches, 2/3 = number of those launches, 4/5 = (scalar digit, point) entries they consumed; 8..15 = device time (ms) per
 * kernel class: digits + radix sort, G1 accumulation, G2 accumulation, head folding, bucket reduction + window sums,
 * QAP rows, NTT passes, joinABC (meaningful per class when the call ran serialised, sb_set_tuning(2, 1)); 16/17 = the part
 * of 11/12 (head folding / bucket reduction) spent in G2 MSMs. */
double sb_last_stat(sb_ctx* ctx, int which);
/* integer-pipe calibration on this device: what = 0 -> IMAD.WIDE.U32 per second, 1 -> register-resident BN254 Fq
 * Montgomery multiplies per second (the modmul-bound roofline denominators, SURVEY.md §8d). */
double sb_calibrate(sb_ctx* ctx, int what);
/* process-wide switches for profiling and tests (every setting computes the same bytes); SB_ERR_ARG for any other key:
 *   1  bucket reduction: 0 = axis sums + warp-shuffle weighted sums (default), 1 = running sums (k_reduce, the path for
 *      windows of more than 2^20 buckets)
 *   2  1 = run every stream of a prove call serialised on one stream (per-kernel-class timing, sb_last_stat 8..15)
 *   3  1 = ignore the precomputed window tables (plain windowed Pippenger on the raw bases)
 *   6  log2 of the points per MSM chunk, 1..23 (test hook; 0 = default: 2^23, the largest chunk the sort and the batch
 *      limits are sized for)
 *   7  log2 of the largest NTT tile (10..12; default 11, the value to restore: 0 is refused)
 *   8  0 = no pinned staging of pageable host buffers
 *  13  MSM window bits c, 3..22 (test hook; 0 = default: chosen from the number of points).  Applies wherever a geometry
 *      is chosen: per chunk for MSMs on unregistered bases, and for window tables when they are built, i.e. when bases are
 *      registered or a key is loaded; a table keeps the c in force at that moment.  Tables are still skipped when
 *      W * n >= 2^31.  A large c costs memory: a plain MSM allocates W * 2^(c-1) buckets.
 *  14  most proofs per sub-batch of sb_groth16_prove_batch, sb_plonk_prove_batch, sb_fflonk_prove_batch and
 *      sb_groth16_verify_batch, sb_plonk_verify_batch, sb_fflonk_verify_batch, and rows per sub-batch of
 *      sb_msm_registered_batch (test hook;
 *      0 = default: as many as the 32-bit bucket keys and free device memory allow)
 * The Python mirror applies SB_TUNE="key=value,..." from the environment when it loads the library. */
int sb_set_tuning(int key, int value);
/* synthetic bases for tests/benchmarks: chunks of 4096 points P_{c,j} = (k0(seed, c) + j*kd(seed)) * G, affine Montgomery, computed
 * on the GPU; the same points as the CPU oracle's incremental generator (oracle/snark_oracle.cpp or_gen_points), see msm.cuh. */
int sb_gen_points(sb_ctx* ctx, int group, uint64_t seed, uint64_t n, uint8_t* out);
int sb_generator(sb_ctx* ctx, int group, uint8_t* out_affine);
/* test hook: one field primitive of the device arithmetic (csrc/fp.cuh, csrc/ec.cuh) over n records, as compiled for the
 * GPU.  The field does not depend on the context's curve; the context supplies the device, stream and buffers.
 *   field: 0 BN254 Fq, 1 BN254 Fr, 2 BLS12-381 Fq, 3 BLS12-381 Fr, 4 BN254 Fq2, 5 BLS12-381 Fq2
 *   in: n records of k little-endian elements (N limbs of 32 bits each: 32 or 48 bytes; an Fq2 element is c0 || c1),
 *   out: n results.  Values are raw residues: "Montgomery" operations compute with R = 2^(32N).
 *   op  fields  in -> out
 *    0  0-3     a, b -> a + b                      7  0-3   T (2N limbs, T < p*R) -> T*R^-1
 *    1  0-3     a, b -> a - b                      8  0-3   a -> a*R (to_mont; any a < 2^(32N))
 *    2  0-3     a -> -a                            9  0-3   a -> a*R^-1 (from_mont; any a < 2^(32N))
 *    3  0-3     a -> 2a                           10  0-3   a -> R^2*a^-1, 0 -> 0 (binary inversion)
 *    4  0-3     a, b -> a*b*R^-1 (mul)            11  0-3   a -> R^2*a^-1, 0 -> 0 (a^(p-2))
 *    5  0-2     x, y, u, v -> (x*y + u*v)*R^-1    12  4-5   x, y -> x*y*R^-1 (dual-product schoolbook)
 *               (mul2: not on BLS12-381 Fr)       13  4-5   x, y -> x*y*R^-1 (lazy Karatsuba)
 *    6  0-3     a, b -> a*b (2N limbs)            14  4-5   x -> x^2*R^-1      15  4-5   x -> R^2*x^-1, 0 -> 0
 *   Point ops (csrc/ec.cuh, a = 0 curves) name the group by its base field: 0 BN254 G1, 2 BLS12-381 G1, 4 BN254 G2,
 *   5 BLS12-381 G2.  Coordinates are Montgomery elements of that field; an affine point is x, y, an XYZZ point
 *   x, y, zz, zzz (x = X/ZZ, y = Y/ZZZ, infinity: zz = 0; the results write infinity as all zeros).
 *   16  0,2,4,5  acc (XYZZ), q (affine) -> acc.add_affine(q)   q must not be infinity, (0, 0): the MSM drops such bases
 *   17  0,2,4,5  acc, q (XYZZ) -> acc.add_i(q)                 (the inlined addition of the MSM reduction kernels)
 *   18  0,2,4,5  acc, q (XYZZ) -> acc.add(q)
 *   19  0,2,4,5  p (XYZZ) -> dbl(p)                 20  0,2,4,5  p (affine) -> dbl_affine(p)
 * Operands other than to_mont / from_mont inputs must be below p.  Any other (field, op) pair is SB_ERR_ARG. */
int sb_field_eval(sb_ctx* ctx, int field, int op, const uint8_t* in, uint64_t n, uint8_t* out);
/* test hook: `count` Fr transforms of n = 2^L elements of the context's curve through the launches the provers use:
 * layout 0 runs fr_ntt_batch (count 1..4, each transform and its scratch at its own device offset, as Groth16's A, B, C),
 * layout 1 runs fr_ntt_strided (count 1..65535 transforms back to back, as a batch of proofs).  inverse selects the
 * twiddle table and does not scale; pre_first / pre_inc (both or neither) = the pre-multiplier first * inc^i by input
 * position i on the first pass; post_scale = optional factor on the last pass.  Host in / out, count * n * 32 bytes,
 * Montgomery, transform k at k * n * 32.  Every part of the device region is followed by a guard of sentinel bytes; a
 * launch that writes into one fails the call with SB_ERR_CUDA.  L outside 0..Fr.s, count outside the layout's range, a
 * layout other than 0 or 1, a null buffer or half a pre-multiplier is SB_ERR_ARG. */
int sb_ntt_eval(sb_ctx* ctx, int L, int count, int layout, int inverse, const uint8_t* pre_first, const uint8_t* pre_inc,
                const uint8_t* post_scale, const uint8_t* in, uint8_t* out);
int sb_sync(sb_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif
