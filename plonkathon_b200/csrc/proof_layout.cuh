// The proof layout: every field of every proof kind, and the challenges of every transcript step.  Host code only
// (prover.cu, capi.cu and the host self-test include it); plonkathon_b200/transcript.py holds the same table.
//
// A prover has a set of blocks (next-row custom gate terms, a shuffle, a lookup argument); its proof is the table
// filtered to the plain block and those blocks, in table order.  The table lists the fields in byte order: the plain
// 15 in Proof.flatten() order, then the next-row block, the shuffle block and the lookup block.  The invariant that
// lets one table give both the byte order and the transcript order:
//
//   within each transcript step, the fields are absorbed in byte order.
//
// Every point is 64 bytes (x then y), every scalar 32.  The five kinds:
//   plain 768, next-row 864, shuffle 896, next-row shuffle 992, lookup (one table or tagged) 1216 bytes.
#pragma once
#include <cstddef>
#include <cstdint>

namespace pb200 {

// blocks: bit flags; the plain block (0) is in every proof
enum : unsigned { BLOCK_PLAIN = 0, BLOCK_NEXT_ROW = 1, BLOCK_SHUFFLE = 2, BLOCK_LOOKUP = 4 };

// transcript steps, in the order the prover runs them (1L: the lookup commitments, between rounds 1 and 2)
enum ProofStep : uint8_t { STEP_1 = 0, STEP_1L, STEP_2, STEP_3, STEP_4, STEP_5, PROOF_STEPS };

enum ProofField {
  F_A, F_B, F_C, F_Z, F_T_LO, F_T_MID, F_T_HI,
  F_A_EVAL, F_B_EVAL, F_C_EVAL, F_S1_EVAL, F_S2_EVAL, F_Z_SHIFTED_EVAL,
  F_W_Z, F_W_ZW,
  F_A_SHIFTED_EVAL, F_B_SHIFTED_EVAL, F_C_SHIFTED_EVAL,
  F_Z3, F_QIN_EVAL, F_Z3_SHIFTED_EVAL,
  F_F, F_H1, F_H2, F_Z2, F_F_EVAL, F_T_EVAL, F_T_SHIFTED_EVAL, F_H2_EVAL, F_H1_SHIFTED_EVAL, F_Z2_SHIFTED_EVAL,
  PROOF_FIELDS
};

struct ProofFieldInfo {
  const char* label;  // the transcript label (and the Python attribute)
  bool is_point;      // G1 point (64 bytes) or scalar (32 bytes)
  uint8_t step;       // ProofStep that absorbs it
  unsigned block;
};

static const ProofFieldInfo PROOF_LAYOUT[PROOF_FIELDS] = {
    {"a_1", true, STEP_1, BLOCK_PLAIN},
    {"b_1", true, STEP_1, BLOCK_PLAIN},
    {"c_1", true, STEP_1, BLOCK_PLAIN},
    {"z_1", true, STEP_2, BLOCK_PLAIN},
    {"t_lo_1", true, STEP_3, BLOCK_PLAIN},
    {"t_mid_1", true, STEP_3, BLOCK_PLAIN},
    {"t_hi_1", true, STEP_3, BLOCK_PLAIN},
    {"a_eval", false, STEP_4, BLOCK_PLAIN},
    {"b_eval", false, STEP_4, BLOCK_PLAIN},
    {"c_eval", false, STEP_4, BLOCK_PLAIN},
    {"s1_eval", false, STEP_4, BLOCK_PLAIN},
    {"s2_eval", false, STEP_4, BLOCK_PLAIN},
    {"z_shifted_eval", false, STEP_4, BLOCK_PLAIN},
    {"W_z_1", true, STEP_5, BLOCK_PLAIN},
    {"W_zw_1", true, STEP_5, BLOCK_PLAIN},
    {"a_shifted_eval", false, STEP_4, BLOCK_NEXT_ROW},
    {"b_shifted_eval", false, STEP_4, BLOCK_NEXT_ROW},
    {"c_shifted_eval", false, STEP_4, BLOCK_NEXT_ROW},
    {"z3_1", true, STEP_2, BLOCK_SHUFFLE},
    {"qin_eval", false, STEP_4, BLOCK_SHUFFLE},
    {"z3_shifted_eval", false, STEP_4, BLOCK_SHUFFLE},
    {"f_1", true, STEP_1L, BLOCK_LOOKUP},
    {"h1_1", true, STEP_1L, BLOCK_LOOKUP},
    {"h2_1", true, STEP_1L, BLOCK_LOOKUP},
    {"z2_1", true, STEP_2, BLOCK_LOOKUP},
    {"f_eval", false, STEP_4, BLOCK_LOOKUP},
    {"t_eval", false, STEP_4, BLOCK_LOOKUP},
    {"t_shifted_eval", false, STEP_4, BLOCK_LOOKUP},
    {"h2_eval", false, STEP_4, BLOCK_LOOKUP},
    {"h1_shifted_eval", false, STEP_4, BLOCK_LOOKUP},
    {"z2_shifted_eval", false, STEP_4, BLOCK_LOOKUP},
};

// the challenges each step draws after absorbing its fields, in drawing order (u: the verifier's only)
enum ProofChallenge {
  CH_BETA, CH_GAMMA, CH_THETA, CH_KAPPA, CH_ETA, CH_DELTA, CH_EPSILON, CH_ALPHA, CH_FFT_COFACTOR, CH_ZETA, CH_V, CH_U,
  PROOF_CHALLENGES
};

struct ProofChallengeInfo {
  const char* label;
  uint8_t step;
  unsigned block;
};

static const ProofChallengeInfo CHALLENGE_LAYOUT[PROOF_CHALLENGES] = {
    {"beta", STEP_1, BLOCK_PLAIN},       {"gamma", STEP_1, BLOCK_PLAIN},    {"theta", STEP_1, BLOCK_SHUFFLE},
    {"kappa", STEP_1, BLOCK_SHUFFLE},    {"eta", STEP_1, BLOCK_LOOKUP},     {"delta", STEP_1L, BLOCK_LOOKUP},
    {"epsilon", STEP_1L, BLOCK_LOOKUP},  {"alpha", STEP_2, BLOCK_PLAIN},    {"fft_cofactor", STEP_2, BLOCK_PLAIN},
    {"zeta", STEP_3, BLOCK_PLAIN},       {"v", STEP_4, BLOCK_PLAIN},        {"u", STEP_5, BLOCK_PLAIN},
};

// whether a field or challenge of `block` is part of the proof of a prover with `blocks`
inline bool block_present(unsigned block, unsigned blocks) { return block == BLOCK_PLAIN || (blocks & block); }

// the blocks that add fields to `step` (every block for step < 0: the whole proof)
inline unsigned step_blocks(int step) {
  unsigned m = 0;
  for (const ProofFieldInfo& f : PROOF_LAYOUT)
    if (step < 0 || f.step == step) m |= f.block;
  return m;
}

// bytes of `step`'s fields (of the whole proof for step < 0) on a prover with `blocks`
inline size_t layout_bytes(unsigned blocks, int step = -1) {
  size_t b = 0;
  for (const ProofFieldInfo& f : PROOF_LAYOUT)
    if ((step < 0 || f.step == step) && block_present(f.block, blocks)) b += f.is_point ? 64 : 32;
  return b;
}

}  // namespace pb200
