// Device buffers and kernel launchers of the BLS batch-verification pipeline (see bls_engine.cu for the flow).
#pragma once
#include <cstddef>
#include <cstdint>

#include "groups.cuh"
#include "fp12.cuh"

namespace b200 {

// G1 operand of the lane-parallel Miller loop: (X Z, Y, Z^3) of a Jacobian point (affine point: (x, y, 1)); the line
// functions absorb the Z^3 scaling, so the aggregate key is never inverted
struct G1Pre {
    Fp xz, y, z3;
    uint32_t inf;
};

// per-tuple flags written by the G1 aggregation kernel
enum : uint32_t { TUPLE_FLAG_EMPTY = 1u, TUPLE_FLAG_AGG_INF = 2u };
// per-signature status written by the signature kernel
enum : int32_t { SIG_OK = 0, SIG_NOT_IN_GROUP = -1 };  // >0: blst decode error code

// K1: key_validate every 48-byte public key -> affine point + blst code
void set_g1_small_n(uint32_t n);
void set_small_cta(int threads);
void set_vm_team16_max(uint32_t n);
void set_vm_cta(int threads);
// cta = 0: by batch size (384-thread CTAs above the small-batch bound, 128 below); 128 / 384 force one (default variant only)
void launch_g1_validate(const uint8_t* keys, uint32_t n, G1Aff* out, int32_t* codes, void* stream, int cta = 0);
// K1's input from n 121-byte Validator records in device memory (public key first): keys[48 i ..] = records[121 j ..][0, 48)
// with j = i, or j = index[i] when `index` (device) is given; `keys` 16-byte aligned
void launch_gather_validator_keys(const uint8_t* records, uint32_t n, uint8_t* keys, void* stream, const uint64_t* index = nullptr);
// K2: per tuple t, sum the validated keys [off[t], off[t+1]) (or gather through `index` when non-null);
//     first failing key (in order) decides pk_code[t]
//     agg == nullptr: only the code scan (aggregate_verify keeps keys separate); extra_flags is OR-ed into flags
//     agg_pre != nullptr: write the un-normalised sum for the VM Miller kernel instead of the affine point
//     tuple_flags != nullptr: per-tuple flags OR-ed into flags[t] as well (aggregate_verify batches: a tuple whose key and
//     message counts differ is flagged EMPTY)
void launch_g1_aggregate(const G1Aff* keys, const int32_t* key_codes, const uint32_t* index, const uint32_t* off,
                         uint32_t n_tuples, G1Aff* agg, G1Pre* agg_pre, int32_t* pk_code, uint32_t* flags,
                         uint32_t extra_flags, void* stream, G1Jac* agg_jac = nullptr, const uint32_t* tuple_flags = nullptr);
// aggregate_verify batches: the G1 operand of key i's pair, keys[i] (or keys[index[i]] when index is non-null), as the VM
// Miller kernel's G1Pre (x, y, 1) into pre[i]
void launch_g1_pair_operands(const G1Aff* keys, const uint32_t* index, uint32_t n, G1Pre* pre, void* stream);
// RLC whole-batch check (bls_rlc.cu): scale per tuple, fold 32 -> 1 per launch, sum -> affine
void launch_rlc_scale(const G1Jac* agg, const G2Aff* sig, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code,
                      const uint32_t* seed_words, uint64_t t0, uint32_t n, G1Pre* out_g1, G2Jac* out_g2, int32_t* bad, void* stream);
uint32_t launch_rlc_reduce(const Fp12* f_in, const G2Jac* q_in, uint32_t n, Fp12* f_out, G2Jac* q_out, void* stream);
void launch_rlc_finish(const G2Jac* q, G2Aff* out, void* stream);
void launch_fp12_one(Fp12* out, void* stream);
// Segmented Gt product, one level (bls_rlc.cu): segment t holds values in[seg_in[t] .. seg_in[t+1]) of the n_in inputs and
// seg_of[i] names value i's segment.  Each 32-value chunk of the input goes to one warp; the part ("piece") of a segment
// inside chunk c, its k-th, leaves as one product: to out[seg_out[t] + k], or with seg_out == nullptr (a level after which
// every segment has at most two pieces) to out[2t + k], with Fp12 one at out[2t + 1] for a segment of one piece -- the
// layout launch_vm_final reads with pair_off[t] = 2t.  With pk_code non-null the segments of failed tuples are skipped.
void launch_fold_segments(const Fp12* in, uint32_t n_in, const uint32_t* seg_of, const uint32_t* seg_in, const uint32_t* seg_out,
                          const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code, Fp12* out, void* stream);
// K3: decompress + subgroup-check every 96-byte signature
//     `threads`: CTA size (32 = spread for latency, 512 = pack onto few SMs while the per-key kernel runs)
void launch_g2_sig_decode(const uint8_t* sigs, uint32_t n, G2Aff* out, int32_t* sig_code, void* stream);
// K4: hash_to_G2 of message i = bytes [moff[i], moff[i+1]) of `msgs`
//     `tmp_jac`: scratch for 2n Jacobian G2 points (288 B each)
void launch_hash_to_g2(const uint8_t* msgs, const uint32_t* moff, uint32_t n, G2Aff* out, void* tmp_jac, void* stream);
// the lane-parallel pairing VM (bls_vm.cu); vm_init returns 0 on success
int vm_init(void* stream);
// replaces one team size's scheduled programs (blob layout: bls_vm.cu); returns 0 on success, 1 on a malformed blob
int vm_load_programs(const uint32_t* blob, size_t n_words, void* stream);
// K5: one Miller loop per pair (g1[g1_idx[i]], g2[g2_idx[i]]); pairs whose tuple already failed are skipped
// K6: per tuple: merge codes with the reference's precedence, final exponentiation of f[pair_off[t]] f[pair_off[t] + 1]
void launch_vm_miller(const G1Pre* g1, const uint32_t* g1_idx, const G2Aff* g2, const uint32_t* g2_idx,
                      const uint32_t* pair_tuple, const int32_t* pk_code, const uint32_t* flags, const int32_t* sig_code,
                      uint32_t n_pairs, Fp12* f, void* stream);
void launch_vm_final(const Fp12* f, const uint32_t* pair_off, const int32_t* pk_code, const uint32_t* flags,
                     const int32_t* sig_code, uint32_t n_tuples, int32_t* out_codes, void* stream);
// `aggregate` over T groups (group g: signatures off[g] .. off[g+1]-1, decoded by K3) in one launch: per chunk of
// `chunk` signatures (g2_aggregate_chunk) its first failure and partial sum; the warp that completes a group's last chunk
// writes the group's verdict and compressed sum (out96[96 g..], zero unless out_code[g] == 0).  Chunks of group g:
// chunk_off[g] .. chunk_off[g+1]-1, at least one per group (empty groups too); chunk c belongs to chunk_group[c].
// `part` / `part_code` hold n_chunks entries; `done` holds T counters, zero at launch.
uint32_t g2_aggregate_chunk(uint32_t n_sigs);
void launch_g2_aggregate(const G2Aff* sigs, const int32_t* sig_code, const uint32_t* off, const uint32_t* chunk_group,
                         const uint32_t* chunk_off, uint32_t n_chunks, uint32_t chunk, G2Jac* part, int32_t* part_code,
                         uint32_t* done, uint8_t* out96, int32_t* out_code, void* stream);
// `eth_aggregate_public_keys` over T groups after K2 (affine sums, codes, flags): code and compressed sum per group
void launch_g1_compress_groups(const G1Aff* agg, const int32_t* pk_code, const uint32_t* flags, uint32_t n_groups, uint8_t* out48,
                               int32_t* out_code, void* stream);
// writes -g1 (the negated generator) in its G1Pre form to *out_pre
void launch_neg_g1(G1Pre* out_pre, void* stream);
// on-device self-test of Fp arithmetic (portable vs tuned paths), returns mismatches in *out
void launch_fp_selftest(uint32_t n, uint32_t seed, uint32_t* out_mismatch, void* stream);
// on-device self-test: one field operation on n raw operand pairs, for comparison with big integers on the host.
// Operand slots are kFpEvalIn words (Fp: words 0..11; Fp2: c0 in 0..11, c1 in 12..23), result slots kFpEvalOut words
// (the same limbs, then one flag word: carry, borrow, "is a square", lex-largest or sgn0).  Limbs are little-endian 32-bit
// words of the raw representative (Montgomery form where the operation works in it).
enum : int32_t {
    FP_EVAL_MUL = 0, FP_EVAL_SQR = 1, FPL_EVAL_MUL = 2, FPL_EVAL_SQR = 3,
    FP_EVAL_ADD = 4, FP_EVAL_SUB = 5, FP_EVAL_NEG = 6, FPL_EVAL_ADD = 7, FPL_EVAL_SUB = 8, FPL_EVAL_NEG = 9,
    FP_EVAL_ADD_RAW = 10, FP_EVAL_SUB_RAW = 11, FP_EVAL_INV_KALISKI = 12, FP_EVAL_INV_FERMAT = 13,
    FP_EVAL_SQRT = 14, FPL_EVAL_POW_SQRT = 15, FP_EVAL_IS_LEX_LARGEST = 16,
    FP_EVAL_N_OPS = 17,                                              // bls_g1.cu: the per-key kernel's build
    FPL_EVAL_SQRT_CHAIN = 18,                                        // bls_g1.cu as well; 17 stays unassigned
    FPL_EVAL_MUL_SUB_MUL = 19, FPL_EVAL_MUL_SUB_8SQR = 20,            // bls_g1.cu: (a0 a1 - b0 b1)/R, (a0 a1 - 8 b0^2)/R
    FPL_EVAL_END = 21,                                               //   (a0 / a1: words 0..11 / 12..23 of operand a)
    FP2_EVAL_MUL = 32, FP2_EVAL_SQR = 33, FP2_EVAL_INV = 34, FP2_EVAL_SQRT = 35, FP2_EVAL_SGN0 = 36,
    FP2_EVAL_END = 37,                                               // bls_g2.cu: the signature / hash kernels' build
    // bls_g1.cu: the FP64 field of the split per-key kernel (fpd.cuh).  An FpD operand or result is words 0..15 of its
    // slot, 8 little-endian binary64 limbs (limb k an integer multiple of 2^(48k)), taken and returned as raw bits
    FPD_EVAL_MUL = 40, FPD_EVAL_SQR = 41, FPD_EVAL_ADD = 42,          // FpD -> FpD
    FPD_EVAL_FROM_FP = 43,                                           // Fp limbs (below 2^384 - 2^383) -> FpD
    FPD_EVAL_TO_FPL = 44,                                            // FpD (|a| < 2p) -> Fp limbs in [0, 2p)
    FPD_EVAL_SQRT_CHAIN = 45,                                        // Fp -> fpd_to_fpl(fpd_sqrt_chain(fpd_from_fp(a)))
    FPD_EVAL_Y_FROM_X = 46,                                          // a: canonical Montgomery x, b word 0: sign flag ->
                                                                     //   g1_y_from_x_fpd's y, flag = on the curve
    FPD_EVAL_END = 47
};
constexpr uint32_t kFpEvalIn = 24, kFpEvalOut = 25;
void launch_fp_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream);
void launch_fp2_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream);
// on-device self-test of single curve stages (b200_curve_eval).  Records of kCurveEvalWords words: X, Y, Z as 24-word
// slots (Fp in the first 12 words, Fp2 as c0 then c1), then a flag word: in, the affine infinity flag of operand a; out,
// the subgroup verdict or the infinity flag of an affine result.  Affine operands are (X, Y) with Z ignored.
enum : int32_t {
    CURVE_G1L_ADD_MIXED = 0, CURVE_G1L_ADD = 1, CURVE_G1L_IN_SUBGROUP = 2,
    CURVE_G1_N_OPS = 3,                                              // bls_g1.cu on FpL: the per-key kernel's formulas
    CURVE_G1L_DOUBLE = 4,                                            // bls_g1.cu as well; 3 stays unassigned
    CURVE_G1_IN_SUBGROUP_ISO = 6,                                    // bls_g1.cu: g1_in_subgroup_iso(X), the split kernel's
                                                                     //   check from x alone; 5 stays unassigned
    CURVE_G2_ADD = 32, CURVE_G2_ADD_MIXED = 33, CURVE_G2_DOUBLE = 34, CURVE_G2_IN_SUBGROUP = 35, CURVE_G2_PSI = 36,
    CURVE_G2_CLEAR_COFACTOR = 37, CURVE_G2_SSWU_ISO = 38, CURVE_G2_H2C_FINISH = 39,
    CURVE_G2_END = 40                                                // bls_g2.cu: the signature / hash kernels' build
};
constexpr uint32_t kCurveEvalWords = 73;
void launch_curve_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream);
void launch_curve2_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream);
// on-device self-test of the pairing (b200_pairing_eval).  Records of kPairingEvalWords words: twelve 12-word Fp slots in
// Fp12 memory order (c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1), raw Montgomery limbs, then a flag word.  Points and
// lines use the leading slots: G1 affine x, y; G1Pre xz, y, z3; G2 affine x.c0, x.c1, y.c0, y.c1; G2 Jacobian x, y, z as
// six slots; a line (A, B, C) as six slots.  The input flag is the infinity flag.
enum : int32_t {
    PAIRING_EVAL_FP6_MUL = 0, PAIRING_EVAL_FP6_INV = 1, PAIRING_EVAL_FP12_MUL = 2, PAIRING_EVAL_FP12_SQR = 3,
    PAIRING_EVAL_FP12_INV = 4, PAIRING_EVAL_FP12_MUL_BY_LINE = 5, PAIRING_EVAL_FP12_FROB1 = 6, PAIRING_EVAL_FP12_FROB2 = 7,
    PAIRING_EVAL_FP12_CYCLO_SQR = 8, PAIRING_EVAL_FP12_POW_Z = 9,
    PAIRING_EVAL_MILLER_DOUBLE = 10, PAIRING_EVAL_MILLER_ADD = 11,   // a: T (Jacobian); b: Q affine (add), xP, yP in slots 4, 5
                                                                     // out: T' in slots 0..5, A B C in 6..11
    PAIRING_EVAL_MILLER_LOOP = 12, PAIRING_EVAL_FINAL_EXP = 13,      // final_exp: the value, flag = final_exp_is_one
    PAIRING_EVAL_END = 14,                                           // bls_pairing.cu: the one-thread kernels' build
    PAIRING_EVAL_VM_MILLER8 = 32, PAIRING_EVAL_VM_MILLER16 = 33,     // a: G1Pre, b: G2 affine -> the kernel's Fp12
    PAIRING_EVAL_VM_FINAL8 = 34, PAIRING_EVAL_VM_FINAL16 = 35,       // a: f0, b: f1 -> the six program outputs, flag = verdict
    PAIRING_EVAL_VM_END = 36,                                        // bls_vm.cu, teams of 8 / 16 lanes under vm_cta
    PAIRING_EVAL_FOLD_FP12 = 48, PAIRING_EVAL_FOLD_G2 = 49,          // n inputs of a (Fp12 / G2 Jacobian) -> record 0: the
                                                                     // product / the affine sum (flag: infinity); bls_rlc.cu
    PAIRING_EVAL_FOLD_SEGMENTS = 50,                                 // a: n Fp12 values; b: words b[0] = T, b[1 .. T+1] = segment
                                                                     // offsets (from 0, non-decreasing, <= n; 2T <= n) -> records
                                                                     // 2t, 2t + 1: the two values segment t folds to (zero when empty)
    PAIRING_EVAL_FOLD_END = 51
};
constexpr uint32_t kPairingEvalWords = 145;
void launch_pairing_eval(int32_t op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out, void* stream);
// the production VM kernels at an explicit team size, with identity indices and every tuple alive; pair_off: 0, 2, 4, ...;
// f_out: the final program's six outputs per tuple (Fp12 memory order), next to its verdict in codes
void launch_vm_miller_team(int team, const G1Pre* g1, const uint32_t* idx, const G2Aff* g2, const uint32_t* zeros, uint32_t n,
                           Fp12* f, void* stream);
void launch_vm_final_team(int team, const Fp12* f, const uint32_t* pair_off, const uint32_t* zeros, uint32_t n, Fp12* f_out,
                          int32_t* codes, void* stream);

}  // namespace b200
