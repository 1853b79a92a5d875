// verifier instantiation unit: BLS12-381 (base field Fp<BlsFq>); the code is verify_curve.inl
#define SB_CURVE bls12381
#define SB_FQ BlsFq
#include "verify_curve.inl"
