// verifier instantiation unit: BN254 (base field Fp<BnFq>); the code is verify_curve.inl
#define SB_CURVE bn254
#define SB_FQ BnFq
#include "verify_curve.inl"
