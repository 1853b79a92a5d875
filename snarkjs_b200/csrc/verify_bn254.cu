// verifier instantiation unit: BN254 (base field Fp<BnFq>), with the fflonk verifier; the code is verify_curve.inl
#define SB_CURVE bn254
#define SB_FQ BnFq
#define SB_PV_FFLONK
#include "verify_curve.inl"
