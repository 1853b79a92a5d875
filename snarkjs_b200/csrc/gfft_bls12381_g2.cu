// group-FFT instantiation unit: bls12381_g2 (coordinate field Fp2<BlsFq>); the code is gfft_group.inl
#define SB_GROUP bls12381_g2
#define SB_FIELD Fp2<BlsFq>
#include "gfft_group.inl"
