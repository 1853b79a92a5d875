// group-FFT instantiation unit: bls12381_g1 (coordinate field Fp<BlsFq>); the code is gfft_group.inl
#define SB_GROUP bls12381_g1
#define SB_FIELD Fp<BlsFq>
#include "gfft_group.inl"
