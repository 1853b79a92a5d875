// group-FFT instantiation unit: bn254_g1 (coordinate field Fp<BnFq>); the code is gfft_group.inl
#define SB_GROUP bn254_g1
#define SB_FIELD Fp<BnFq>
#include "gfft_group.inl"
