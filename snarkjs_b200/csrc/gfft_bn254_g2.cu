// group-FFT instantiation unit: bn254_g2 (coordinate field Fp2<BnFq>); the code is gfft_group.inl
#define SB_GROUP bn254_g2
#define SB_FIELD Fp2<BnFq>
#include "gfft_group.inl"
