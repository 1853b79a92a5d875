// pairing.cuh — the optimal-ate pairing on BN254 and BLS12-381 for the device Groth16 verifier, templated on the base
// field like ec.cuh.  Every function is __host__ __device__: the host computes with the same code (fp.cuh's host multiply).
//
// Tower (ffjavascript's): Fq2 = Fq[u]/(u^2 + 1) (ec.cuh), Fq6 = Fq2[v]/(v^3 - xi), Fq12 = Fq6[w]/(w^2 - v), xi = 9 + u on
// BN254 and 1 + u on BLS12-381.  An Fq12 element is 12 Fq coefficients in the order c0.c0.a, c0.c0.b, c0.c1.a, ...,
// c1.c2.b, i.e. the Fq2 coefficient of w^(2j + k) sits at c_k.c_j.
//
// Miller loop.  G2 points live on the sextic twist: D-type on BN254 (y^2 = x^3 + 3/xi, untwisted by (x w^2, y w^3)),
// M-type on BLS12-381 (y^2 = x^3 + 4 xi, untwisted by (x / w^2, y / w^3)).  The running point is homogeneous projective
// (X, Y, Z) over Fq2, so no step inverts; each doubling or addition yields a line with three Fq2 coefficients, scaled by the
// G1 point's x and y and multiplied into f as a sparse element (w^0, w^1, w^3 on BN254, w^0, w^2, w^3 on BLS12-381).  Lines
// differ from the affine ones by factors in proper subfields of Fq12, which the final exponentiation removes.
//   BN254:     the bits of 6x + 2 below its top bit (64 doublings, 36 additions), then additions of pi(Q) and -pi^2(Q)
//              (pi = the q-power Frobenius, on the twist (conj(x) gamma(1,2), conj(y) gamma(1,3)), etc.).
//   BLS12-381: the bits of |x| = 0xd201000000010000 below its top bit (63 doublings, 5 additions); x < 0, so f is
//              conjugated at the end.
// A pair with either point at infinity contributes 1.  Nothing here checks subgroup membership: on-curve points outside
// the r-torsion go through the same formulas, as in the reference's pairingEq.  (A G2 point of tiny order, for which the
// running point would meet +-Q, would give a degenerate line; no such point lies on either twist's subgroup.)
//
// Final exponentiation.  Easy part f^((q^6 - 1)(q^2 + 1)), then a hard part by an addition chain in x that computes a
// fixed multiple c of (q^4 - q^2 + 1)/r:
//   BN254:     c = 2x(6x^2 + 3x + 1), x = 4965661367192848881 (Fuentes-Castaneda, Knapp, Rodriguez-Henriquez)
//   BLS12-381: c = 3 (Hayashida, Hayasaka, Teruya)
// gcd(c, r) = 1 on both curves, so e(P, Q) = 1 exactly when the textbook f^((q^12 - 1)/r) is 1: every verdict is the same.
#pragma once
#include "ec.cuh"

namespace sb {

// gamma(k, i) = xi^(i (q^k - 1) / 6), the Frobenius coefficients (row 5(k-1) + i-1), generated from the formula with Python
// big integers; the twist's b; 1/2.  Montgomery limbs.
#define SB_PAIR_BNFQ_FROB SB_L(0x33144907u, 0xaf9ba696u, 0x87afb78au, 0xca6b1d73u, 0xf08a2087u, 0x11bded5eu, 0x1a1f3a7cu, 0x02f34d75u, 0x4c492d72u, 0xa222ae23u, 0x565de15bu, 0xd00f02a4u, 0x53dfc926u, 0xdc2ff3a2u, 0xb3899551u, 0x10a75716u, \
    0x4563ab30u, 0xb5773b10u, 0xa9aa6454u, 0x347f91c8u, 0x242e0991u, 0x7a007127u, 0x118214ecu, 0x1956bcd8u, 0xa0aa4757u, 0x6e849f1eu, 0x89f89141u, 0xaa1c7b6du, 0xfae0ca3au, 0xb6e713cdu, 0x4e82ebc3u, 0x26694fbbu, \
    0x2936b629u, 0xe4bbdd0cu, 0xe133bacbu, 0xbb30f162u, 0xf9645366u, 0x31a9d1b6u, 0xa500f8ddu, 0x253570beu, 0x5ffe77c7u, 0xa1d77ce4u, 0x7826d1dbu, 0x07affd11u, 0xbb7edc6bu, 0x6d16bd27u, 0x85defeccu, 0x2c872002u, \
    0x843abe92u, 0x7361d77fu, 0x273411fbu, 0xa5bb2bd3u, 0x4b3e2399u, 0x9c941f31u, 0xbb9fd3ecu, 0x15df9cddu, 0x4bd8c949u, 0x5dddfd15u, 0xa4445b60u, 0x62cb29a5u, 0x0c7dd2b9u, 0x37bc870au, 0x3171f0fdu, 0x24830a9du, \
    0x41690fe7u, 0xc970692fu, 0x27694b0bu, 0xe2403421u, 0x83c459e8u, 0x32bee66bu, 0x0ab08841u, 0x12aabcedu, 0x40aebfa9u, 0x0d485d23u, 0xab2fcc57u, 0x05193418u, 0x8a4910f5u, 0xd3b0a40bu, 0x35d2925au, 0x2f21ebb5u, \
    0x00fa1bf2u, 0xca8d8005u, 0x68b39769u, 0xf0c5d614u, 0xad0d4418u, 0x0e201271u, 0xbad856e6u, 0x04290f65u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x13e80b9cu, 0x3350c88eu, 0xdb5e56b9u, 0x7dce557cu, 0xb615564au, 0x6001b4b8u, 0x020217e0u, 0x2682e617u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x12edefaau, 0x68c34889u, 0x72aabf4fu, 0x8d087f68u, 0x09081231u, 0x51e1a247u, 0x4729c0fau, 0x2259d6b1u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0xd782e155u, 0x71930c11u, 0xffbe3323u, 0xa6bb947cu, 0xd4741444u, 0xaa303344u, 0x26594943u, 0x2c3b3f0du, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0xc494f1abu, 0x08cfc388u, 0x8d1373d4u, 0x19b31514u, 0xcb6c0213u, 0x584e90fdu, 0xdf2f8849u, 0x09e1685bu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x4e46d97du, 0x36531618u, 0xd4c96d9fu, 0x0af7129eu, 0xca1009b5u, 0x659da72fu, 0x83a20d23u, 0x08116d89u, 0xc39c1939u, 0xb1df4af7u, 0x8a73bf7fu, 0x3d9f0287u, 0x8caf0ae0u, 0x9b222092u, 0xeff054a6u, 0x26684515u, \
    0x16ad6badu, 0xc9af22f7u, 0x4aa662b2u, 0xb311782au, 0xe248c7f4u, 0x19eeaf64u, 0xe3439f82u, 0x20273e77u, 0xf7ce93acu, 0xacc02860u, 0x7ba76b4cu, 0x3933d581u, 0x446c8467u, 0x69e6188bu, 0x4417cc55u, 0x0a46036du, \
    0xaf46471eu, 0x5764af0au, 0x873e0fc1u, 0xdc50792eu, 0x881d04f6u, 0x86a673ffu, 0x3c30a74cu, 0x0b2eddb4u, 0x787e8580u, 0x9a490f32u, 0xf04af8b1u, 0x8fd16d7fu, 0xc6027bf2u, 0x4b39888eu, 0x5b52a15du, 0x03dd2e70u, \
    0x7b6762dfu, 0x448a93a5u, 0x28fdeadfu, 0xbfd62df5u, 0x0e9bd47au, 0xd858f5d0u, 0x3476ec58u, 0x06b03d4du, 0xbcc936d1u, 0x2b19daf4u, 0x56f4299fu, 0xa1a54e7au, 0x5adeaef1u, 0xb533eee0u, 0x84dda0b2u, 0x170c812bu, \
    0x75cf559fu, 0xe0bc4b22u, 0xc154e60fu, 0xc238b945u, 0x929a7d5eu, 0x803982a5u, 0xf7e4a37eu, 0x15ce052du, 0xbf3799a7u, 0x2d28efbdu, 0x1ad60773u, 0x9b097e3cu, 0xaf4a535bu, 0x982d4113u, 0xe3056063u, 0x24e18991u)
#define SB_PAIR_BNFQ_TWIST_B SB_L(0x77b802a8u, 0x3bf938e3u, 0x3633535du, 0x020b1b27u, 0x49755260u, 0x26b7edf0u, 0x4384a86du, 0x2514c632u, 0xd1dcff67u, 0x38e7ecccu, 0x93ce0d3eu, 0x65f0b37du, 0x22ac00aau, 0xd749d0ddu, 0x4a688d4du, 0x0141b9ceu)
#define SB_PAIR_BNFQ_TWO_INV SB_L(0x4f060572u, 0x87bee7d2u, 0x2f1c6ae5u, 0xd0fd2addu, 0xfcfd4f44u, 0x8f5f7492u, 0x3d9cbfacu, 0x1f37631au)
#define SB_PAIR_BLSFQ_FROB SB_L(0xb319d465u, 0x07089552u, 0xb50a8313u, 0xc6695f92u, 0xd117228fu, 0x97e83cccu, 0xb2dc29eeu, 0xa35baecau, 0x5daace4du, 0x1ce393eau, 0xb0fb66ebu, 0x08f2220fu, 0x4ce5d646u, 0xb2f66aadu, 0xfc497cecu, 0x5842a06bu, 0x2599d394u, 0xcf4895d4u, 0x40a8e8d0u, 0xc11b9cbau, 0xe5a0de89u, 0x2e3813cbu, 0x88847fafu, 0x110eefdau, \
    0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x8671f071u, 0xcd03c9e4u, 0x1fcda5d2u, 0x5dab2246u, 0xd3851b95u, 0x587042afu, 0x01bacb9eu, 0x8eb60ebeu, 0x83d050d2u, 0x03f97d6eu, 0x54638741u, 0x18f02065u, \
    0x5aa30fdau, 0x7bcfa7a2u, 0x2a927e7cu, 0xdc17dec1u, 0x6b4ebef1u, 0x2f088dd8u, 0xda74d4a7u, 0xd1ca2087u, 0x96cebc1du, 0x2da25966u, 0xbbfd87d2u, 0x0e2b7eedu, 0x5aa30fdau, 0x7bcfa7a2u, 0x2a927e7cu, 0xdc17dec1u, 0x6b4ebef1u, 0x2f088dd8u, 0xda74d4a7u, 0xd1ca2087u, 0x96cebc1du, 0x2da25966u, 0xbbfd87d2u, 0x0e2b7eedu, \
    0x867545c3u, 0x890dc9e4u, 0x3285a5d5u, 0x2af32253u, 0x309b7e2cu, 0x50880866u, 0x7e881024u, 0xa20d1b8cu, 0xe2db9068u, 0x14e4f04fu, 0x1564853au, 0x14e56d3fu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x0dbce43fu, 0x82d83cf5u, 0xdf9d018fu, 0xa2813e53u, 0x3c65e181u, 0xc6f0caa5u, 0x8d50fe95u, 0x7525cf52u, 0xf4798a6bu, 0x4a85ed50u, 0x6cf8eebdu, 0x171da0fdu, 0xf242c66cu, 0x3726c30au, 0xd1b6fe70u, 0x7c2ac1aau, 0xba4b14a2u, 0xa04007fbu, 0x66341429u, 0xef517c32u, 0x4ed2226bu, 0x0095ba65u, 0xcc86f7ddu, 0x02e370ecu, \
    0x798dba3au, 0xecfb361bu, 0x91865a2cu, 0xc100ddb8u, 0x232bda8eu, 0x0ec08ff1u, 0xf1ca4721u, 0xd5c13cc6u, 0xbf7b5c04u, 0x47222a47u, 0xe51c5f59u, 0x0110f184u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x798a64e8u, 0x30f1361bu, 0x7ece5a2au, 0xf3b8ddabu, 0xc61577f7u, 0x16a8ca3au, 0x74fd029bu, 0xc26a2ff8u, 0x60701c6eu, 0x3636b766u, 0x241b6160u, 0x051ba4abu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0xfffcaaaeu, 0x43f5ffffu, 0xed47fffdu, 0x32b7fff2u, 0xa2e99d69u, 0x07e83a49u, 0x8332bb7au, 0xeca8f331u, 0xa0f4c069u, 0xef148d1eu, 0x3eff0206u, 0x040ab326u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x8671f071u, 0xcd03c9e4u, 0x1fcda5d2u, 0x5dab2246u, 0xd3851b95u, 0x587042afu, 0x01bacb9eu, 0x8eb60ebeu, 0x83d050d2u, 0x03f97d6eu, 0x54638741u, 0x18f02065u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x867545c3u, 0x890dc9e4u, 0x3285a5d5u, 0x2af32253u, 0x309b7e2cu, 0x50880866u, 0x7e881024u, 0xa20d1b8cu, 0xe2db9068u, 0x14e4f04fu, 0x1564853au, 0x14e56d3fu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0xa55c9ad1u, 0x3e2f585du, 0x86c18183u, 0x4294213du, 0x8b623732u, 0x382844c8u, 0x19103e18u, 0x92ad2afdu, 0xac7cf0b9u, 0x1d794e4fu, 0x7d825ec8u, 0x0bd592fcu, 0x5aa30fdau, 0x7bcfa7a2u, 0x2a927e7cu, 0xdc17dec1u, 0x6b4ebef1u, 0x2f088dd8u, 0xda74d4a7u, 0xd1ca2087u, 0x96cebc1du, 0x2da25966u, 0xbbfd87d2u, 0x0e2b7eedu, \
    0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu, 0x53c758bau, 0x5f489857u, 0x70525745u, 0x77ce5853u, 0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u, \
    0xa55c9ad1u, 0x3e2f585du, 0x86c18183u, 0x4294213du, 0x8b623732u, 0x382844c8u, 0x19103e18u, 0x92ad2afdu, 0xac7cf0b9u, 0x1d794e4fu, 0x7d825ec8u, 0x0bd592fcu, 0xa55c9ad1u, 0x3e2f585du, 0x86c18183u, 0x4294213du, 0x8b623732u, 0x382844c8u, 0x19103e18u, 0x92ad2afdu, 0xac7cf0b9u, 0x1d794e4fu, 0x7d825ec8u, 0x0bd592fcu, \
    0xfffcaaaeu, 0x43f5ffffu, 0xed47fffdu, 0x32b7fff2u, 0xa2e99d69u, 0x07e83a49u, 0x8332bb7au, 0xeca8f331u, 0xa0f4c069u, 0xef148d1eu, 0x3eff0206u, 0x040ab326u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, \
    0x5aa30fdau, 0x7bcfa7a2u, 0x2a927e7cu, 0xdc17dec1u, 0x6b4ebef1u, 0x2f088dd8u, 0xda74d4a7u, 0xd1ca2087u, 0x96cebc1du, 0x2da25966u, 0xbbfd87d2u, 0x0e2b7eedu, 0xa55c9ad1u, 0x3e2f585du, 0x86c18183u, 0x4294213du, 0x8b623732u, 0x382844c8u, 0x19103e18u, 0x92ad2afdu, 0xac7cf0b9u, 0x1d794e4fu, 0x7d825ec8u, 0x0bd592fcu)
#define SB_PAIR_BLSFQ_TWIST_B SB_L(0x000cfff3u, 0xaa270000u, 0xfc34000au, 0x53cc0032u, 0x6b0a807fu, 0x478fe97au, 0xe6ba24d7u, 0xb1d37ebeu, 0xbf78ab2fu, 0x8ec9733bu, 0x3d83de7eu, 0x09d64551u, 0x000cfff3u, 0xaa270000u, 0xfc34000au, 0x53cc0032u, 0x6b0a807fu, 0x478fe97au, 0xe6ba24d7u, 0xb1d37ebeu, 0xbf78ab2fu, 0x8ec9733bu, 0x3d83de7eu, 0x09d64551u)
#define SB_PAIR_BLSFQ_TWO_INV SB_L(0x00015554u, 0x18040000u, 0x3ab00001u, 0x85500005u, 0x253c276fu, 0x633cb57cu, 0x31ebb502u, 0x6e22d1ecu, 0xf2d14ca2u, 0xd3916126u, 0x1a006596u, 0x17fbb857u)

template <class P> struct PairingCurve;
template <> struct PairingCurve<BnFq> {
    static constexpr bool M_TWIST = false, X_NEG = false;
    static constexpr uint64_t X = 0x44e992b44a6909f1ull;          // the curve parameter x
    static constexpr uint64_t LOOP = 0x9d797039be763ba8ull;       // 6x + 2 = 2^64 + LOOP
    static constexpr int LOOP_BITS = 64;
    SB_CONSTEXPR_HD static constexpr uint32_t frob(int i) { constexpr uint32_t v[15 * 16] = SB_PAIR_BNFQ_FROB; return v[i]; }
    SB_CONSTEXPR_HD static constexpr uint32_t twist_b(int i) { constexpr uint32_t v[16] = SB_PAIR_BNFQ_TWIST_B; return v[i]; }
    SB_CONSTEXPR_HD static constexpr uint32_t two_inv(int i) { constexpr uint32_t v[8] = SB_PAIR_BNFQ_TWO_INV; return v[i]; }
};
template <> struct PairingCurve<BlsFq> {
    static constexpr bool M_TWIST = true, X_NEG = true;
    static constexpr uint64_t X = 0xd201000000010000ull;          // |x|
    static constexpr uint64_t LOOP = 0xd201000000010000ull;       // |x| = 2^63 + (LOOP mod 2^63)
    static constexpr int LOOP_BITS = 63;
    SB_CONSTEXPR_HD static constexpr uint32_t frob(int i) { constexpr uint32_t v[15 * 24] = SB_PAIR_BLSFQ_FROB; return v[i]; }
    SB_CONSTEXPR_HD static constexpr uint32_t twist_b(int i) { constexpr uint32_t v[24] = SB_PAIR_BLSFQ_TWIST_B; return v[i]; }
    SB_CONSTEXPR_HD static constexpr uint32_t two_inv(int i) { constexpr uint32_t v[12] = SB_PAIR_BLSFQ_TWO_INV; return v[i]; }
};

template <class P> struct Fq6 { Fp2<P> c0, c1, c2; };
template <class P> struct Fq12 { Fq6<P> c0, c1; };
template <class P> struct PairLine { Fp2<P> c0, c1, c2; };      // one Miller-loop line, before scaling by the G1 point
template <class P> struct G2Proj { Fp2<P> x, y, z; };

template <class P> struct Pairing {
    typedef Fp<P> F;
    typedef Fp2<P> F2;
    typedef Fq6<P> F6;
    typedef Fq12<P> F12;
    typedef PairLine<P> Line;
    typedef PairingCurve<P> C;
    static constexpr int N = F::N;

    SB_CONSTEXPR_HD static constexpr int popcount(uint64_t v, int bits) { return bits ? (int)(v & 1) + popcount(v >> 1, bits - 1) : 0; }
    // lines per G2 point in the Miller loop
    static constexpr int NLINES = C::LOOP_BITS + popcount(C::LOOP, C::LOOP_BITS) + (C::M_TWIST ? 0 : 2);

    // ---- Fq2 helpers --------------------------------------------------------------------------------------------
    SB_HD static F2 frob_coef(int k, int i) {    // gamma(k, i)
        F2 r; const int o = (5 * (k - 1) + i - 1) * 2 * N;
_Pragma("unroll")
        for (int j = 0; j < N; j++) { r.a.v[j] = C::frob(o + j); r.b.v[j] = C::frob(o + N + j); }
        return r;
    }
    SB_HD static F2 twist_b() { F2 r;
_Pragma("unroll")
        for (int j = 0; j < N; j++) { r.a.v[j] = C::twist_b(j); r.b.v[j] = C::twist_b(N + j); }
        return r; }
    SB_HD static F two_inv() { F r;
_Pragma("unroll")
        for (int j = 0; j < N; j++) r.v[j] = C::two_inv(j);
        return r; }
    SB_HD static F2 conj2(const F2& a) { F2 r; r.a = a.a; r.b = F::neg(a.b); return r; }
    SB_HD static F2 mulf(const F2& a, const F& s) { F2 r; r.a = F::mul(a.a, s); r.b = F::mul(a.b, s); return r; }
    SB_HD static F2 mul_xi(const F2& a) {
        F2 r;
        if constexpr (C::M_TWIST) { r.a = F::sub(a.a, a.b); r.b = F::add(a.a, a.b); }   // (1 + u)
        else {                                                                             // (9 + u)
            F2 t = F2::dbl(F2::dbl(F2::dbl(a))); t = F2::add(t, a);
            r.a = F::sub(t.a, a.b); r.b = F::add(a.a, t.b);
        }
        return r;
    }

    // ---- Fq6 --------------------------------------------------------------------------------------------------------
    SB_HD static F6 add6(const F6& a, const F6& b) { F6 r; r.c0 = F2::add(a.c0, b.c0); r.c1 = F2::add(a.c1, b.c1); r.c2 = F2::add(a.c2, b.c2); return r; }
    SB_HD static F6 sub6(const F6& a, const F6& b) { F6 r; r.c0 = F2::sub(a.c0, b.c0); r.c1 = F2::sub(a.c1, b.c1); r.c2 = F2::sub(a.c2, b.c2); return r; }
    SB_HD static F6 neg6(const F6& a) { F6 r; r.c0 = F2::neg(a.c0); r.c1 = F2::neg(a.c1); r.c2 = F2::neg(a.c2); return r; }
    SB_HD static F6 mul_v(const F6& a) { F6 r; r.c0 = mul_xi(a.c2); r.c1 = a.c0; r.c2 = a.c1; return r; }
    // Karatsuba: 6 Fq2 multiplies
    SB_HD_NOINLINE static F6 mul6(const F6& a, const F6& b) {
        const F2 aa = F2::mul(a.c0, b.c0), bb = F2::mul(a.c1, b.c1), cc = F2::mul(a.c2, b.c2);
        F6 r;
        r.c0 = F2::add(mul_xi(F2::sub(F2::sub(F2::mul(F2::add(a.c1, a.c2), F2::add(b.c1, b.c2)), bb), cc)), aa);
        r.c1 = F2::add(F2::sub(F2::sub(F2::mul(F2::add(a.c0, a.c1), F2::add(b.c0, b.c1)), aa), bb), mul_xi(cc));
        r.c2 = F2::sub(F2::add(F2::sub(F2::mul(F2::add(a.c0, a.c2), F2::add(b.c0, b.c2)), aa), bb), cc);
        return r;
    }
    // a * (b0 + b1 v)
    SB_HD_NOINLINE static F6 mul6_01(const F6& a, const F2& b0, const F2& b1) {
        const F2 aa = F2::mul(a.c0, b0), bb = F2::mul(a.c1, b1);
        F6 r;
        r.c0 = F2::add(mul_xi(F2::sub(F2::mul(F2::add(a.c1, a.c2), b1), bb)), aa);
        r.c1 = F2::sub(F2::sub(F2::mul(F2::add(b0, b1), F2::add(a.c0, a.c1)), aa), bb);
        r.c2 = F2::add(F2::sub(F2::mul(F2::add(a.c0, a.c2), b0), aa), bb);
        return r;
    }
    // a * (b1 v)
    SB_HD static F6 mul6_1(const F6& a, const F2& b1) {
        F6 r;
        r.c0 = mul_xi(F2::mul(a.c2, b1));
        r.c1 = F2::mul(a.c0, b1);
        r.c2 = F2::mul(a.c1, b1);
        return r;
    }
    SB_HD static F6 inv6(const F6& a) {
        const F2 A = F2::sub(F2::sqr(a.c0), mul_xi(F2::mul(a.c1, a.c2)));
        const F2 B = F2::sub(mul_xi(F2::sqr(a.c2)), F2::mul(a.c0, a.c1));
        const F2 Cc = F2::sub(F2::sqr(a.c1), F2::mul(a.c0, a.c2));
        const F2 t = F2::inv(F2::add(F2::mul(a.c0, A), mul_xi(F2::add(F2::mul(a.c2, B), F2::mul(a.c1, Cc)))));
        F6 r; r.c0 = F2::mul(A, t); r.c1 = F2::mul(B, t); r.c2 = F2::mul(Cc, t); return r;
    }

    // ---- Fq12 -------------------------------------------------------------------------------------------------------
    SB_HD static F12 one() { F12 r; r.c0.c0 = F2::one(); r.c0.c1 = F2::zero(); r.c0.c2 = F2::zero(); r.c1.c0 = F2::zero(); r.c1.c1 = F2::zero(); r.c1.c2 = F2::zero(); return r; }
    SB_HD static bool eq(const F12& a, const F12& b) {
        return (a.c0.c0 == b.c0.c0) & (a.c0.c1 == b.c0.c1) & (a.c0.c2 == b.c0.c2) & (a.c1.c0 == b.c1.c0) & (a.c1.c1 == b.c1.c1) & (a.c1.c2 == b.c1.c2);
    }
    SB_HD static F12 conj(const F12& a) { F12 r; r.c0 = a.c0; r.c1 = neg6(a.c1); return r; }
    // Karatsuba over Fq6: 3 Fq6 multiplies
    SB_HD_NOINLINE static F12 mul(const F12& a, const F12& b) {
        const F6 aa = mul6(a.c0, b.c0), bb = mul6(a.c1, b.c1);
        F12 r;
        r.c1 = sub6(sub6(mul6(add6(a.c0, a.c1), add6(b.c0, b.c1)), aa), bb);
        r.c0 = add6(aa, mul_v(bb));
        return r;
    }
    // complex squaring: 2 Fq6 multiplies
    SB_HD_NOINLINE static F12 sqr(const F12& a) {
        const F6 t = mul6(a.c0, a.c1);
        F12 r;
        r.c0 = sub6(sub6(mul6(add6(a.c0, a.c1), add6(a.c0, mul_v(a.c1))), t), mul_v(t));
        r.c1 = add6(t, t);
        return r;
    }
    SB_HD static F12 inv(const F12& a) {   // (a0 - a1 w) / (a0^2 - v a1^2)
        const F6 t = inv6(sub6(mul6(a.c0, a.c0), mul_v(mul6(a.c1, a.c1))));
        F12 r; r.c0 = mul6(a.c0, t); r.c1 = neg6(mul6(a.c1, t)); return r;
    }
    // a^(q^k), k = 1..3: the coefficient of w^i is conjugated k times and multiplied by gamma(k, i)
    SB_HD_NOINLINE static F12 frob(const F12& a, int k) {
        const bool cj = k & 1;
        auto f = [&](const F2& x, int i) -> F2 {
            const F2 y = cj ? conj2(x) : x;
            return i ? F2::mul(y, frob_coef(k, i)) : y;
        };
        F12 r;
        r.c0.c0 = f(a.c0.c0, 0); r.c1.c0 = f(a.c1.c0, 1); r.c0.c1 = f(a.c0.c1, 2);
        r.c1.c1 = f(a.c1.c1, 3); r.c0.c2 = f(a.c0.c2, 4); r.c1.c2 = f(a.c1.c2, 5);
        return r;
    }
    // (x + y s)^2 in Fq4 = Fq2[s]/(s^2 - xi): (x^2 + xi y^2, 2xy)
    SB_HD static void sqr4(const F2& x, const F2& y, F2& r0, F2& r1) {
        const F2 t = F2::mul(x, y);
        r0 = F2::sub(F2::sub(F2::mul(F2::add(x, y), F2::add(x, mul_xi(y))), t), mul_xi(t));
        r1 = F2::dbl(t);
    }
    // Granger-Scott squaring, for elements of the cyclotomic subgroup (after the easy part of the final exponentiation)
    SB_HD_NOINLINE static F12 cyc_sqr(const F12& a) {
        F2 z0 = a.c0.c0, z4 = a.c0.c1, z3 = a.c0.c2, z2 = a.c1.c0, z1 = a.c1.c1, z5 = a.c1.c2;
        F2 t0, t1, t2, t3, t4, t5;
        sqr4(z0, z1, t0, t1); sqr4(z2, z3, t2, t3); sqr4(z4, z5, t4, t5);
        z0 = F2::sub(t0, z0); z0 = F2::add(F2::dbl(z0), t0);
        z1 = F2::add(t1, z1); z1 = F2::add(F2::dbl(z1), t1);
        const F2 x5 = mul_xi(t5);
        z2 = F2::add(x5, z2); z2 = F2::add(F2::dbl(z2), x5);
        z3 = F2::sub(t4, z3); z3 = F2::add(F2::dbl(z3), t4);
        z4 = F2::sub(t2, z4); z4 = F2::add(F2::dbl(z4), t2);
        z5 = F2::add(t3, z5); z5 = F2::add(F2::dbl(z5), t3);
        F12 r; r.c0.c0 = z0; r.c0.c1 = z4; r.c0.c2 = z3; r.c1.c0 = z2; r.c1.c1 = z1; r.c1.c2 = z5;
        return r;
    }
    // f * (c0 + c3 w + c4 w^3)  (D-type lines)
    SB_HD_NOINLINE static F12 mul_034(const F12& f, const F2& c0, const F2& c3, const F2& c4) {
        F6 a; a.c0 = F2::mul(f.c0.c0, c0); a.c1 = F2::mul(f.c0.c1, c0); a.c2 = F2::mul(f.c0.c2, c0);
        const F6 b = mul6_01(f.c1, c3, c4);
        const F6 e = mul6_01(add6(f.c0, f.c1), F2::add(c0, c3), c4);
        F12 r; r.c1 = sub6(e, add6(a, b)); r.c0 = add6(a, mul_v(b));
        return r;
    }
    // f * (c0 + c1 w^2 + c4 w^3)  (M-type lines)
    SB_HD_NOINLINE static F12 mul_014(const F12& f, const F2& c0, const F2& c1, const F2& c4) {
        const F6 aa = mul6_01(f.c0, c0, c1), bb = mul6_1(f.c1, c4);
        const F6 e = mul6_01(add6(f.c0, f.c1), c0, F2::add(c1, c4));
        F12 r; r.c1 = sub6(sub6(e, aa), bb); r.c0 = add6(aa, mul_v(bb));
        return r;
    }

    // ---- Miller loop ------------------------------------------------------------------------------------------------
    // R = 2R (homogeneous projective, a = 0)
    SB_HD_NOINLINE static Line dbl_step(G2Proj<P>& R) {
        const F h2 = two_inv();
        const F2 a = mulf(F2::mul(R.x, R.y), h2);
        const F2 b = F2::sqr(R.y), c = F2::sqr(R.z);
        const F2 e = F2::mul(twist_b(), F2::add(F2::dbl(c), c));
        const F2 f = F2::add(F2::dbl(e), e);
        const F2 g = mulf(F2::add(b, f), h2);
        const F2 h = F2::sub(F2::sqr(F2::add(R.y, R.z)), F2::add(b, c));
        const F2 i = F2::sub(e, b);
        const F2 j = F2::sqr(R.x);
        const F2 e2 = F2::sqr(e);
        R.x = F2::mul(a, F2::sub(b, f));
        R.y = F2::sub(F2::sqr(g), F2::add(F2::dbl(e2), e2));
        R.z = F2::mul(b, h);
        Line l;
        if constexpr (C::M_TWIST) { l.c0 = i; l.c1 = F2::add(F2::dbl(j), j); l.c2 = F2::neg(h); }
        else { l.c0 = F2::neg(h); l.c1 = F2::add(F2::dbl(j), j); l.c2 = i; }
        return l;
    }
    // R = R + (qx, qy)
    SB_HD_NOINLINE static Line add_step(G2Proj<P>& R, const F2& qx, const F2& qy) {
        const F2 theta = F2::sub(R.y, F2::mul(qy, R.z));
        const F2 lambda = F2::sub(R.x, F2::mul(qx, R.z));
        const F2 c = F2::sqr(theta), d = F2::sqr(lambda);
        const F2 e = F2::mul(lambda, d), f = F2::mul(R.z, c), g = F2::mul(R.x, d);
        const F2 h = F2::sub(F2::add(e, f), F2::dbl(g));
        R.x = F2::mul(lambda, h);
        R.y = F2::sub(F2::mul(theta, F2::sub(g, h)), F2::mul(e, R.y));
        R.z = F2::mul(R.z, e);
        const F2 j = F2::sub(F2::mul(theta, qx), F2::mul(lambda, qy));
        Line l;
        if constexpr (C::M_TWIST) { l.c0 = j; l.c1 = F2::neg(theta); l.c2 = lambda; }
        else { l.c0 = lambda; l.c1 = F2::neg(theta); l.c2 = j; }
        return l;
    }
    // f * line(P)
    SB_HD static F12 ell(const F12& f, const Line& l, const F& px, const F& py) {
        if constexpr (C::M_TWIST) return mul_014(f, l.c0, mulf(l.c1, px), mulf(l.c2, py));
        else return mul_034(f, mulf(l.c0, py), mulf(l.c1, px), l.c2);
    }
    // pi^k(Q) on the twist, k = 1, 2 (BN254's last two additions)
    SB_HD static void frob_twist(const F2& x, const F2& y, int k, F2& ox, F2& oy) {
        ox = F2::mul(k & 1 ? conj2(x) : x, frob_coef(k, 2));
        oy = F2::mul(k & 1 ? conj2(y) : y, frob_coef(k, 3));
    }

    // The lines of one G2 point (not infinity), in the order miller() consumes them: NLINES entries.
    SB_HD static void prepare(const F2& qx, const F2& qy, Line* out) {
        G2Proj<P> R; R.x = qx; R.y = qy; R.z = F2::one();
        int li = 0;
#pragma unroll 1
        for (int i = C::LOOP_BITS - 1; i >= 0; i--) {
            out[li++] = dbl_step(R);
            if ((C::LOOP >> i) & 1) out[li++] = add_step(R, qx, qy);
        }
        if constexpr (!C::M_TWIST) {
            F2 x1, y1, x2, y2;
            frob_twist(qx, qy, 1, x1, y1); frob_twist(qx, qy, 2, x2, y2);
            out[li++] = add_step(R, x1, y1);
            out[li++] = add_step(R, x2, F2::neg(y2));
        }
    }

    // Multi-Miller loop sharing the squarings of f: pair 0 is (p0, q) with q's lines computed on the fly, pairs 1 and 2 are
    // (p1, lines t1) and (p2, lines t2) with precomputed lines.  live* = false drops a pair (a point at infinity).
    SB_HD static F12 miller(const F& p0x, const F& p0y, const F2& qx, const F2& qy, bool live0,
                            const F& p1x, const F& p1y, const Line* t1, bool live1,
                            const F& p2x, const F& p2y, const Line* t2, bool live2) {
        F12 f = one();
        G2Proj<P> R; R.x = qx; R.y = qy; R.z = F2::one();
        int li = 0;
        auto step = [&](bool add, const F2& ax, const F2& ay) {
            if (live0) f = ell(f, add ? add_step(R, ax, ay) : dbl_step(R), p0x, p0y);
            if (live1) f = ell(f, t1[li], p1x, p1y);
            if (live2) f = ell(f, t2[li], p2x, p2y);
            li++;
        };
#pragma unroll 1
        for (int i = C::LOOP_BITS - 1; i >= 0; i--) {
            if (i != C::LOOP_BITS - 1) f = sqr(f);
            step(false, qx, qy);
            if ((C::LOOP >> i) & 1) step(true, qx, qy);
        }
        if constexpr (!C::M_TWIST) {
            F2 x1, y1, x2, y2;
            frob_twist(qx, qy, 1, x1, y1); frob_twist(qx, qy, 2, x2, y2);
            step(true, x1, y1);
            step(true, x2, F2::neg(y2));
        }
        if constexpr (C::X_NEG) f = conj(f);
        return f;
    }

    // ---- final exponentiation ---------------------------------------------------------------------------------------
    SB_CONSTEXPR_HD static constexpr int topbit(uint64_t v) { return v >> 1 ? 1 + topbit(v >> 1) : 0; }
    // a^|x| for a in the cyclotomic subgroup
    SB_HD static F12 pow_x(const F12& a) {
        F12 r = a;
#pragma unroll 1
        for (int i = topbit(C::X) - 1; i >= 0; i--) {
            r = cyc_sqr(r);
            if ((C::X >> i) & 1) r = mul(r, a);
        }
        return r;
    }
    SB_HD static F12 final_exp(const F12& f) {
        F12 r = mul(conj(f), inv(f));          // f^(q^6 - 1)
        r = mul(frob(r, 2), r);                // ^(q^2 + 1)
        if constexpr (!C::M_TWIST) {
            // BN254: r^(2x(6x^2 + 3x + 1)(q^4 - q^2 + 1)/r); conj(pow_x) = a^-x in the cyclotomic subgroup
            const F12 y0 = conj(pow_x(r));
            const F12 y1 = cyc_sqr(y0);
            const F12 y2 = cyc_sqr(y1);
            F12 y3 = mul(y2, y1);
            const F12 y4 = conj(pow_x(y3));
            const F12 y5 = cyc_sqr(y4);
            F12 y6 = conj(pow_x(y5));
            y3 = conj(y3); y6 = conj(y6);
            const F12 y7 = mul(y6, y4);
            F12 y8 = mul(y7, y3);
            const F12 y9 = mul(y8, y1);
            const F12 y10 = mul(y8, y4);
            const F12 y11 = mul(y10, r);
            const F12 y13 = mul(frob(y9, 1), y11);
            y8 = frob(y8, 2);
            const F12 y14 = mul(y8, y13);
            const F12 y15 = frob(mul(conj(r), y9), 3);
            return mul(y15, y14);
        } else {
            // BLS12-381: r^(3(q^4 - q^2 + 1)/r); exp_x(a) = a^x = conj(a^|x|)
            auto exp_x = [](const F12& a) { return conj(pow_x(a)); };
            const F12 y0 = cyc_sqr(r);
            F12 y1 = exp_x(r);
            F12 y2 = conj(r);
            y1 = mul(y1, y2);
            y2 = exp_x(y1);
            y1 = conj(y1);
            y1 = mul(y1, y2);
            y2 = exp_x(y1);
            y1 = frob(y1, 1);
            y1 = mul(y1, y2);
            r = mul(r, y0);
            const F12 z0 = exp_x(y1);
            y2 = exp_x(z0);
            const F12 z1 = frob(y1, 2);
            y1 = conj(y1);
            y1 = mul(y1, y2);
            y1 = mul(y1, z1);
            return mul(r, y1);
        }
    }

    // ---- points -----------------------------------------------------------------------------------------------------
    // a coordinate as stored: Montgomery, below q
    SB_HD static bool canonical(const F& a) {
        bool lt = false, decided = false;
_Pragma("unroll")
        for (int i = N - 1; i >= 0; i--) {
            const uint32_t p = P::p(i);
            lt = (!decided && a.v[i] != p) ? a.v[i] < p : lt;
            decided = decided || a.v[i] != p;
        }
        return lt;
    }
    // G1.isValid / G2.isValid: on the curve, or the point at infinity (all zero)
    SB_HD static bool g1_valid(const F& x, const F& y) {
        if (!canonical(x) || !canonical(y)) return false;
        if (x.is_zero() && y.is_zero()) return true;
        const F one = F::one();
        F b = F::add(F::add(one, one), one);
        if constexpr (C::M_TWIST) b = F::add(b, one);
        return F::sqr(y) == F::add(F::mul(F::sqr(x), x), b);
    }
    SB_HD static bool g2_valid(const F2& x, const F2& y) {
        if (!canonical(x.a) || !canonical(x.b) || !canonical(y.a) || !canonical(y.b)) return false;
        if (x.is_zero() && y.is_zero()) return true;
        return F2::sqr(y) == F2::add(F2::mul(F2::sqr(x), x), twist_b());
    }
};

// ---- the test hook's records (sb_pairing_eval) --------------------------------------------------------------------------
// Fq elements per input / output record of op; false for an op that is not defined.  The ops: 0 a*b, 1 a^2, 2 cyclotomic
// a^2, 3 a^-1, 4 (a^q, a^(q^2), a^(q^3)), 5 Miller loop of (P, Q), 6 final exponentiation, 7 e(P, Q) = 6 of 5.  Tower
// elements are 12 Fq coefficients; P = x, y and Q = x.c0, x.c1, y.c0, y.c1 (affine, all zero = infinity).
inline bool pair_eval_shape(int op, int* in_elems, int* out_elems) {
    static const int I[8] = {24, 12, 12, 12, 12, 6, 12, 6}, O[8] = {12, 12, 12, 12, 36, 12, 12, 12};
    if (op < 0 || op > 7) return false;
    *in_elems = I[op]; *out_elems = O[op];
    return true;
}
template <class P> SB_HD void pair_eval_record(int op, const Fp<P>* in, Fp<P>* out) {
    typedef Pairing<P> T;
    typedef typename T::F12 F12;
    typedef typename T::F2 F2;
    auto get12 = [&](int o) { F12 a; Fp<P>* d = (Fp<P>*)&a;
        for (int i = 0; i < 12; i++) d[i] = in[o + i];
        return a; };
    auto put12 = [&](int o, const F12& a) { const Fp<P>* s = (const Fp<P>*)&a;
        for (int i = 0; i < 12; i++) out[o + i] = s[i]; };
    if (op == 0) put12(0, T::mul(get12(0), get12(12)));
    else if (op == 1) put12(0, T::sqr(get12(0)));
    else if (op == 2) put12(0, T::cyc_sqr(get12(0)));
    else if (op == 3) put12(0, T::inv(get12(0)));
    else if (op == 4) { const F12 a = get12(0); put12(0, T::frob(a, 1)); put12(12, T::frob(a, 2)); put12(24, T::frob(a, 3)); }
    else if (op == 6) put12(0, T::final_exp(get12(0)));
    else if (op == 5 || op == 7) {
        F2 qx, qy; qx.a = in[2]; qx.b = in[3]; qy.a = in[4]; qy.b = in[5];
        const bool live = !(in[0].is_zero() && in[1].is_zero()) && !(qx.is_zero() && qy.is_zero());
        F12 f = T::miller(in[0], in[1], qx, qy, live, in[0], in[1], nullptr, false, in[0], in[1], nullptr, false);
        put12(0, op == 7 ? T::final_exp(f) : f);
    }
}

}  // namespace sb
