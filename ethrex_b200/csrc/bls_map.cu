// bls_map.cu -- EIP-2537 map-to-curve on the device, `count` items per call: the Prague precompiles 0x10 MAP_FP_TO_G1 and
// 0x11 MAP_FP2_TO_G2 behind the reference's Crypto::bls12_381_fp_to_g1 / _fp2_to_g2
// (/root/reference/crates/common/crypto/provider.rs:674-700; levm precompiles.rs:1403-1479).
//
// The output for a field element u is clear_cofactor(iso_map(map_to_curve_simple_swu(u))), RFC 9380 sections 6.6.2,
// 6.6.3 and 7 with the BLS12-381 parameters of its 8.8.1 (G1) and 8.8.2 (G2).  One template over the coordinate field,
// Fp381 (G1) or Fp2_381 (G2), one thread per item: each item is a long serial chain that shares nothing with its neighbours.
//   SSWU:     on E': y^2 = x^3 + A' x + B' in the straight-line form of 6.6.2, one inversion (inv0) and one or two square-root
//             candidates, each checked by squaring (g(x1) non-square implies g(Z u^2 x1) = Z^3 u^6 g(x1) square); y takes
//             the sign of u under sgn0.
//   iso_map:  Horner in Montgomery form over the four polynomials of RFC Appendix E.2 (G1, 11-isogeny) or E.3 (G2, 3-isogeny),
//             numerators and denominators kept apart and folded into one XYZZ point with ZZ = t^2, ZZZ = t^3, t = x_den y_den:
//             no inversion.  A vanishing denominator gives the identity.
//   cofactor: G1 multiplies by h_eff = 1 - z = 0xd201000000010001 (64-bit chain); G2 uses the psi form of RFC Appendix G.3,
//             [z^2 - z - 1] P + [z - 1] psi(P) + psi^2(2 P): two 64-bit chains in |z| instead of the 636-bit h_eff.
//   One inversion normalises the result.  The curve law is curve.cuh's XYZZ over E and E2 (a = 0); nothing runs on E'.
// The zero Fp2 input needs no special case: plain RFC arithmetic gives levm's FP2_ZERO_MAPPED_TO_G2.
#include "bls12.cuh"

namespace b200zk {
namespace {

typedef Fp2_381 F2;

// ---- constants: canonical little-endian 32-bit limbs, converted with to_mont at use.  Printed and checked by
// tests/golden/make_bls12_map_constants.py (G1: point count of E', iso_map onto E and additive, Z by find_z_sswu; G2:
// re-derived by Velu from E2''s 3-division polynomial and pinned by levm's FP2_ZERO_MAPPED_TO_G2);
// tests/test_bls12_map_host.py checks that these tables equal its output.
enum { kA = 0, kB = 1, kZ = 2, kNegBA = 3, kBZA = 4, kPsiX = 5, kPsiY = 6 };  // A', B', Z, -B'/A', B'/(Z A'), psi's c_x, c_y (G2)

// G1, RFC 9380 8.8.1: A', B', Z = 11, -B'/A', B'/(Z A')
__constant__ uint32_t kG1Consts[5][12] = {
    {0x2d584c1du, 0x5cf42808u, 0xa0e0f97fu, 0x98936f8du, 0xefd881acu, 0xd8e8981au, 0x83ee66a8u, 0xb0ea9853u, 0xc96d4982u, 0x3d693a02u, 0xa3b8e943u, 0x00144698u},
    {0x8e172be0u, 0xd1cc48e9u, 0x316ceaa5u, 0x5a23215au, 0xcef35ef5u, 0xa0b9c14fu, 0xf24f4070u, 0x2016c1f0u, 0x753eee3bu, 0x018b12e8u, 0x11688030u, 0x12e2908du},
    {0x0000000bu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u},
    {0x5e4c9c7cu, 0x29d67067u, 0x5a84188eu, 0x51bdfcf9u, 0xaa278ba7u, 0x1df39753u, 0x5bdbfac2u, 0xa928ad9fu, 0x460c78f6u, 0x66ef2470u, 0xd85631d9u, 0x0793154fu},
    {0xf76d2814u, 0xf7d4816au, 0xbe8e2c4fu, 0xf79a5d5cu, 0xd27d1aadu, 0x310d5ce1u, 0x62efb105u, 0x683bca0cu, 0x591ea140u, 0xe772bc7au, 0x1626a32du, 0x123939a3u},
};

// G1 11-isogeny, RFC 9380 Appendix E.2: x_num k_(1,0..11), x_den k_(2,0..9), y_num k_(3,0..15), y_den k_(4,0..14); both
// denominators monic, their leading 1 not listed
__constant__ uint32_t kG1Iso[53][12] = {
    {0x734649b7u, 0xaeac1662u, 0xf2e62d6eu, 0x5610c2d5u, 0xcdb4e2c8u, 0xf2627b56u, 0xa2d7005fu, 0x6b303e88u, 0xd9981585u, 0xb809101du, 0x1e833340u, 0x11a05f2bu},
    {0xb3cb83bbu, 0xe834eef1u, 0xf318c356u, 0x4838f2a6u, 0x70d1e86bu, 0xf565e33cu, 0x2f6a8417u, 0x7c17e75bu, 0x2147a81cu, 0x0588bab2u, 0xe943ab2fu, 0x17294ed3u},
    {0xac9edcb0u, 0xe0179f9du, 0x2a09729fu, 0x958c3e3du, 0xec68e25cu, 0x6878e501u, 0x295983e5u, 0xce032473u, 0xd10a9a1bu, 0x1d1048c5u, 0xb97678ecu, 0x0d54005du},
    {0x1d9b6861u, 0xc5b38864u, 0xe3107193u, 0x5336e25cu, 0xf1b33083u, 0xf1b33289u, 0x6a8dbf25u, 0xd7f5e465u, 0x07e55412u, 0x4e0609d3u, 0x6fcc6db7u, 0x1778e716u},
    {0xac8895d9u, 0x51154ce9u, 0x301e77c4u, 0x985a286fu, 0x982fac18u, 0x086eeb65u, 0x1257fb3fu, 0x99db995au, 0xe4118e54u, 0x6642b4b3u, 0x3199f443u, 0x0e99726au},
    {0x6f652983u, 0xcd13c1c6u, 0xcae73d19u, 0xa0870d2du, 0x97e68f90u, 0x9ed3ab90u, 0xd952799bu, 0xdb3cb17du, 0xf7a74ab5u, 0x01d1201bu, 0x0d7313ffu, 0x1630c325u},
    {0xa139ed84u, 0xddd7f225u, 0xc1052ecau, 0x8da25128u, 0xf9c86b2au, 0x9008e218u, 0x4f0f8ce1u, 0xb1158626u, 0x8ae652bfu, 0x6a3726c3u, 0x3fe44d29u, 0x0d6ed655u},
    {0xe3f0c88eu, 0x9ccb5618u, 0xc8f475afu, 0x39b7c8f8u, 0xf0f27533u, 0xa682c62eu, 0x275b4db1u, 0x356de5abu, 0xd1117e53u, 0xe8743884u, 0x01abdbe2u, 0x17b81e77u},
    {0x8497e317u, 0x6d71986au, 0x96b74e95u, 0x4fa295f2u, 0x28c5d1deu, 0xa2c596c9u, 0xe79f5574u, 0xc43b756cu, 0x63be990du, 0x7b90b335u, 0xf9a78fc4u, 0x080d3cf1u},
    {0xbe390c9eu, 0x7f241067u, 0xdc032779u, 0xa3190b2eu, 0xf4bb1b7fu, 0x676314bau, 0x3a0c5c99u, 0xdd2ecb80u, 0x5d138f22u, 0x2e0c3751u, 0x1bcfa7c4u, 0x169b1f8eu},
    {0x1605fb7bu, 0xca67df3fu, 0x8c285decu, 0xf69b771fu, 0x03b14866u, 0xd50af360u, 0xe6787f96u, 0xfa7dccddu, 0xd2565b0du, 0x72d8ec09u, 0x79ce07e2u, 0x10321da0u},
    {0x8ba2d229u, 0xa9c8ba2eu, 0xb64d391fu, 0xc24b1b80u, 0xc24c6b68u, 0x23c0bf1bu, 0x22c837bcu, 0x31d79d7eu, 0x81edee3du, 0xbd1e9623u, 0x8e260e70u, 0x06e08c24u},
    {0x40d21b1cu, 0x993cf9fau, 0xbe343df8u, 0xb558d681u, 0x7fc8ac62u, 0x9c958861u, 0xa35b48bau, 0x01d5ef4bu, 0x4bd3fa6fu, 0x18b2e62fu, 0x8cff19aeu, 0x08ca8d54u},
    {0xc82b3bffu, 0xe5c8276eu, 0x6cb026e9u, 0x13daa884u, 0x8c48bf57u, 0x0126c258u, 0x0cf0800cu, 0x7041e8cau, 0x98e53636u, 0x48b47112u, 0xeb559c43u, 0x12561a5du},
    {0x5cb83e19u, 0xfcc239bau, 0x7c94fedcu, 0xd6a3d096u, 0xb11aceacu, 0xfca64e00u, 0x5a718cd1u, 0x6f89416fu, 0xbff2991fu, 0x8137e629u, 0x57a3225eu, 0x0b2962feu},
    {0x8dc62cd8u, 0x130de893u, 0x3eecf5c4u, 0x4976d524u, 0xc28d6fd0u, 0x54cca8abu, 0x16b16551u, 0x5b08243fu, 0x7c40eb54u, 0xc83aafefu, 0xa58ae2feu, 0x03425581u},
    {0x3532a21eu, 0x539d395bu, 0x1f35781du, 0x9bd29ba8u, 0x33b306dau, 0x8d6b44e8u, 0xa12062bbu, 0xffdfc759u, 0x43e7a07du, 0x0a6f1d5fu, 0x022914a8u, 0x13a8e162u},
    {0x9f6304a5u, 0xc02df9a2u, 0xc4228f11u, 0x7400d24bu, 0x24b8982fu, 0x0a43bcefu, 0xce9cad4du, 0x395735e9u, 0x0506c6e9u, 0x55390f7fu, 0xe4e667b9u, 0x0e7355f8u},
    {0x6ee84a3au, 0xec257449u, 0x8f0de06cu, 0xea73b353u, 0x62aede9cu, 0x4e2e0730u, 0xaf53a189u, 0x570f5799u, 0xe0596721u, 0x0f3e0c63u, 0xf1693619u, 0x0772caacu},
    {0xbdcc5a5eu, 0x11f7d99bu, 0x9d11e2d3u, 0x0fa5b948u, 0xf9822c58u, 0x1996e1cdu, 0x1bca68a8u, 0x6e7f63c2u, 0x74cf0199u, 0x30b3f5b0u, 0x9d64a8b2u, 0x14a7ac2au},
    {0x79a1d641u, 0x4776ec3au, 0xabba4370u, 0x03826692u, 0x7f398835u, 0x74100da6u, 0x7161366bu, 0xe07f8d1du, 0xafc7a3ccu, 0x5e920b3du, 0xada54f82u, 0x0a10ecf6u},
    {0x68ecdd0au, 0x2d6384d1u, 0x4b786500u, 0x93174e4bu, 0x78f31c15u, 0x76df5339u, 0x96f7d037u, 0xf682b4eeu, 0xb3a56680u, 0x476d6e3eu, 0xb9e92ad4u, 0x095fc13au},
    {0x9707bb33u, 0xbe984571u, 0x9b3ba3c2u, 0xcd0c7aeeu, 0x956543d3u, 0x2b52af6cu, 0x48a86952u, 0x11ad138eu, 0x4980dcfau, 0x259d1f09u, 0x1ba24ee0u, 0x090d97c8u},
    {0x2e41c696u, 0xe097e75au, 0x962fa8bfu, 0xd6c56711u, 0xeb67ad34u, 0x0f906343u, 0x254f383du, 0x1223e96cu, 0x76fb4683u, 0xd51036d7u, 0x04ee5811u, 0x134996a1u},
    {0xc72de1f6u, 0xb8dfe240u, 0x28b00523u, 0xd26d5216u, 0x91400da7u, 0xc344be4bu, 0x58a31ce2u, 0x2552e2d6u, 0x6a3b4994u, 0xf4a384c8u, 0xaa966e66u, 0x00cc786bu},
    {0xb0e5f4cbu, 0xa6355c77u, 0x9ec61decu, 0xde405abau, 0x03251cf9u, 0x09e4a3ecu, 0x0eeb791cu, 0xd42aa7b9u, 0xd8746757u, 0x7898751au, 0xe8981c21u, 0x01f86376u},
    {0xf2e8fedbu, 0x41b6daecu, 0x099040a8u, 0x2ee7f8dcu, 0x21351adcu, 0x79833fd2u, 0xe3ce50b8u, 0x195536fbu, 0xa21529c4u, 0x5caf4fe2u, 0xefe0ff13u, 0x08cc03fdu},
    {0x3633a5f0u, 0x99b23ab1u, 0xc95a8072u, 0x203f6326u, 0x3ad5544eu, 0x76505c3du, 0xafadb7bdu, 0x74a7d0d4u, 0xb8f0a6a0u, 0x2211e11du, 0x40634b6au, 0x16603fcau},
    {0x5fe9d6f2u, 0xc961f885u, 0x460f415eu, 0x47a87ac2u, 0x4d634f37u, 0x5231413cu, 0x2be184cbu, 0xe75bb8cau, 0x27796b3cu, 0xb2c977d0u, 0xcfac1bbcu, 0x04ab0b9bu},
    {0x1870fb29u, 0xa15e4ca3u, 0xfedfe935u, 0x42f64550u, 0xc26c8426u, 0xfd038da6u, 0xe3bdd81fu, 0x170a05bfu, 0x2ca6c674u, 0xde9926bdu, 0x333ab86fu, 0x0987c8d5u},
    {0x7bdba587u, 0x60370e57u, 0xc78607a3u, 0x69d65201u, 0x1f20cabeu, 0x1e8b6e6au, 0x679dc26cu, 0x8f3abd16u, 0x1e4da1bbu, 0xe88c9e22u, 0xbd96684bu, 0x09fc4018u},
    {0xca731c30u, 0x2bafaaebu, 0xdd4eba6fu, 0x9b3f7055u, 0xd1e4d43bu, 0x06985e7eu, 0x915af6feu, 0xc42a0ca7u, 0xada14a23u, 0x223abde7u, 0x1186bdb5u, 0x0e1bba7au},
    {0xd011c132u, 0xe813711au, 0xce3fbafcu, 0x31bf3a5cu, 0x6389e610u, 0xd1183e41u, 0x6caf493fu, 0xcd2fcbcbu, 0x1d43fb93u, 0x0dfd0b8fu, 0x937cd1beu, 0x19713e47u},
    {0xd0074d8eu, 0xce07c8a4u, 0x1b44d606u, 0x49d9cdf4u, 0x911f6432u, 0x2e6bfe7fu, 0xaaf0c246u, 0x523559b8u, 0xfed2edccu, 0xb918c143u, 0x8f36f6deu, 0x18b46a90u},
    {0x0b971ef8u, 0x0d4c04f0u, 0x919211f2u, 0x06c851c1u, 0x07b4633fu, 0xc02710e8u, 0x3426b08eu, 0x7aa7b12au, 0x04f53f44u, 0xd1550960u, 0x101b9399u, 0x0b182cacu},
    {0xdb980133u, 0x42d9d3f5u, 0x1c232a64u, 0xc6cf90adu, 0x3c40659cu, 0x13e6632du, 0x0d4c1580u, 0x757b3b08u, 0x7be315dcu, 0x72fc00aeu, 0xad1eca9bu, 0x0245a394u},
    {0x5475224bu, 0x866b1e71u, 0x6579afb7u, 0x6ba1049bu, 0x396a7ce4u, 0xd9ab0f5du, 0xd7e86568u, 0x5e673d81u, 0x48c4a3fcu, 0x02a159f7u, 0x5e44cf11u, 0x05c12964u},
    {0x69c8b604u, 0x04b456beu, 0xfec01c77u, 0xb665027eu, 0x95af01b2u, 0x57add4fau, 0x84965a39u, 0xcb181d8fu, 0x42df2eb5u, 0x4ea50b3bu, 0x990f03ceu, 0x15e6be4eu},
    {0xb03663c1u, 0x01479253u, 0xf60c206du, 0x07f3688eu, 0x5be72e7au, 0xeec3232bu, 0x78980be6u, 0x601a6de5u, 0xfad0eae9u, 0x52181140u, 0x3a9c98b2u, 0x16112c4cu},
    {0x2e49a03du, 0x32f6102cu, 0x63529e35u, 0x78a42607u, 0xf453e01fu, 0xa4a10356u, 0x31c4d59cu, 0x85c84ff7u, 0x43c348b8u, 0x1a0cbd6cu, 0x2381201eu, 0x1962d75cu},
    {0x3dbf67f2u, 0x1e2538b5u, 0x36f96f89u, 0xa6757cd6u, 0x279cd2ecu, 0x0c35a5ddu, 0x51ae7f31u, 0x78c48555u, 0x6e8eb157u, 0x6faaae7du, 0x6640da27u, 0x058df330u},
    {0x445f5416u, 0xa8d26d98u, 0xc28297adu, 0x727364f2u, 0xe726af41u, 0x123da489u, 0xddbcd30eu, 0xd115c5dbu, 0x89edb4d1u, 0xf20d23bfu, 0x798e5395u, 0x16b7d288u},
    {0x11a5001du, 0xda391423u, 0x0fd2ededu, 0xa20b15dcu, 0xc9dec916u, 0x542eda0fu, 0x0f69bbb0u, 0xc6d19c9fu, 0xf8228ddcu, 0xb00cc912u, 0x545f43e4u, 0x0be0e079u},
    {0xaaf9b7acu, 0x02c6477fu, 0xdfa9cce2u, 0x49f38db9u, 0x6f0f5a64u, 0xc5ecd87bu, 0x5550d881u, 0xb70152c6u, 0xac783182u, 0x9fb266eau, 0x7186db2du, 0x08d9e529u},
    {0x126a775cu, 0x3d1a1399u, 0xa58b1fb9u, 0xd5fa9c01u, 0x400a0051u, 0x5dd365bcu, 0x8d0cf8efu, 0x5eecfdfau, 0xace9824bu, 0xc3ba8734u, 0x8a99db2fu, 0x166007c0u},
    {0x15812ed9u, 0x60ee415au, 0x0801dee4u, 0xb920f5b0u, 0x06357132u, 0xfeb34fd2u, 0xfa1f4fd7u, 0xe5a4375eu, 0xbba6ff6eu, 0x03bcddfau, 0xbe3ea7eau, 0x16a3ef08u},
    {0x55535d4au, 0x6b233d9du, 0xbb924883u, 0x52cfe2f7u, 0x4bf39b48u, 0xabc5750cu, 0xc6af5920u, 0xf9fb0ce4u, 0xd1d74cc4u, 0x1a1be54fu, 0x336c6123u, 0x1866c8edu},
    {0xb8913f55u, 0x346ef48bu, 0xd529b35eu, 0xc7385ea3u, 0x7ea7d4fbu, 0x5308592eu, 0xe13d87bbu, 0x3216f763u, 0xd94a8490u, 0xea820597u, 0xa70a6e1cu, 0x167a55cdu},
    {0xba8f6aa8u, 0x00f8b49cu, 0x4f830604u, 0x71a5c29fu, 0xe636a5c8u, 0x0e591b36u, 0xbb61a629u, 0x9c6dd039u, 0x1ad2911du, 0x48f010a0u, 0xeea405bdu, 0x04d2f259u},
    {0xe2561092u, 0x9684b529u, 0x6f7ebbeau, 0x16f96898u, 0xcea79135u, 0x8c0f9a88u, 0xefce42d2u, 0x7f94ff8au, 0x48c50c47u, 0xf5852c1eu, 0x481d033fu, 0x0accbb67u},
    {0x573345ccu, 0x1e99b138u, 0xe3b90ac1u, 0x93000763u, 0xa00d9b86u, 0x7d5ceef9u, 0x8adf0226u, 0x543346d9u, 0xb45f1496u, 0xc3613144u, 0x4c767fe3u, 0x0ad6b951u},
    {0x26ed06f7u, 0xd1fadc13u, 0x8714cc80u, 0x420517bdu, 0x7942480eu, 0xcb748df2u, 0xe72927c1u, 0xbf565b94u, 0x53cd76f2u, 0x628bdd0du, 0xeb2e4f3bu, 0x02660400u},
    {0x1d634b8fu, 0x4415473au, 0xf1349780u, 0x5ca2f570u, 0x356caa20u, 0x324efcd6u, 0xe273b853u, 0x71c40f65u, 0x0d7819c1u, 0x6b24255eu, 0x16ddc03eu, 0x0e0fa1d8u},
};

// G2, RFC 9380 8.8.2: A' = 240 i, B' = 1012 (1 + i), Z = -(2 + i), -B'/A', B'/(Z A'), then psi's c_x = 1/(1+i)^((p-1)/3) and
// c_y = 1/(1+i)^((p-1)/2); each entry {c0, c1}
__constant__ uint32_t kG2Consts[7][2][12] = {
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0x000000f0u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
    {{0x000003f4u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0x000003f4u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
    {{0xffffaaa9u, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}, {0xffffaaaau, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}},
    {{0xccccb1c3u, 0x725d8cccu, 0xda498888u, 0xd6834443u, 0x2bfc4df1u, 0x02cf75e6u, 0x6f3f7923u, 0x9b8c2d3fu, 0x0cc6e5aau, 0xfe2f284fu, 0x1abdd5d2u, 0x083c1279u}, {0x3332f8e8u, 0x47a17333u, 0xd70a7777u, 0x4828bbbau, 0xcab4a832u, 0x64615cbau, 0x8445999cu, 0xc8eb1e45u, 0x3684c72cu, 0x4cec7f67u, 0x1ec210c7u, 0x11c4ff71u}},
    {{0x28f5bd27u, 0xe3ac4f5cu, 0x5edb81b4u, 0x5e1a40dau, 0xa265a930u, 0x66f64ac7u, 0x7ca64b6du, 0xebe8d5d9u, 0x028e2deeu, 0x32d63b43u, 0x6bbf912au, 0x01a59d4bu}, {0x851e7336u, 0x0efa11ebu, 0x94c17ae1u, 0x045d3d6fu, 0x0f7ffa93u, 0x324df24au, 0x7d923077u, 0xa0bcc9f8u, 0x3ba1230au, 0xb298f5edu, 0xf641331bu, 0x15103a07u}},
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0x0000aaadu, 0x8bfd0000u, 0x4f49fffdu, 0x409427ebu, 0x0fb85f9bu, 0x897d2965u, 0x89759ad4u, 0xaa0d857du, 0x63d4de85u, 0xec024086u, 0x397fe699u, 0x1a0111eau}},
    {{0x121bdea2u, 0xf1ee7b04u, 0x3e67fa0au, 0x304466cfu, 0xf61eb45eu, 0xef396489u, 0x30b1cf60u, 0x1c3dedd9u, 0xd77a2cd9u, 0xe2e9c448u, 0x0180a68eu, 0x135203e6u}, {0xede3cc09u, 0xc81084fbu, 0x72ec05f4u, 0xee67992fu, 0x009241c5u, 0x77f76e17u, 0xc2d3435eu, 0x48395dabu, 0x6bd17ffeu, 0x6831e36du, 0x37ff400bu, 0x06af0e04u}},
};

// G2 3-isogeny, RFC 9380 Appendix E.3: x_num k_(1,0..3), x_den k_(2,0..1), y_num k_(3,0..3), y_den k_(4,0..2)
__constant__ uint32_t kG2Iso[13][2][12] = {
    {{0xaaaa97d6u, 0x6238aaaau, 0x43d9c71cu, 0x5c2638e3u, 0xc50ae15du, 0x88b58423u, 0xfd3a042au, 0x32c52d39u, 0x47d7ed85u, 0xbb5b7a9au, 0x7e8e333eu, 0x05c75950u}, {0xaaaa97d6u, 0x6238aaaau, 0x43d9c71cu, 0x5c2638e3u, 0xc50ae15du, 0x88b58423u, 0xfd3a042au, 0x32c52d39u, 0x47d7ed85u, 0xbb5b7a9au, 0x7e8e333eu, 0x05c75950u}},
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0xffffc71au, 0x26a9ffffu, 0xcb8d5555u, 0x1472aaa9u, 0x4f20a418u, 0x9a208c6bu, 0xf7ae0c7fu, 0x984f87adu, 0xd787c88fu, 0x32126fceu, 0x7baa99bcu, 0x11560bf1u}},
    {{0xffffc71eu, 0x26a9ffffu, 0xcb8d5555u, 0x1472aaa9u, 0x4f20a418u, 0x9a208c6bu, 0xf7ae0c7fu, 0x984f87adu, 0xd787c88fu, 0x32126fceu, 0x7baa99bcu, 0x11560bf1u}, {0xffffe38du, 0x9354ffffu, 0xe5c6aaaau, 0x0a395554u, 0xa790520cu, 0xcd104635u, 0xfbd7063fu, 0xcc27c3d6u, 0x6bc3e447u, 0x190937e7u, 0xbdd54cdeu, 0x08ab05f8u}},
    {{0xaaaa5ed1u, 0x88e2aaaau, 0x0f671c71u, 0x7098e38du, 0x142b8575u, 0x22d6108fu, 0xf4e810aau, 0xcb14b4e7u, 0x1f5fb614u, 0xed6dea69u, 0xfa38ccfau, 0x171d6541u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0xffffaa63u, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}},
    {{0x0000000cu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0xffffaa9fu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}},
    {{0x71c6d706u, 0x12cfc71cu, 0xf8c92f68u, 0xfc8c25ebu, 0x7d27e500u, 0xf54439d8u, 0xa07f649bu, 0x0f7da5d4u, 0x076d1193u, 0x59a4c18bu, 0x7ab4113bu, 0x1530477cu}, {0x71c6d706u, 0x12cfc71cu, 0xf8c92f68u, 0xfc8c25ebu, 0x7d27e500u, 0xf54439d8u, 0xa07f649bu, 0x0f7da5d4u, 0x076d1193u, 0x59a4c18bu, 0x7ab4113bu, 0x1530477cu}},
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0xaaaa97beu, 0x6238aaaau, 0x43d9c71cu, 0x5c2638e3u, 0xc50ae15du, 0x88b58423u, 0xfd3a042au, 0x32c52d39u, 0x47d7ed85u, 0xbb5b7a9au, 0x7e8e333eu, 0x05c75950u}},
    {{0xffffc71cu, 0x26a9ffffu, 0xcb8d5555u, 0x1472aaa9u, 0x4f20a418u, 0x9a208c6bu, 0xf7ae0c7fu, 0x984f87adu, 0xd787c88fu, 0x32126fceu, 0x7baa99bcu, 0x11560bf1u}, {0xffffe38fu, 0x9354ffffu, 0xe5c6aaaau, 0x0a395554u, 0xa790520cu, 0xcd104635u, 0xfbd7063fu, 0xcc27c3d6u, 0x6bc3e447u, 0x190937e7u, 0xbdd54cdeu, 0x08ab05f8u}},
    {{0x1c718b10u, 0xe1b371c7u, 0x56dc4bd9u, 0x4e79097au, 0x9aa27452u, 0xb0e977c6u, 0xa1e26286u, 0x761b0f37u, 0xe3811ad0u, 0xfbf7043du, 0x3b6cf79bu, 0x124c9ad4u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
    {{0xffffa8fbu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}, {0xffffa8fbu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}},
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0xffffa9d3u, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}},
    {{0x00000012u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}, {0xffffaa99u, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau}},
};


constexpr uint64_t kZAbs = 0xd201000000010000ull;    // |z|, z = -0xd201000000010000
constexpr uint64_t kHeffG1 = 0xd201000000010001ull;  // 1 - z

B2_D Fp381 fp_const(const uint32_t (&c)[12]) {
  Fp381 v;
#pragma unroll
  for (int k = 0; k < 12; ++k) v.v[k] = c[k];
  return Fp381::to_mont(v);
}

template <class F> struct MapCurve;
template <> struct MapCurve<Fp381> {
  static constexpr int kXNum = 12, kXDen = 10, kYNum = 16, kYDen = 15;
  static B2_D Fp381 k(int i) { return fp_const(kG1Consts[i]); }
  static B2_D Fp381 iso(int i) { return fp_const(kG1Iso[i]); }
  static B2_D uint32_t sgn0(const Fp381& a) { return Fp381::from_mont(a).v[0] & 1; }  // parity of the canonical value
};
template <> struct MapCurve<F2> {
  static constexpr int kXNum = 4, kXDen = 2, kYNum = 4, kYDen = 3;
  static B2_D F2 k(int i) { return {fp_const(kG2Consts[i][0]), fp_const(kG2Consts[i][1])}; }
  static B2_D F2 iso(int i) { return {fp_const(kG2Iso[i][0]), fp_const(kG2Iso[i][1])}; }
  static B2_D uint32_t sgn0(const F2& a) {  // sgn0(c0) OR (c0 = 0 AND sgn0(c1))
    const Fp381 c0 = Fp381::from_mont(a.c0), c1 = Fp381::from_mont(a.c1);
    return (c0.v[0] & 1) | (c0.is_zero() ? c1.v[0] & 1 : 0u);
  }
};

// Horner over table entries [off, off + n) in ascending powers; a monic polynomial's leading 1 is not in the table
template <class F> B2_D F horner(int off, int n, bool monic, const F& x) {
  F acc = monic ? F::one() : MapCurve<F>::iso(off + n - 1);
#pragma unroll 1
  for (int i = monic ? n - 1 : n - 2; i >= 0; --i) acc = F::add(F::mul(acc, x), MapCurve<F>::iso(off + i));
  return acc;
}

template <class F> B2_D F curve_rhs(const F& x) {  // g(x) = x^3 + A' x + B' on E'
  return F::add(F::mul(F::add(F::sqr(x), MapCurve<F>::k(kA)), x), MapCurve<F>::k(kB));
}

// map_to_curve_simple_swu: a point (x, y) of E'
template <class F> __device__ __noinline__ void sswu(const F& u, F* x, F* y) {
  typedef MapCurve<F> C;
  const F zu2 = F::mul(C::k(kZ), F::sqr(u));
  const F tv1 = F::inv(F::add(F::sqr(zu2), zu2));  // inv0: 0 when Z^2 u^4 + Z u^2 = 0
  const F x1 = tv1.is_zero() ? C::k(kBZA) : F::mul(C::k(kNegBA), F::add(F::one(), tv1));
  const F g1 = curve_rhs(x1);
  *y = F::sqrt_candidate(g1);
  *x = x1;
  if (F::sqr(*y) != g1) {  // g(x1) is not a square, so g(Z u^2 x1) = Z^3 u^6 g(x1) is
    *x = F::mul(zu2, x1);
    *y = F::sqrt_candidate(curve_rhs(*x));
  }
  if (C::sgn0(u) != C::sgn0(*y)) *y = F::neg(*y);
}

// iso_map onto E / E2 as an XYZZ point: (x_num / x_den, y y_num / y_den) = (X / t^2, Y / t^3) with t = x_den y_den,
// X = x_num x_den y_den^2, Y = y y_num x_den^3 y_den^2; the identity when t = 0
template <class F> __device__ __noinline__ XYZZ<F> iso_map(const F& x, const F& y) {
  typedef MapCurve<F> C;
  const F xn = horner(0, C::kXNum, false, x), xd = horner(C::kXNum, C::kXDen, true, x);
  const F yn = horner(C::kXNum + C::kXDen, C::kYNum, false, x), yd = horner(C::kXNum + C::kXDen + C::kYNum, C::kYDen, true, x);
  const F t = F::mul(xd, yd);
  if (t.is_zero()) return XYZZ<F>::identity();
  const F yd2 = F::sqr(yd);
  XYZZ<F> r;
  r.x = F::mul(F::mul(xn, xd), yd2);
  r.y = F::mul(F::mul(y, yn), F::mul(F::mul(F::sqr(xd), xd), yd2));
  r.zz = F::sqr(t);
  r.zzz = F::mul(r.zz, t);
  return r;
}

// k P for a 64-bit k > 0 (double-and-add, MSB first)
template <class F> __device__ __noinline__ XYZZ<F> mul_u64(uint64_t k, const XYZZ<F>& p) {
  XYZZ<F> acc = p;
#pragma unroll 1
  for (int i = 62 - __clzll(k); i >= 0; --i) {
    acc = xyzz_dbl(acc);
    if ((k >> i) & 1) xyzz_add(acc, p);
  }
  return acc;
}

template <class F> B2_D XYZZ<F> xyzz_neg(XYZZ<F> p) { p.y = F::neg(p.y); return p; }

// acc += q, one out-of-line copy for the psi chain's five additions
__device__ __noinline__ void add_to(XYZZ<F2>& acc, const XYZZ<F2>& q) { xyzz_add(acc, q); }

B2_D XYZZ<Fp381> clear_cofactor(const XYZZ<Fp381>& p) { return mul_u64(kHeffG1, p); }

// psi(x, y) = (c_x conj(x), c_y conj(y)); on XYZZ coordinates conj also applies to ZZ and ZZZ
__device__ __noinline__ XYZZ<F2> psi(const XYZZ<F2>& p) {
  return {F2::mul(MapCurve<F2>::k(kPsiX), F2::conj(p.x)), F2::mul(MapCurve<F2>::k(kPsiY), F2::conj(p.y)), F2::conj(p.zz), F2::conj(p.zzz)};
}

B2_D XYZZ<F2> mul_z(const XYZZ<F2>& p) { return xyzz_neg(mul_u64(kZAbs, p)); }

// RFC 9380 Appendix G.3: [z^2 - z - 1] P + [z - 1] psi(P) + psi^2(2 P) = h_eff P
__device__ __noinline__ XYZZ<F2> clear_cofactor(const XYZZ<F2>& p) {
  const XYZZ<F2> t1 = mul_z(p);
  XYZZ<F2> t2 = psi(p);
  XYZZ<F2> t3 = psi(psi(xyzz_dbl(p)));
  add_to(t3, xyzz_neg(t2));
  add_to(t2, t1);
  add_to(t3, mul_z(t2));
  add_to(t3, xyzz_neg(t1));
  add_to(t3, xyzz_neg(p));
  return t3;
}

// ---- kernel -------------------------------------------------------------------------------------------------------------
// one thread per item: out[i] = map(u[i]), st[i] = 0, 1 (the identity) or 2 (nonzero padding or a value >= p)
template <class F>
__global__ void __launch_bounds__(64) bls_map(const uint8_t* __restrict__ in, size_t n, uint8_t* out, uint8_t* st) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> r = {F::zero(), F::zero()};
  F u;
  uint32_t s;
  if (!load_fe64(in + fe_bytes<F>() * i, &u)) s = B200ZK_ERR_NOT_IN_FIELD;
  else {
    F x, y;
    sswu(u, &x, &y);
    r = xyzz_to_affine(clear_cofactor(iso_map(x, y)));
    s = r.is_inf() ? B200ZK_OK_INFINITY : B200ZK_OK;
  }
  store_point64(out + point_bytes<F>() * i, r);
  st[i] = (uint8_t)s;
}

// ---- host side ----------------------------------------------------------------------------------------------------------
template <class F>
int map_batch(b200zk_ctx* ctx, const char* what, const uint8_t* in, size_t count, uint8_t* out, uint8_t* status) {
  const std::string w = what;
  if (!ctx || (count && (!in || !out || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, (w + ": null argument").c_str());
  NvtxRange nvtx(("b200zk:" + w).c_str());
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  constexpr size_t kFe = fe_bytes<F>(), kPt = point_bytes<F>();
  cudaStream_t st = ctx->stream;
  uint8_t *din, *dout, *dst;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) { din = c.take<uint8_t>(kFe * count); dout = c.take<uint8_t>(kPt * count); dst = c.take<uint8_t>(count); }));
  B2_CUDA(ctx, cudaMemcpyAsync(din, in, kFe * count, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_map<F>, (unsigned)((count + 63) / 64), 64, 0, st, (const uint8_t*)din, count, dout, dst);
  B2_CUDA(ctx, cudaMemcpyAsync(out, dout, kPt * count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, dst, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_bls12_381_map_fp_to_g1_batch(b200zk_ctx* ctx, const uint8_t* fps, size_t count, uint8_t* out, uint8_t* status) {
  return map_batch<Fp381>(ctx, "bls12_381_map_fp_to_g1_batch", fps, count, out, status);
}

int b200zk_bls12_381_map_fp2_to_g2_batch(b200zk_ctx* ctx, const uint8_t* fp2s, size_t count, uint8_t* out, uint8_t* status) {
  return map_batch<F2>(ctx, "bls12_381_map_fp2_to_g2_batch", fp2s, count, out, status);
}

}  // extern "C"
