// Drives <curve>::ToLagrangeG1 of the C++ host mirror (include/gmsm.hpp): the reference's error texts and, on the GPU, tiny known
// answers on bn254 G1.  Built and run by tests/test_gpu_to_lagrange.py.
#include <cstdio>
#include <string>
#include <vector>

#include "gmsm.hpp"

using namespace gmsm_host;

static int fails = 0;
#define CHECK(cond) do { if (!(cond)) { std::printf("FAIL line %d: %s\n", __LINE__, #cond); fails++; } } while (0)

template <class Fn>
static std::string error_of(Fn&& fn) {
  try { fn(); } catch (const Error& e) { return e.what(); }
  return "";
}

int main() {
  // bn254 G1 generator (1, 2) in Montgomery limbs (ecc/bn254/bn254.go:111-113)
  bn254::G1Affine G, inf;
  G.X = {0xd35d438dc58f0d9dull, 0x0a78eb28f5c70b3dull, 0x666ea36f7879462cull, 0x0e0a77c19a07df2full};
  G.Y = {0xa6ba871b8b1e1b3aull, 0x14f1d651eb8e167bull, 0xccdd46def0f28c58ull, 0x1c14ef83340fbe5eull};

  const std::string pow2 = "len(coeffs) must be a power of 2";
  CHECK(error_of([&] { bn254::ToLagrangeG1({}); }) == pow2);
  CHECK(error_of([&] { bn254::ToLagrangeG1({G, G, G}); }) == pow2);
  CHECK(error_of([&] { bls12381::ToLagrangeG1(std::vector<bls12381::G1Affine>(6)); }) == pow2);
  CHECK(error_of([&] { bls12377::ToLagrangeG1(std::vector<bls12377::G1Affine>(3)); }) == pow2);
  CHECK(error_of([&] { bls24315::ToLagrangeG1(std::vector<bls24315::G1Affine>(3)); }) == pow2);
  CHECK(error_of([&] { bls24317::ToLagrangeG1(std::vector<bls24317::G1Affine>(3)); }) == pow2);
  CHECK(error_of([&] { bw6633::ToLagrangeG1(std::vector<bw6633::G1Affine>(3)); }) == pow2);
  CHECK(error_of([&] { bw6761::ToLagrangeG1(std::vector<bw6761::G1Affine>(3)); }) == pow2);

  // n = 1 is the identity; (G, G) -> ([1/2](G + G), [1/2](G - G)) = (G, infinity); (G, inf, inf, inf) -> [1/4]G everywhere
  CHECK(bn254::ToLagrangeG1({G}) == std::vector<bn254::G1Affine>{G});
  const std::vector<bn254::G1Affine> two = bn254::ToLagrangeG1({G, G});
  CHECK(two.size() == 2 && two[0] == G && two[1].IsInfinity());
  const std::vector<bn254::G1Affine> four = bn254::ToLagrangeG1({G, inf, inf, inf});
  CHECK(four.size() == 4 && !four[0].IsInfinity() && four[1] == four[0] && four[2] == four[0] && four[3] == four[0]);
  const std::vector<bn254::G1Affine> again = bn254::ToLagrangeG1({four[0], four[0]});   // (P, P) -> (P, infinity) again
  CHECK(again[0] == four[0] && again[1].IsInfinity());

  if (fails) return 1;
  std::printf("LAGRANGE_OK\n");
  return 0;
}
