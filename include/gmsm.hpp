// gmsm.hpp -- C++ host-side mirror of the reference interface for the MultiExp path, over the C ABI (gmsm.h).
//
// The reference is Go (compiled), and there is no Go toolchain in this environment; this header is what a
// compiled-language caller binds instead of the cgo shim of INTEGRATION.md.  Same names, argument meaning
// and error behaviour as ecc/<curve>/multiexp.go (reference tree):
//
//   (*G1Jac).MultiExp(points []G1Affine, scalars []fr.Element, config ecc.MultiExpConfig) (*G1Jac, error)
//        ecc/bn254/multiexp.go:32 (G1Affine :20, G2Jac :357, G2Affine :345), ecc/bls12-381/multiexp.go:20-355
//   ecc.MultiExpConfig{NbTasks int}                                      ecc/ecc.go:107-110
//   errors: "len(points) != len(scalars)" (multiexp.go:61-64), "invalid config: config.NbTasks > 1024" (:69-71)
//   kzg.ToLagrangeG1(coeffs []G1Affine) ([]G1Affine, error)              ecc/<curve>/kzg/utils.go:25-64 (pairing curves)
//
// Types are the reference's memory images: Element<L> = [L]uint64 little-endian Montgomery limbs.
#pragma once
#include <array>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "gmsm.h"

namespace gmsm_host {

struct MultiExpConfig {  // ecc.MultiExpConfig
  int NbTasks = 0;
};

struct Error : std::runtime_error {  // the Go `error`
  using std::runtime_error::runtime_error;
};

template <int L>
using Element = std::array<uint64_t, L>;

// EXT = 1: coordinates in Fp, 2: in Fp2 (E2{A0,A1}); LR = fr.Limbs (4; 5 for bw6-633, 6 for bw6-761)
template <gmsm_curve_t CURVE, int L, int EXT, int LR = 4>
struct Group {
  static constexpr gmsm_curve_t curve = CURVE;
  using Coord = std::array<uint64_t, L * EXT>;
  using Scalar = Element<LR>;  // fr.Element

  struct Affine {  // G1Affine / G2Affine: {X, Y}; infinity = all zero (g1.go:41-47)
    Coord X{}, Y{};
    bool IsInfinity() const {
      for (auto v : X) if (v) return false;
      for (auto v : Y) if (v) return false;
      return true;
    }
    bool operator==(const Affine& o) const { return X == o.X && Y == o.Y; }
  };

  struct Jac {  // G1Jac / G2Jac: {X, Y, Z}
    Coord X{}, Y{}, Z{};

    // (*G1Jac).MultiExp: the receiver is overwritten and returned
    Jac& MultiExp(const std::vector<Affine>& points, const std::vector<Scalar>& scalars, MultiExpConfig config = {}) {
      if (points.size() != scalars.size()) throw Error("len(points) != len(scalars)");
      static_assert(sizeof(Affine) == 2 * sizeof(Coord) && sizeof(Jac) == 3 * sizeof(Coord), "Go memory layout");
      int rc = gmsm_multiexp(CURVE, points.empty() ? nullptr : points[0].X.data(),
                             scalars.empty() ? nullptr : scalars[0].data(), points.size(), config.NbTasks, X.data());
      if (rc != GMSM_OK) throw Error(gmsm_last_error());
      return *this;
    }
    bool IsInfinity() const {
      for (auto v : Z) if (v) return false;
      return true;
    }
  };

  // (*G1Affine).MultiExp (multiexp.go:20-27): Jacobian MultiExp, then FromJacobian.  The engine returns the
  // affine-normalised representative (x, y, One) or (0,0,0), so FromJacobian (g1.go:150-166) is a copy.
  static Affine MultiExpAffine(const std::vector<Affine>& points, const std::vector<Scalar>& scalars,
                               MultiExpConfig config = {}) {
    Jac j;
    j.MultiExp(points, scalars, config);
    Affine a;
    if (!j.IsInfinity()) { a.X = j.X; a.Y = j.Y; }
    return a;
  }

  // Resident bases (gmsm_bases_*): the static-SRS flow of kzg.Commit (kzg/kzg.go:159-176 passes pk.G1[:len(p)]):
  // bases uploaded once, scalars per call.  Precompute() replaces them by window tables (gmsm_bases_precompute).
  class ResidentBases {
   public:
    explicit ResidentBases(const std::vector<Affine>& points, int device = 0)
        : n_(points.size()), h_(gmsm_bases_upload(CURVE, points.empty() ? nullptr : points[0].X.data(), points.size(), device)) {
      if (!h_) throw Error(gmsm_last_error());
    }
    ResidentBases(const ResidentBases&) = delete;
    ResidentBases& operator=(const ResidentBases&) = delete;
    ~ResidentBases() { gmsm_bases_free(h_); }
    // MultiExp over bases[offset, offset + len(scalars))
    Jac MultiExp(const std::vector<Scalar>& scalars, MultiExpConfig config = {}, size_t offset = 0) const {
      if (offset > n_ || scalars.size() > n_ - offset) throw Error("len(points) != len(scalars)");
      Jac j;
      int rc = gmsm_bases_multiexp(h_, offset, scalars.empty() ? nullptr : scalars[0].data(), scalars.size(), config.NbTasks, j.X.data());
      if (rc != GMSM_OK) throw Error(gmsm_last_error());
      return j;
    }
    int Precompute(int c = 0) {   // returns the table window width
      if (gmsm_bases_precompute(h_, c) != GMSM_OK) throw Error(gmsm_last_error());
      return gmsm_bases_table_bits(h_);
    }

   private:
    size_t n_;
    gmsm_bases_t* h_;
  };

  // BatchScalarMultiplicationG1 / G2 (g1.go:1039-1118)
  static std::vector<Affine> BatchScalarMultiplication(const Affine& base, const std::vector<Scalar>& scalars) {
    std::vector<Affine> out(scalars.size());
    int rc = gmsm_batch_scalar_mul(CURVE, base.X.data(), scalars.empty() ? nullptr : scalars[0].data(), scalars.size(),
                                   out.empty() ? nullptr : out[0].X.data());
    if (rc != GMSM_OK) throw Error(gmsm_last_error());
    return out;
  }
};

// kzg.ToLagrangeG1 (ecc/<curve>/kzg/utils.go:25-64): the Lagrange form of a canonical SRS, len(coeffs) a power of two; the
// input is left unmodified.  Wrapped below as <curve>::ToLagrangeG1 for the seven pairing curves.
template <class G1>
std::vector<typename G1::Affine> to_lagrange_g1(const std::vector<typename G1::Affine>& coeffs, int device) {
  std::vector<typename G1::Affine> out(coeffs.size());
  int rc = gmsm_g1_to_lagrange(G1::curve, coeffs.empty() ? nullptr : coeffs[0].X.data(), coeffs.size(), device,
                               out.empty() ? nullptr : out[0].X.data());
  if (rc != GMSM_OK) throw Error(gmsm_last_error());
  return out;
}
#define GMSM_HOST_TO_LAGRANGE                                                                                          \
  inline std::vector<G1Affine> ToLagrangeG1(const std::vector<G1Affine>& coeffs, int device = 0) {                  \
    return to_lagrange_g1<G1>(coeffs, device);                                                                       \
  }

// pairing.go MillerLoop / FinalExponentiation / Pair / PairingCheck for bn254 and bls12-381 (gmsm_pair*): GT = E12 as 12
// Montgomery fp.Elements.  Wrapped below in the two curve namespaces.
template <class G1, class G2, int L>
struct Pairing {
  using GT = std::array<uint64_t, 12 * L>;
  static void sizes(size_t np, size_t nq) {
    if (np == 0 || np != nq) throw Error("invalid inputs sizes");
  }
  static GT MillerLoop(const std::vector<typename G1::Affine>& P, const std::vector<typename G2::Affine>& Q) {
    sizes(P.size(), Q.size());
    GT out{};
    if (gmsm_pairing_miller_loop(G1::curve, P[0].X.data(), Q[0].X.data(), P.size(), out.data()) != GMSM_OK) throw Error(gmsm_last_error());
    return out;
  }
  static GT FinalExponentiation(const GT& z, const std::vector<GT>& zs = {}) {
    std::vector<GT> all{z};
    all.insert(all.end(), zs.begin(), zs.end());
    GT out{};
    if (gmsm_pairing_final_exp(G1::curve, all[0].data(), all.size(), out.data()) != GMSM_OK) throw Error(gmsm_last_error());
    return out;
  }
  static GT Pair(const std::vector<typename G1::Affine>& P, const std::vector<typename G2::Affine>& Q) {
    sizes(P.size(), Q.size());
    GT out{};
    if (gmsm_pair(G1::curve, P[0].X.data(), Q[0].X.data(), P.size(), out.data()) != GMSM_OK) throw Error(gmsm_last_error());
    return out;
  }
  // Pair(P, Q) == 1; the one of GT is the Miller loop of a pair at infinity, which the library returns as 1
  static bool PairingCheck(const std::vector<typename G1::Affine>& P, const std::vector<typename G2::Affine>& Q) {
    const GT f = Pair(P, Q);
    return f == MillerLoop({typename G1::Affine{}}, {typename G2::Affine{}});
  }
};
#define GMSM_HOST_PAIRING(L)                                                                                                        \
  using GT = Pairing<G1, G2, L>::GT;                                                                                                \
  inline GT MillerLoop(const std::vector<G1Affine>& P, const std::vector<G2Affine>& Q) { return Pairing<G1, G2, L>::MillerLoop(P, Q); } \
  inline GT FinalExponentiation(const GT& z, const std::vector<GT>& zs = {}) { return Pairing<G1, G2, L>::FinalExponentiation(z, zs); } \
  inline GT Pair(const std::vector<G1Affine>& P, const std::vector<G2Affine>& Q) { return Pairing<G1, G2, L>::Pair(P, Q); }            \
  inline bool PairingCheck(const std::vector<G1Affine>& P, const std::vector<G2Affine>& Q) { return Pairing<G1, G2, L>::PairingCheck(P, Q); }

namespace bn254 {
using G1 = Group<GMSM_BN254_G1, 4, 1>;
using G2 = Group<GMSM_BN254_G2, 4, 2>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
using G2Affine = G2::Affine;
using G2Jac = G2::Jac;
GMSM_HOST_TO_LAGRANGE
GMSM_HOST_PAIRING(4)
}  // namespace bn254
namespace bls12381 {
using G1 = Group<GMSM_BLS12381_G1, 6, 1>;
using G2 = Group<GMSM_BLS12381_G2, 6, 2>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
using G2Affine = G2::Affine;
using G2Jac = G2::Jac;
GMSM_HOST_TO_LAGRANGE
GMSM_HOST_PAIRING(6)
}  // namespace bls12381
namespace bls12377 {   // ecc/bls12-377
using G1 = Group<GMSM_BLS12377_G1, 6, 1>;
using G2 = Group<GMSM_BLS12377_G2, 6, 2>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
using G2Affine = G2::Affine;
using G2Jac = G2::Jac;
GMSM_HOST_TO_LAGRANGE
}  // namespace bls12377
namespace secp256k1 {   // ecc/secp256k1 (G1 only)
using G1 = Group<GMSM_SECP256K1_G1, 4, 1>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
}  // namespace secp256k1
namespace bw6761 {   // ecc/bw6-761: both groups over the 12-word Fp, fr.Element = [6]uint64
using G1 = Group<GMSM_BW6761_G1, 12, 1, 6>;
using G2 = Group<GMSM_BW6761_G2, 12, 1, 6>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
using G2Affine = G2::Affine;
using G2Jac = G2::Jac;
GMSM_HOST_TO_LAGRANGE
}  // namespace bw6761
namespace bls24315 {   // ecc/bls24-315 (G1; G2 is over Fp4 and stays on the CPU path)
using G1 = Group<GMSM_BLS24315_G1, 5, 1>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
GMSM_HOST_TO_LAGRANGE
}  // namespace bls24315
namespace bls24317 {   // ecc/bls24-317 (G1)
using G1 = Group<GMSM_BLS24317_G1, 5, 1>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
GMSM_HOST_TO_LAGRANGE
}  // namespace bls24317
namespace bw6633 {   // ecc/bw6-633: both groups over the 10-word Fp, fr.Element = [5]uint64
using G1 = Group<GMSM_BW6633_G1, 10, 1, 5>;
using G2 = Group<GMSM_BW6633_G2, 10, 1, 5>;
using G1Affine = G1::Affine;
using G1Jac = G1::Jac;
using G2Affine = G2::Affine;
using G2Jac = G2::Jac;
GMSM_HOST_TO_LAGRANGE
}  // namespace bw6633

#undef GMSM_HOST_TO_LAGRANGE

}  // namespace gmsm_host
