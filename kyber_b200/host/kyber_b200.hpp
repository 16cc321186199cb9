// kyber_b200.hpp -- C++ host mirror of dedis/kyber's plugin interfaces for the BLS12-381 backend, on top
// of the C ABI (include/b2kyber.h).  The reference is Go; no Go toolchain exists in the build image, so the
// host side is written in C++ with the SAME names, argument meaning and error behaviour:
//
//   kyber::Scalar   <- kyber.Scalar   group.go:23-77     (implemented like mod.Int, group/mod/int.go)
//   kyber::Point    <- kyber.Point    group.go:84-131    (receiver is the destination and is returned)
//   kyber::Group    <- kyber.Group    group.go:175-183
//   pairing::Suite  <- pairing.Suite  pairing/pairing.go:8-20
//   b200::G1Elt / G2Elt / GTElt / Suite   <- pairing/bls12381/kilic/{g1,g2,gt,suite}.go
//   b200::BatchGroup (MulBatch, MSM), Suite::ValidatePairingBatch  -- the batch extension the reference lacks
//
// Conventions copied from the adapters: Mul(s, nullptr) multiplies the base point (kilic/g1.go:111-113);
// aliasing receiver == argument is legal; only (Un)MarshalBinary report errors (here: std::runtime_error for
// "error" returns, std::logic_error for the Go panics); points are host-resident operand bytes, no device
// handles, no finalizers.  All arithmetic runs in the sm_90a kernels behind the C ABI -- there is no CPU
// curve code in this file (scalars are host-side bookkeeping, as in the reference).
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/b2kyber.h"

namespace kyber {

using Bytes = std::vector<uint8_t>;

// ---- 256-bit modular scalar (the role of mod.Int with the BLS12-381 group order) --------------------------
class Scalar {
 public:
  using u128 = unsigned __int128;
  static constexpr uint64_t R[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};
  uint64_t v[4] = {0, 0, 0, 0};

  Scalar() = default;
  explicit Scalar(int64_t x) { SetInt64(x); }
  bool Equal(const Scalar& o) const { return std::memcmp(v, o.v, sizeof v) == 0; }
  Scalar& Set(const Scalar& a) { std::memcpy(v, a.v, sizeof v); return *this; }
  Scalar Clone() const { return *this; }
  Scalar& Zero() { std::memset(v, 0, sizeof v); return *this; }
  Scalar& One() { Zero(); v[0] = 1; return *this; }
  Scalar& SetInt64(int64_t x) {
    Zero();
    if (x >= 0) { v[0] = (uint64_t)x; return *this; }
    Scalar t; t.v[0] = (uint64_t)(-(x + 1)) + 1;
    return Neg(t);
  }
  Scalar& Add(const Scalar& a, const Scalar& b) {
    uint64_t t[4]; u128 c = 0;
    for (int i = 0; i < 4; i++) { c += (u128)a.v[i] + b.v[i]; t[i] = (uint64_t)c; c >>= 64; }
    if (c || geq(t)) sub_r(t);
    std::memcpy(v, t, sizeof v); return *this;
  }
  Scalar& Sub(const Scalar& a, const Scalar& b) { Scalar nb; nb.Neg(b); return Add(a, nb); }
  Scalar& Neg(const Scalar& a) {
    if (a.is_zero()) return Zero();
    uint64_t t[4]; u128 br = 0;
    for (int i = 0; i < 4; i++) { u128 d = (u128)R[i] - a.v[i] - (uint64_t)br; t[i] = (uint64_t)d; br = (d >> 64) & 1; }
    std::memcpy(v, t, sizeof v); return *this;
  }
  Scalar& Mul(const Scalar& a, const Scalar& b) {           // schoolbook 512-bit product, bitwise reduction
    uint64_t p[8] = {0};
    for (int i = 0; i < 4; i++) { u128 c = 0; for (int j = 0; j < 4; j++) { c += (u128)a.v[i] * b.v[j] + p[i + j]; p[i + j] = (uint64_t)c; c >>= 64; } p[i + 4] = (uint64_t)c; }
    uint64_t r[4] = {0, 0, 0, 0};
    for (int bit = 511; bit >= 0; bit--) {
      uint64_t top = r[3] >> 63;
      for (int i = 3; i > 0; i--) r[i] = (r[i] << 1) | (r[i - 1] >> 63);
      r[0] = (r[0] << 1) | ((p[bit >> 6] >> (bit & 63)) & 1);
      if (top || geq(r)) sub_r(r);
    }
    std::memcpy(v, r, sizeof v); return *this;
  }
  Scalar& Inv(const Scalar& a) {                            // Fermat: a^(r-2)
    uint64_t e[4]; std::memcpy(e, R, sizeof e); e[0] -= 2;
    Scalar acc; acc.One(); Scalar base = a;
    for (int bit = 254; bit >= 0; bit--) { acc.Mul(acc, acc); if ((e[bit >> 6] >> (bit & 63)) & 1) acc.Mul(acc, base); }
    return Set(acc);
  }
  Scalar& Div(const Scalar& a, const Scalar& b) { Scalar i; i.Inv(b); return Mul(a, i); }
  // MarshalBinary: 32 bytes big-endian (group/mod/int.go:334-349)
  Bytes MarshalBinary() const { Bytes b(32); for (int i = 0; i < 4; i++) for (int k = 0; k < 8; k++) b[(3 - i) * 8 + k] = (uint8_t)(v[i] >> (56 - 8 * k)); return b; }
  int MarshalSize() const { return 32; }
  // UnmarshalBinary: rejects wrong length and values >= r (int.go:359-372)
  void UnmarshalBinary(const Bytes& b) {
    if (b.size() != 32) throw std::runtime_error("UnmarshalBinary: wrong size buffer");
    uint64_t t[4];
    for (int i = 0; i < 4; i++) { uint64_t x = 0; for (int k = 0; k < 8; k++) x = (x << 8) | b[(3 - i) * 8 + k]; t[i] = x; }
    if (geq(t)) throw std::runtime_error("UnmarshalBinary: value out of range");
    std::memcpy(v, t, sizeof v);
  }
  // SetBytes: big-endian, reduced mod r (int.go:404-411)
  Scalar& SetBytes(const Bytes& b) {
    Scalar acc, k256; k256.SetInt64(256);
    for (uint8_t x : b) { acc.Mul(acc, k256); Scalar d; d.v[0] = x; acc.Add(acc, d); }
    return Set(acc);
  }
  bool is_zero() const { return (v[0] | v[1] | v[2] | v[3]) == 0; }

 private:
  static bool geq(const uint64_t* t) { for (int i = 3; i >= 0; i--) { if (t[i] > R[i]) return true; if (t[i] < R[i]) return false; } return true; }
  static void sub_r(uint64_t* t) { u128 br = 0; for (int i = 0; i < 4; i++) { u128 d = (u128)t[i] - R[i] - (uint64_t)br; t[i] = (uint64_t)d; br = (d >> 64) & 1; } }
};

// ---- kyber.Point / kyber.Group as abstract interfaces -----------------------------------------------------------
class Point {
 public:
  virtual ~Point() = default;
  virtual bool Equal(const Point& o) const = 0;
  virtual Point& Null() = 0;
  virtual Point& Base() = 0;
  virtual Point& Set(const Point& p) = 0;
  virtual std::unique_ptr<Point> Clone() const = 0;
  virtual Point& Add(const Point& a, const Point& b) = 0;
  virtual Point& Sub(const Point& a, const Point& b) = 0;
  virtual Point& Neg(const Point& a) = 0;
  virtual Point& Mul(const Scalar& s, const Point* p) = 0;     // p == nullptr: base point
  virtual Bytes MarshalBinary() const = 0;
  virtual void UnmarshalBinary(const Bytes& b) = 0;
  virtual int MarshalSize() const = 0;
  virtual std::string String() const = 0;
  // Embed / Data / EmbedLen panic for BLS12-381 (kilic/g1.go:78-88)
  virtual int EmbedLen() const { throw std::logic_error("bls12-381: unsupported operation"); }
};

class Group {
 public:
  virtual ~Group() = default;
  virtual std::string String() const = 0;
  virtual int ScalarLen() const = 0;
  virtual Scalar NewScalar() const { return Scalar(); }
  virtual int PointLen() const = 0;
  virtual std::unique_ptr<Point> NewPoint() const = 0;
  virtual bool IsPrimeOrder() const { return true; }
};

}  // namespace kyber

namespace b200 {

using kyber::Bytes;
using kyber::Point;
using kyber::Scalar;

inline std::string hex(const Bytes& b) { static const char* d = "0123456789abcdef"; std::string s; for (uint8_t x : b) { s += d[x >> 4]; s += d[x & 15]; } return s; }

// One engine (C-ABI context) shared by the elements of a suite.
class Engine {
 public:
  explicit Engine(int device = 0) { if (b2k_create(device, &ctx_) != 0) throw std::runtime_error("b2kyber: no sm_90 device (no CPU fallback)"); }
  ~Engine() { b2k_destroy(ctx_); }
  Engine(const Engine&) = delete;
  b2k_ctx* ctx() const { return ctx_; }
  void check(int rc) const { if (rc != 0) throw std::logic_error(std::string("b2kyber: ") + b2k_last_error(ctx_)); }   // Go: panic
 private:
  b2k_ctx* ctx_ = nullptr;
};

static const uint8_t G1_GEN[96] = {
    0x17, 0xf1, 0xd3, 0xa7, 0x31, 0x97, 0xd7, 0x94, 0x26, 0x95, 0x63, 0x8c, 0x4f, 0xa9, 0xac, 0x0f, 0xc3, 0x68, 0x8c, 0x4f, 0x97, 0x74, 0xb9, 0x05,
    0xa1, 0x4e, 0x3a, 0x3f, 0x17, 0x1b, 0xac, 0x58, 0x6c, 0x55, 0xe8, 0x3f, 0xf9, 0x7a, 0x1a, 0xef, 0xfb, 0x3a, 0xf0, 0x0a, 0xdb, 0x22, 0xc6, 0xbb,
    0x08, 0xb3, 0xf4, 0x81, 0xe3, 0xaa, 0xa0, 0xf1, 0xa0, 0x9e, 0x30, 0xed, 0x74, 0x1d, 0x8a, 0xe4, 0xfc, 0xf5, 0xe0, 0x95, 0xd5, 0xd0, 0x0a, 0xf6,
    0x00, 0xdb, 0x18, 0xcb, 0x2c, 0x04, 0xb3, 0xed, 0xd0, 0x3c, 0xc7, 0x44, 0xa2, 0x88, 0x8a, 0xe4, 0x0c, 0xaa, 0x23, 0x29, 0x46, 0xc5, 0xe7, 0xe1};
static const uint8_t G2_GEN_COMPRESSED[96] = {   // ZCash compressed generator; expanded once through the engine
    0x93, 0xe0, 0x2b, 0x60, 0x52, 0x71, 0x9f, 0x60, 0x7d, 0xac, 0xd3, 0xa0, 0x88, 0x27, 0x4f, 0x65, 0x59, 0x6b, 0xd0, 0xd0, 0x99, 0x20, 0xb6, 0x1a,
    0xb5, 0xda, 0x61, 0xbb, 0xdc, 0x7f, 0x50, 0x49, 0x33, 0x4c, 0xf1, 0x12, 0x13, 0x94, 0x5d, 0x57, 0xe5, 0xac, 0x7d, 0x05, 0x5d, 0x04, 0x2b, 0x7e,
    0x02, 0x4a, 0xa2, 0xb2, 0xf0, 0x8f, 0x0a, 0x91, 0x26, 0x08, 0x05, 0x27, 0x2d, 0xc5, 0x10, 0x51, 0xc6, 0xe4, 0x7a, 0xd4, 0xfa, 0x40, 0x3b, 0x02,
    0xb4, 0x51, 0x0b, 0x64, 0x7a, 0xe3, 0xd1, 0x77, 0x0b, 0xac, 0x03, 0x26, 0xa8, 0x05, 0xbb, 0xef, 0xd4, 0x80, 0x56, 0xc8, 0xc1, 0x21, 0xbd, 0xb8};

// Element of G1 (AFF = 96, WIRE = 48) or G2 (AFF = 192, WIRE = 96): host-resident operand bytes.
template <int AFF, int WIRE, bool IS_G1>
class Elt : public Point {
 public:
  explicit Elt(std::shared_ptr<Engine> e) : eng_(std::move(e)) { aff_.fill(0); }
  std::array<uint8_t, AFF> aff_;

  static const Elt& cast(const Point& p) {
    auto* q = dynamic_cast<const Elt*>(&p);
    if (!q) throw std::logic_error("bls12-381: point of a different group");   // gnark adapter panics (gnark/g1.go:63)
    return *q;
  }
  bool Equal(const Point& o) const override {
    auto* q = dynamic_cast<const Elt*>(&o);
    return q && aff_ == q->aff_;                                              // kilic returns false on foreign types (g1.go:45-51)
  }
  Point& Null() override { aff_.fill(0); return *this; }
  Point& Base() override {
    if (IS_G1) { std::memcpy(aff_.data(), G1_GEN, 96); return *this; }
    Bytes c(G2_GEN_COMPRESSED, G2_GEN_COMPRESSED + 96);
    UnmarshalBinary(c);
    return *this;
  }
  Point& Set(const Point& p) override { aff_ = cast(p).aff_; return *this; }
  std::unique_ptr<Point> Clone() const override { return std::make_unique<Elt>(*this); }
  Point& Add(const Point& a, const Point& b) override { return lin(cast(a), cast(b), false); }
  Point& Sub(const Point& a, const Point& b) override { return lin(cast(a), cast(b), true); }
  Point& Neg(const Point& a) override {
    Scalar m1; m1.SetInt64(-1);
    return Mul(m1, &a);
  }
  Point& Mul(const Scalar& s, const Point* p) override {
    std::array<uint8_t, AFF> src;
    if (p) src = cast(*p).aff_; else { Elt b(eng_); b.Base(); src = b.aff_; }
    Bytes sb = s.MarshalBinary();
    std::array<uint8_t, AFF> out;
    if (IS_G1) eng_->check(b2k_bls12381_g1_mul_batch_affine(eng_->ctx(), 1, sb.data(), src.data(), out.data()));
    else eng_->check(b2k_bls12381_g2_mul_batch_affine(eng_->ctx(), 1, sb.data(), src.data(), out.data()));
    aff_ = out;
    return *this;
  }
  Bytes MarshalBinary() const override {
    Scalar one; one.One();
    Bytes sb = one.MarshalBinary(), out(WIRE);
    if (IS_G1) eng_->check(b2k_bls12381_g1_mul_batch(eng_->ctx(), 1, sb.data(), aff_.data(), out.data()));
    else eng_->check(b2k_bls12381_g2_mul_batch(eng_->ctx(), 1, sb.data(), aff_.data(), out.data()));
    return out;
  }
  void UnmarshalBinary(const Bytes& b) override {
    if ((int)b.size() != WIRE) throw std::runtime_error("bls12-381: wrong buffer size");
    uint8_t ok = 0;
    std::array<uint8_t, AFF> out;
    if (IS_G1) eng_->check(b2k_bls12381_g1_decompress(eng_->ctx(), 1, b.data(), out.data(), &ok));
    else eng_->check(b2k_bls12381_g2_decompress(eng_->ctx(), 1, b.data(), out.data(), &ok));
    if (!ok) throw std::runtime_error("bls12-381: invalid point encoding");
    aff_ = out;
  }
  int MarshalSize() const override { return WIRE; }
  std::string String() const override { return std::string(IS_G1 ? "bls12-381.G1: " : "bls12-381.G2: ") + hex(MarshalBinary()); }
  bool IsInCorrectGroup() const {                                              // kyber.SubGroupElement (group.go:191-194)
    try { Elt t(eng_); t.UnmarshalBinary(MarshalBinary()); return true; } catch (const std::runtime_error&) { return false; }
  }
  // kyber.HashablePoint (hash.go:13-15), G1 only: Hash(msg) with the suite's DST
  Point& Hash(const Bytes& msg, const std::string& dst = "BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_") {
    static_assert(true, "");
    if (!IS_G1) throw std::logic_error("b200: hash to G2 is not built yet");
    uint32_t offs[2] = {0, (uint32_t)msg.size()};
    uint8_t dummy = 0;
    eng_->check(b2k_bls12381_hash_to_g1(eng_->ctx(), 1, msg.empty() ? &dummy : msg.data(), offs, (const uint8_t*)dst.data(),
                                        (uint32_t)dst.size(), aff_.data()));
    return *this;
  }
  std::shared_ptr<Engine> engine() const { return eng_; }

 private:
  // a + b / a - b on the device (kilic/g1.go:92-108 Add / Sub): one launch, every exceptional case of the group law handled
  Point& lin(const Elt& a, const Elt& b, bool sub) {
    std::array<uint8_t, AFF> x = a.aff_, y = b.aff_, out;            // receiver may alias an argument (bls.go:73)
    if (IS_G1) eng_->check(b2k_bls12381_g1_add_batch(eng_->ctx(), 1, x.data(), y.data(), sub ? 1 : 0, out.data()));
    else eng_->check(b2k_bls12381_g2_add_batch(eng_->ctx(), 1, x.data(), y.data(), sub ? 1 : 0, out.data()));
    aff_ = out;
    return *this;
  }
  std::shared_ptr<Engine> eng_;
};

using G1Elt = Elt<96, 48, true>;
using G2Elt = Elt<192, 96, false>;

// GT element (kilic/gt.go:15-117): held as its 576 MarshalBinary bytes; GT is written additively like every kyber group --
// Add = Fp12 product, Neg = inverse, Mul = exponentiation, Null = 1 (gt.go:33-38, 59-83); Base / Pick panic (gt.go:40-46).
class GTElt {
 public:
  Bytes bytes = one_bytes();
  GTElt() = default;
  explicit GTElt(std::shared_ptr<Engine> e) : eng_(std::move(e)) {}
  static Bytes one_bytes() { Bytes b(576, 0); b[575] = 1; return b; }
  bool Equal(const GTElt& o) const { return bytes == o.bytes; }
  GTElt& Null() { bytes = one_bytes(); return *this; }
  GTElt& Base() { throw std::logic_error("bls12-381.GT.Base(): unsupported operation"); }
  GTElt& Set(const GTElt& o) { bytes = o.bytes; return *this; }
  GTElt Clone() const { return *this; }
  GTElt& Add(const GTElt& a, const GTElt& b) {
    Bytes x = a.bytes, y = b.bytes, out(576);
    eng()->check(b2k_bls12381_gt_mul(eng()->ctx(), 1, x.data(), y.data(), out.data()));
    bytes = out; return *this;
  }
  GTElt& Neg(const GTElt& a) {
    Bytes x = a.bytes, out(576);
    eng()->check(b2k_bls12381_gt_inv(eng()->ctx(), 1, x.data(), out.data()));
    bytes = out; return *this;
  }
  GTElt& Sub(const GTElt& a, const GTElt& b) { GTElt nb(eng_); nb.Neg(b); return Add(a, nb); }      // kilic/gt.go:66-69
  GTElt& Mul(const Scalar& s, const GTElt& q) {
    Bytes sb = s.MarshalBinary(), x = q.bytes, out(576);
    eng()->check(b2k_bls12381_gt_exp(eng()->ctx(), 1, sb.data(), x.data(), out.data()));
    bytes = out; return *this;
  }
  Bytes MarshalBinary() const { return bytes; }
  void UnmarshalBinary(const Bytes& b) {
    if (b.size() != 576) throw std::runtime_error("bls12-381: wrong buffer size for a GT element");
    GTElt t(eng_); t.bytes = b;
    GTElt one(eng_);
    try { one.Add(t, one); } catch (const std::logic_error&) { throw std::runtime_error("bls12-381: GT coefficient is not a canonical field element"); }
    bytes = b;
  }
  int MarshalSize() const { return 576; }
  std::string String() const { return "bls12-381.GT: " + hex(bytes); }
  void bind(std::shared_ptr<Engine> e) { eng_ = std::move(e); }
 private:
  const std::shared_ptr<Engine>& eng() const { if (!eng_) throw std::logic_error("GTElt: no engine bound"); return eng_; }
  std::shared_ptr<Engine> eng_;
};

// kyber.Group for GT (kilic/group.go:74-78: "bls12-381.GT", PointLen 576, not prime-order-flagged)
class GroupGT {
 public:
  explicit GroupGT(std::shared_ptr<Engine> e) : eng_(std::move(e)) {}
  std::string String() const { return "bls12-381.GT"; }
  int ScalarLen() const { return 32; }
  int PointLen() const { return 576; }
  bool IsPrimeOrder() const { return false; }
  GTElt NewPoint() const { return GTElt(eng_); }
 private:
  std::shared_ptr<Engine> eng_;
};

template <class E, int AFF, int WIRE, bool IS_G1>
class GroupImpl : public kyber::Group {
 public:
  explicit GroupImpl(std::shared_ptr<Engine> e) : eng_(std::move(e)) {}
  std::string String() const override { return IS_G1 ? "bls12-381.G1" : "bls12-381.G2"; }   // kilic/group.go:62,70
  int ScalarLen() const override { return 32; }
  int PointLen() const override { return WIRE; }
  std::unique_ptr<Point> NewPoint() const override { return std::make_unique<E>(eng_); }
  // ---- batch extension (SURVEY 8b): dst[i] = s[i] * p[i]
  std::vector<E> MulBatch(const std::vector<Scalar>& s, const std::vector<E>& p) const {
    size_t n = s.size();
    if (p.size() != n) throw std::logic_error("MulBatch: length mismatch");
    Bytes sb(32 * n), pb((size_t)AFF * n), out((size_t)AFF * n);
    for (size_t i = 0; i < n; i++) { Bytes b = s[i].MarshalBinary(); std::memcpy(&sb[32 * i], b.data(), 32); std::memcpy(&pb[(size_t)AFF * i], p[i].aff_.data(), AFF); }
    if (IS_G1) eng_->check(b2k_bls12381_g1_mul_batch_affine(eng_->ctx(), n, sb.data(), pb.data(), out.data()));
    else eng_->check(b2k_bls12381_g2_mul_batch_affine(eng_->ctx(), n, sb.data(), pb.data(), out.data()));
    std::vector<E> r(n, E(eng_));
    for (size_t i = 0; i < n; i++) std::memcpy(r[i].aff_.data(), &out[(size_t)AFF * i], AFF);
    return r;
  }
  // sum s[i] * p[i]  (replaces the Mul+Add loops of share/poly.go:461-473, sign/bdn/bdn.go:126-161)
  E MSM(const std::vector<Scalar>& s, const std::vector<E>& p) const {
    size_t n = s.size();
    if (p.size() != n || n == 0) throw std::logic_error("MSM: length mismatch");
    Bytes sb(32 * n), pb((size_t)AFF * n);
    for (size_t i = 0; i < n; i++) { Bytes b = s[i].MarshalBinary(); std::memcpy(&sb[32 * i], b.data(), 32); std::memcpy(&pb[(size_t)AFF * i], p[i].aff_.data(), AFF); }
    E r(eng_);
    if (IS_G1) eng_->check(b2k_bls12381_g1_msm_affine(eng_->ctx(), n, sb.data(), pb.data(), r.aff_.data()));
    else eng_->check(b2k_bls12381_g2_msm_affine(eng_->ctx(), n, sb.data(), pb.data(), r.aff_.data()));
    return r;
  }
 private:
  std::shared_ptr<Engine> eng_;
};

using GroupG1 = GroupImpl<G1Elt, 96, 48, true>;
using GroupG2 = GroupImpl<G2Elt, 192, 96, false>;

// pairing.Suite (pairing/pairing.go:8-20) for BLS12-381 on the GPU engine, shaped like kilic.Suite
class Suite {
 public:
  explicit Suite(int device = 0) : eng_(std::make_shared<Engine>(device)), g1_(eng_), g2_(eng_), gt_(eng_) {}
  const GroupG1& G1() const { return g1_; }
  const GroupG2& G2() const { return g2_; }
  const GroupGT& GT() const { return gt_; }
  std::string String() const { return "bls12-381.b200"; }
  // Pair(p1, p2): p1 in G1, p2 in G2 (kilic/suite.go:70-75)
  GTElt Pair(const Point& p1, const Point& p2) const {
    GTElt r(eng_);
    eng_->check(b2k_bls12381_pair(eng_->ctx(), 1, G1Elt::cast(p1).aff_.data(), G2Elt::cast(p2).aff_.data(), r.bytes.data()));
    return r;
  }
  // ValidatePairing(p1, p2, inv1, inv2): e(p1,p2) == e(inv1,inv2) (kilic/suite.go:57-68)
  bool ValidatePairing(const Point& p1, const Point& p2, const Point& inv1, const Point& inv2) const {
    uint8_t ok = 0;
    eng_->check(b2k_bls12381_pairing_check(eng_->ctx(), 1, G1Elt::cast(p1).aff_.data(), G2Elt::cast(p2).aff_.data(),
                                           G1Elt::cast(inv1).aff_.data(), G2Elt::cast(inv2).aff_.data(), &ok));
    return ok != 0;
  }
  // batch extension
  std::vector<bool> ValidatePairingBatch(const std::vector<G1Elt>& p1, const std::vector<G2Elt>& p2,
                                         const std::vector<G1Elt>& i1, const std::vector<G2Elt>& i2) const {
    size_t n = p1.size();
    Bytes a1(96 * n), a2(192 * n), b1(96 * n), b2(192 * n), ok(n);
    for (size_t i = 0; i < n; i++) {
      std::memcpy(&a1[96 * i], p1[i].aff_.data(), 96); std::memcpy(&a2[192 * i], p2[i].aff_.data(), 192);
      std::memcpy(&b1[96 * i], i1[i].aff_.data(), 96); std::memcpy(&b2[192 * i], i2[i].aff_.data(), 192);
    }
    eng_->check(b2k_bls12381_pairing_check(eng_->ctx(), n, a1.data(), a2.data(), b1.data(), b2.data(), ok.data()));
    return std::vector<bool>(ok.begin(), ok.end());
  }
  // prod_i e(g1[i], g2[i]) == 1: n Miller loops, ONE final exponentiation (what pointGT.Miller / Finalize are exported for,
  // pairing/bn254/point.go:768-786)
  bool PairingProductIsOne(const std::vector<G1Elt>& g1, const std::vector<G2Elt>& g2) const {
    size_t n = g1.size();
    if (g2.size() != n) throw std::logic_error("PairingProductIsOne: length mismatch");
    if (n == 0) return true;
    Bytes a(96 * n), b(192 * n);
    for (size_t i = 0; i < n; i++) { std::memcpy(&a[96 * i], g1[i].aff_.data(), 96); std::memcpy(&b[192 * i], g2[i].aff_.data(), 192); }
    uint8_t ok = 0;
    eng_->check(b2k_bls12381_pairing_product_check(eng_->ctx(), n, a.data(), b.data(), &ok));
    return ok != 0;
  }
  // Miller / Finalize: Finalize(Miller(p, q)) == Pair(p, q); several Miller values may be multiplied (GTElt::Add) first
  GTElt Miller(const Point& p1, const Point& p2) const {
    GTElt r(eng_);
    eng_->check(b2k_bls12381_miller(eng_->ctx(), 1, G1Elt::cast(p1).aff_.data(), G2Elt::cast(p2).aff_.data(), r.bytes.data()));
    return r;
  }
  GTElt Finalize(const GTElt& f) const {
    GTElt r(eng_);
    Bytes x = f.bytes;
    eng_->check(b2k_bls12381_final_exp(eng_->ctx(), 1, x.data(), r.bytes.data()));
    return r;
  }
  std::shared_ptr<Engine> engine() const { return eng_; }
 private:
  std::shared_ptr<Engine> eng_;
  GroupG1 g1_;
  GroupG2 g2_;
  GroupGT gt_;
};

// ---- group/edwards25519 on the engine: Point.Mul and its batch form (group/edwards25519/point.go:235-258) --------------------
// Points travel as their 32-byte compressed encodings (ge.go:99-150), scalars as 32 raw little-endian bytes (scalar.go:187-189).
namespace ed25519 {
using PointBytes = std::array<uint8_t, 32>;
static const PointBytes BASE = {0x58, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66,
                                0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66, 0x66};
class Curve {
 public:
  explicit Curve(std::shared_ptr<Engine> e) : eng_(std::move(e)) {}
  std::string String() const { return "Ed25519"; }                 // group/edwards25519/curve.go:18-20
  int ScalarLen() const { return 32; }
  int PointLen() const { return 32; }
  // out[i] = s[i] * A[i]  (n x Point.Mul; BASELINE.json configs[0])
  std::vector<PointBytes> MulBatch(const std::vector<PointBytes>& s, const std::vector<PointBytes>& A) const {
    size_t n = s.size();
    if (A.size() != n) throw std::logic_error("MulBatch: length mismatch");
    std::vector<PointBytes> out(n);
    if (n == 0) return out;
    eng_->check(b2k_ed25519_mul_batch(eng_->ctx(), n, s[0].data(), A[0].data(), out[0].data()));
    return out;
  }
  PointBytes Mul(const PointBytes& s, const PointBytes* A) const { return MulBatch({s}, {A ? *A : BASE})[0]; }   // nil = base point
  // status[i] = 0 iff eddsa.VerifyWithChecks(pks[i], msgs[i], sigs[i]) == nil (sign/eddsa/eddsa.go:149-229), else the
  // B2K_ED_* code of the first check that fails.  Signatures are R || s; a signature of another length is the caller's
  // ErrSignatureLength.
  std::vector<uint8_t> VerifyBatch(const std::vector<PointBytes>& pks, const std::vector<std::vector<uint8_t>>& msgs,
                                   const std::vector<std::array<uint8_t, 64>>& sigs) const {
    size_t n = pks.size();
    if (msgs.size() != n || sigs.size() != n) throw std::logic_error("VerifyBatch: length mismatch");
    std::vector<uint8_t> status(n);
    if (n == 0) return status;
    std::vector<uint32_t> offs(n + 1, 0);
    std::vector<uint8_t> blob;
    for (size_t i = 0; i < n; i++) {
      blob.insert(blob.end(), msgs[i].begin(), msgs[i].end());
      offs[i + 1] = (uint32_t)blob.size();
    }
    if (blob.empty()) blob.push_back(0);
    eng_->check(b2k_ed25519_verify(eng_->ctx(), n, pks[0].data(), blob.data(), offs.data(), sigs[0].data(), status.data()));
    return status;
  }
 private:
  std::shared_ptr<Engine> eng_;
};
}  // namespace ed25519

// ---- one process driving several GPUs: the sharded MSM of BASELINE.json configs[4] (b2k_bls12381_g1_msm_multi_gpu) -------------
class MultiGPU {
 public:
  explicit MultiGPU(int ngpu) {
    for (int g = 0; g < ngpu; g++) {
      b2k_ctx* c = nullptr;
      if (b2k_create(g, &c) != 0) { close(); throw std::runtime_error("b2kyber: device unavailable"); }
      ctxs_.push_back(c);
      b2k_comm* cm = nullptr;
      if (b2k_comm_create(c, ngpu, g, &cm) != 0) { close(); throw std::runtime_error(std::string("b2kyber: ") + b2k_last_error(c)); }
      comms_.push_back(cm);
    }
    if (b2k_comm_connect_local(comms_.data(), ngpu) != 0) { close(); throw std::runtime_error("b2kyber: peer access between the devices is not available"); }
  }
  ~MultiGPU() { close(); }
  MultiGPU(const MultiGPU&) = delete;
  // 48-byte compressed sum of s[i] * p[i] over all devices
  Bytes MSM(const Bytes& scalars, const Bytes& points) const {
    size_t n = scalars.size() / 32;
    Bytes out(48);
    int rc = b2k_bls12381_g1_msm_multi_gpu(const_cast<b2k_comm**>(comms_.data()), (int)comms_.size(), n, scalars.data(), points.data(), out.data());
    if (rc != 0) throw std::logic_error(std::string("b2kyber: ") + b2k_last_error(ctxs_[0]));
    return out;
  }
 private:
  void close() {
    for (auto* c : comms_) b2k_comm_destroy(c);
    for (auto* c : ctxs_) b2k_destroy(c);
    comms_.clear(); ctxs_.clear();
  }
  std::vector<b2k_ctx*> ctxs_;
  std::vector<b2k_comm*> comms_;
};

// sign/bls scheme on G1 (sign/bls/bls.go:33-44): Sign = x * H(m), Verify = ValidatePairing(H(m), X, sig, G2 base)
class SchemeOnG1 {
 public:
  explicit SchemeOnG1(const Suite& s) : s_(s) {}
  Bytes Sign(const Scalar& x, const Bytes& msg) const {
    G1Elt hm(s_.engine());
    hm.Hash(msg);
    hm.Mul(x, &hm);                                  // aliasing receiver == argument, as bls.go:73
    return hm.MarshalBinary();
  }
  // returns true where Go returns nil, false where it returns an error (bls.go:82-96)
  bool Verify(const Point& X, const Bytes& msg, const Bytes& sig) const {
    G1Elt hm(s_.engine()), sg(s_.engine());
    hm.Hash(msg);
    try { sg.UnmarshalBinary(sig); } catch (const std::runtime_error&) { return false; }
    G2Elt base(s_.engine());
    base.Base();
    return s_.ValidatePairing(hm, X, sg, base);
  }
 private:
  const Suite& s_;
};

// ---- sign/bdn on the engine (signatures on G1, public keys on G2: bdn.NewSchemeOnG1, sign/bdn/bdn.go:74-87) -------------
namespace bdn {

// bdn.Mask (sign/bdn/mask.go:13-140), the participation bitmask over a roster, plus the rogue-key factors c_i + 1 of every
// roster member (hashPointToR, bdn.go:29-63, through b2k_bdn_coefficients).  The reference precomputes the terms
// (c_i + 1) * PK_i with a Mul+Add loop at construction (mask.go:57-61); here they are folded into the one MSM of
// AggregatePublicKeys.
class Mask {
 public:
  Mask(const Suite& suite, std::vector<G2Elt> publics) : publics_(std::move(publics)), mask_((publics_.size() + 7) / 8, 0) {
    (void)suite;
    const size_t n = publics_.size();
    Bytes blob(96 * n), fac(32 * n);
    for (size_t i = 0; i < n; i++) { Bytes b = publics_[i].MarshalBinary(); std::memcpy(&blob[96 * i], b.data(), 96); }
    if (b2k_bdn_coefficients(n, blob.data(), 96, 1, fac.data()) != B2K_OK) throw std::runtime_error("bdn: failed to hash public keys");
    factors_.resize(n);
    for (size_t i = 0; i < n; i++) factors_[i].UnmarshalBinary(Bytes(fac.begin() + 32 * i, fac.begin() + 32 * (i + 1)));
  }
  int Len() const { return (int)mask_.size(); }
  Bytes MaskBytes() const { return mask_; }
  void SetMask(const Bytes& m) { if (m.size() != mask_.size()) throw std::runtime_error("mismatching mask lengths"); mask_ = m; }
  bool GetBit(int i) const { range(i); return (mask_[i / 8] >> (i & 7)) & 1; }
  void SetBit(int i, bool enable) {
    range(i);
    if (enable) mask_[i / 8] |= (uint8_t)(1u << (i & 7)); else mask_[i / 8] &= (uint8_t)~(1u << (i & 7));
  }
  int CountEnabled() const { int c = 0; for (size_t i = 0; i < publics_.size(); i++) c += GetBit((int)i); return c; }
  int CountTotal() const { return (int)publics_.size(); }
  const std::vector<G2Elt>& Publics() const { return publics_; }
  const std::vector<Scalar>& Factors() const { return factors_; }       // c_i + 1
 private:
  void range(int i) const { if (i < 0 || (size_t)i >= publics_.size()) throw std::runtime_error("index out of range"); }
  std::vector<G2Elt> publics_;
  std::vector<Scalar> factors_;
  Bytes mask_;
};

class SchemeOnG1 {
 public:
  explicit SchemeOnG1(const Suite& s) : s_(s), bls_(s) {}
  Bytes Sign(const Scalar& x, const Bytes& msg) const { return bls_.Sign(x, msg); }
  bool Verify(const Point& X, const Bytes& msg, const Bytes& sig) const { return bls_.Verify(X, msg, sig); }
  // sum over the enabled signers of (c_i + 1) * S_i, signatures given in roster order of the enabled bits (bdn.go:126-161);
  // a count mismatch or an undecodable signature is an error, as in Go.
  G1Elt AggregateSignatures(const std::vector<Bytes>& sigs, const Mask& mask) const {
    std::vector<Scalar> f;
    std::vector<G1Elt> pts;
    size_t k = 0;
    for (int i = 0; i < mask.CountTotal(); i++) {
      if (!mask.GetBit(i)) continue;
      if (k >= sigs.size()) throw std::runtime_error("length of signatures and public keys must match");
      G1Elt sg(s_.engine());
      sg.UnmarshalBinary(sigs[k++]);
      f.push_back(mask.Factors()[i]);
      pts.push_back(sg);
    }
    if (k != sigs.size()) throw std::runtime_error("length of signatures and public keys must match");
    if (pts.empty()) { G1Elt z(s_.engine()); z.Null(); return z; }
    return s_.G1().MSM(f, pts);
  }
  // sum over the enabled signers of (c_i + 1) * PK_i (bdn.go:166-181 with the terms of mask.go:57-61)
  G2Elt AggregatePublicKeys(const Mask& mask) const {
    std::vector<Scalar> f;
    std::vector<G2Elt> pts;
    for (int i = 0; i < mask.CountTotal(); i++) {
      if (!mask.GetBit(i)) continue;
      f.push_back(mask.Factors()[i]);
      pts.push_back(mask.Publics()[i]);
    }
    if (pts.empty()) { G2Elt z(s_.engine()); z.Null(); return z; }
    return s_.G2().MSM(f, pts);
  }
 private:
  const Suite& s_;
  b200::SchemeOnG1 bls_;
};

}  // namespace bdn

// ---- share (share/poly.go) on the engine, over BLS12-381 G1 (the group drand keeps its distributed key in) ----------------
namespace share {

struct PriShare { uint32_t I; Scalar V; };       // share/poly.go:29-32
struct PubShare { uint32_t I; G1Elt V; };        // share/poly.go:299-302

// share.PubPoly (poly.go:304-409) with base point = the group generator: Eval is Horner over the commitments at x = i + 1
// (poly.go:340-347), Check compares it with V * B (poly.go:405-409).  EvalBatch / CheckBatch are the batch extension the
// verification loops of share/vss and share/dkg re-point to (one device call for every share of every dealer).
class PubPoly {
 public:
  PubPoly(const Suite& s, std::vector<G1Elt> commits) : s_(s), commits_(std::move(commits)) {
    if (commits_.empty()) throw std::logic_error("share: empty commitment vector");
  }
  int Threshold() const { return (int)commits_.size(); }
  const G1Elt& Commit() const { return commits_[0]; }                                     // poly.go:335-338
  PubShare Eval(uint32_t i) const { return EvalBatch({i})[0]; }
  std::vector<PubShare> EvalBatch(const std::vector<uint32_t>& idx) const {
    const size_t t = commits_.size(), n = idx.size();
    Bytes cb(96 * t), out(96 * n);
    for (size_t j = 0; j < t; j++) std::memcpy(&cb[96 * j], commits_[j].aff_.data(), 96);
    s_.engine()->check(b2k_bls12381_g1_pubpoly_eval(s_.engine()->ctx(), t, cb.data(), n, idx.data(), out.data()));
    std::vector<PubShare> r;
    for (size_t k = 0; k < n; k++) { PubShare ps{idx[k], G1Elt(s_.engine())}; std::memcpy(ps.V.aff_.data(), &out[96 * k], 96); r.push_back(ps); }
    return r;
  }
  bool Check(const PriShare& sh) const { return CheckBatch({this}, {{sh}})[0][0]; }
  // ok[d][k] = polys[d]->Check(shares[d][k]); every dealer must bring the same number of shares and the same threshold
  static std::vector<std::vector<bool>> CheckBatch(const std::vector<const PubPoly*>& polys, const std::vector<std::vector<PriShare>>& shares) {
    const size_t m = polys.size();
    if (m == 0 || shares.size() != m) throw std::logic_error("share: dealers and share lists must match");
    const size_t t = polys[0]->commits_.size(), n = shares[0].size();
    Bytes cb(96 * m * t), sb(32 * m * n), ok(m * n);
    std::vector<uint32_t> idx(m * n);
    for (size_t d = 0; d < m; d++) {
      if (polys[d]->commits_.size() != t || shares[d].size() != n) throw std::logic_error("share: ragged batch");
      for (size_t j = 0; j < t; j++) std::memcpy(&cb[96 * (d * t + j)], polys[d]->commits_[j].aff_.data(), 96);
      for (size_t k = 0; k < n; k++) { idx[d * n + k] = shares[d][k].I; Bytes b = shares[d][k].V.MarshalBinary(); std::memcpy(&sb[32 * (d * n + k)], b.data(), 32); }
    }
    const Suite& s = polys[0]->s_;
    s.engine()->check(b2k_bls12381_g1_pubpoly_check(s.engine()->ctx(), m, t, cb.data(), n, idx.data(), sb.data(), ok.data()));
    std::vector<std::vector<bool>> r(m, std::vector<bool>(n));
    for (size_t d = 0; d < m; d++) for (size_t k = 0; k < n; k++) r[d][k] = ok[d * n + k] != 0;
    return r;
  }
 private:
  const Suite& s_;
  std::vector<G1Elt> commits_;
};

// share.RecoverCommit (poly.go:449-476): the caller passes the first t shares after xyCommit's sort by index (poly.go:418-445)
inline G1Elt RecoverCommit(const Suite& s, const std::vector<PubShare>& shares) {
  const size_t t = shares.size();
  if (t == 0) throw std::runtime_error("share: not enough good public shares to reconstruct secret commitment");
  std::vector<uint32_t> idx(t);
  Bytes pb(96 * t), out(48);
  for (size_t k = 0; k < t; k++) { idx[k] = shares[k].I; std::memcpy(&pb[96 * k], shares[k].V.aff_.data(), 96); }
  s.engine()->check(b2k_bls12381_g1_recover_commit(s.engine()->ctx(), t, idx.data(), pb.data(), out.data()));
  G1Elt r(s.engine());
  r.UnmarshalBinary(out);
  return r;
}

}  // namespace share

}  // namespace b200
