//go:build b200

// Batch forms of proof/dleq and share/pvss verification on edwards25519:
//   DLEQVerifyBatch        dleq.Proof.Verify (proof/dleq/dleq.go:161-172) for n proofs (b2k_ed25519_dleq_verify)
//   VerifyEncShareBatch    pvss.VerifyEncShareBatch (share/pvss/pvss.go:168-194); VerifyEncShareBatches runs m deals in one
//                          call (b2k_ed25519_pvss_verify_enc_shares)
//   VerifyDecShareBatch    pvss.VerifyDecShareBatch (pvss.go:281-299, b2k_ed25519_pvss_verify_dec_shares)
//   RecoverSecret          pvss.RecoverSecret (pvss.go:303-323): VerifyDecShareBatch, then RecoverCommit (share.go)
// The errors wrap the reference's sentinels, so errors.Is holds against pvss.Err* and dleq.Err*.  Scalars travel as their 32
// little-endian bytes, read raw as Point.Mul reads them.  UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"fmt"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/proof/dleq"
	"go.dedis.ch/kyber/v4/share"
	"go.dedis.ch/kyber/v4/share/pvss"
)

func packProof(p *dleq.Proof) []byte {
	b := make([]byte, 0, 128)
	b = append(b, packScalars([]kyber.Scalar{p.C, p.R})...)
	return append(b, packPoints([]kyber.Point{p.VG, p.VH})...)
}

func packProofs(ps []*pvss.PubVerShare) ([]byte, []kyber.Point) {
	b := make([]byte, 0, 128*len(ps))
	v := make([]kyber.Point, len(ps))
	for i, s := range ps {
		b = append(b, packProof(&s.P)...)
		v[i] = s.S.V
	}
	return b, v
}

// dleqStatusError maps a B2K_DLEQ_* status to the reference's error for that check (nil for OK)
func dleqStatusError(st byte, challengeErr, verifyErr error) error {
	switch st {
	case C.B2K_DLEQ_OK:
		return nil
	case C.B2K_DLEQ_CHALLENGE:
		return fmt.Errorf("didn't verify: %w", challengeErr)
	case C.B2K_DLEQ_INVALID:
		return fmt.Errorf("didn't verify: %w", verifyErr)
	default:
		return fmt.Errorf("didn't verify: %w: %w", verifyErr, errInvalidPoint)
	}
}

// DLEQVerifyBatch returns errs[i] = proofs[i].Verify(suite, G[i], H[i], xG[i], xH[i]) (nil when the proof holds)
func DLEQVerifyBatch(G, H, xG, xH []kyber.Point, proofs []*dleq.Proof) ([]error, error) {
	n := len(proofs)
	if len(G) != n || len(H) != n || len(xG) != n || len(xH) != n {
		return nil, fmt.Errorf("invalid: %w", dleq.ErrDifferentLengths)
	}
	errs := make([]error, n)
	if n == 0 {
		return errs, nil
	}
	pb := make([]byte, 0, 128*n)
	for _, p := range proofs {
		pb = append(pb, packProof(p)...)
	}
	gb, hb, xgb, xhb, st := packPoints(G), packPoints(H), packPoints(xG), packPoints(xH), make([]byte, n)
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_dleq_verify(c, C.size_t(n), ptr(gb), ptr(hb), ptr(xgb), ptr(xhb), ptr(pb), ptr(st))
	})
	for i := range errs {
		if st[i] != C.B2K_DLEQ_OK {
			errs[i] = fmt.Errorf("invalid. %w", dleq.ErrInvalidProof)
		}
	}
	return errs, nil
}

// EncDeal is one dealer's input to VerifyEncShareBatches
type EncDeal struct {
	H         kyber.Point
	X, SH     []kyber.Point
	Commit    *share.PubPoly
	EncShares []*pvss.PubVerShare
}

// VerifyEncShareBatches checks m deals that share one threshold and one share count in one call; errs[d][i] is the error
// pvss.VerifyEncShare would return for share i of deal d
func VerifyEncShareBatches(deals []EncDeal) ([][]error, error) {
	m := len(deals)
	if m == 0 {
		return nil, nil
	}
	_, c0 := deals[0].Commit.Info()
	t, n := len(c0), len(deals[0].X)
	var hb, cb, xb, shb, vb, pb []byte
	for _, d := range deals {
		_, cm := d.Commit.Info()
		if len(d.X) != n || len(d.SH) != n || len(d.EncShares) != n || len(cm) != t {
			return nil, fmt.Errorf("didn't verify: %w", pvss.ErrDifferentLengths)
		}
		proofs, v := packProofs(d.EncShares)
		hb = append(hb, packPoints([]kyber.Point{d.H})...)
		cb = append(cb, packPoints(cm)...)
		xb = append(xb, packPoints(d.X)...)
		shb = append(shb, packPoints(d.SH)...)
		vb = append(vb, packPoints(v)...)
		pb = append(pb, proofs...)
	}
	errs := make([][]error, m)
	if n == 0 || t == 0 {
		return errs, nil
	}
	st := make([]byte, m*n)
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_pvss_verify_enc_shares(c, C.size_t(m), C.size_t(t), C.size_t(n), ptr(hb), ptr(cb), ptr(xb), ptr(shb),
			ptr(vb), ptr(pb), ptr(st))
	})
	for d := range errs {
		errs[d] = make([]error, n)
		for i := range errs[d] {
			errs[d][i] = dleqStatusError(st[d*n+i], pvss.ErrGlobalChallengeVerification, pvss.ErrEncVerification)
		}
	}
	return errs, nil
}

// VerifyEncShareBatch is pvss.VerifyEncShareBatch: the good public keys K and encrypted shares E
func VerifyEncShareBatch(H kyber.Point, X, sH []kyber.Point, commit *share.PubPoly, encShares []*pvss.PubVerShare) (
	[]kyber.Point, []*pvss.PubVerShare, error) {
	if len(X) != len(sH) || len(sH) != len(encShares) {
		return nil, nil, fmt.Errorf("didn't verify: %w", pvss.ErrDifferentLengths)
	}
	if len(X) == 0 {
		return nil, nil, nil
	}
	errs, err := VerifyEncShareBatches([]EncDeal{{H: H, X: X, SH: sH, Commit: commit, EncShares: encShares}})
	if err != nil {
		return nil, nil, err
	}
	var K []kyber.Point
	var E []*pvss.PubVerShare
	for i, e := range errs[0] {
		if e == nil {
			K = append(K, X[i])
			E = append(E, encShares[i])
		}
	}
	return K, E, nil
}

// verifyDec returns the VerifyDecShare error of every share
func verifyDec(G kyber.Point, X []kyber.Point, encShares, decShares []*pvss.PubVerShare) ([]error, error) {
	n := len(X)
	if len(encShares) != n || len(decShares) != n {
		return nil, fmt.Errorf("didn't verify: %w", pvss.ErrDifferentLengths)
	}
	errs := make([]error, n)
	if n == 0 {
		return errs, nil
	}
	_, ev := packProofs(encShares)
	pb, dv := packProofs(decShares)
	gb, xb, eb, db, st := packPoints([]kyber.Point{G}), packPoints(X), packPoints(ev), packPoints(dv), make([]byte, n)
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_pvss_verify_dec_shares(c, C.size_t(n), ptr(gb), ptr(xb), ptr(eb), ptr(db), ptr(pb), ptr(st))
	})
	for i := range errs {
		errs[i] = dleqStatusError(st[i], pvss.ErrDecShareChallengeVerification, pvss.ErrDecVerification)
	}
	return errs, nil
}

// VerifyDecShareBatch is pvss.VerifyDecShareBatch: the good decrypted shares
func VerifyDecShareBatch(G kyber.Point, X []kyber.Point, encShares, decShares []*pvss.PubVerShare) ([]*pvss.PubVerShare, error) {
	errs, err := verifyDec(G, X, encShares, decShares)
	if err != nil {
		return nil, err
	}
	var D []*pvss.PubVerShare
	for i, e := range errs {
		if e == nil {
			D = append(D, decShares[i])
		}
	}
	return D, nil
}

// RecoverSecret is pvss.RecoverSecret: the valid decrypted shares, then RecoverCommit over them (xyCommit's selection)
func RecoverSecret(G kyber.Point, X []kyber.Point, encShares, decShares []*pvss.PubVerShare, t, n uint32) (kyber.Point, error) {
	D, err := VerifyDecShareBatch(G, X, encShares, decShares)
	if err != nil {
		return nil, err
	}
	if uint32(len(D)) < t {
		return nil, fmt.Errorf("didn't verify: %w", pvss.ErrTooFewShares)
	}
	shares := make([]*share.PubShare, len(D))
	for i, s := range D {
		shares[i] = &s.S
	}
	return RecoverCommit(shares, t, n)
}
