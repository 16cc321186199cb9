//go:build b200

package b200

/*
#include <b2kyber.h>
*/
import "C"

import (
	"errors"
	"fmt"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/sign/schnorr"
)

// sign/schnorr over BLS12-381 keys on G1 or on G2: schnorr.VerifyWithChecks (sign/schnorr/schnorr.go:89-183) for every
// signature of a batch in one device call (b2k_bls12381_g{1,2}_schnorr_verify), e.g. the packet signatures of a DKG phase
// (dkg.VerifyPacketSignature, share/dkg/pedersen/structs.go:293-348).  errs[i] is nil or the reference's error.

var (
	errSchnorrPK      = errors.New("schnorr: error unmarshalling public key")
	errSchnorrInvalid = errors.New("schnorr: invalid signature")
)

// SchnorrVerifyWithChecksBatch returns errs[i] = schnorr.VerifyWithChecks(g, pubs[i], msgs[i], sigs[i]) for every i; g is the
// suite's G1 (keys on G1, 80-byte signatures) or G2 (keys on G2, 128-byte signatures).  A signature of the wrong length gets
// the reference's length error on the host.  A key of the wrong length travels as zero bytes (compression flag clear), which
// does not decode: it fails with "error unmarshalling public key" after the signature's own checks, as in the reference.
// For a signature whose R or s does not decode, the reference itself is run on the host for that signature: it fails before
// the key is read and returns kilic's or mod.Int's exact error.
func SchnorrVerifyWithChecksBatch(g kyber.Group, pubs, msgs, sigs [][]byte) []error {
	n := len(sigs)
	if len(pubs) != n || len(msgs) != n {
		panic("b200: SchnorrVerifyWithChecksBatch: pubs, msgs and sigs must have the same length")
	}
	pl := g.PointLen()
	if pl != 48 && pl != 96 {
		panic("b200: SchnorrVerifyWithChecksBatch: g must be the G1 or the G2 of BLS12-381")
	}
	sigLen := pl + g.ScalarLen()
	errs := make([]error, n)
	idx := make([]int, 0, n) // the signatures that go to the device
	for i := range sigs {
		if len(sigs[i]) != sigLen {
			errs[i] = fmt.Errorf("schnorr: signature of invalid length %d instead of %d", len(sigs[i]), sigLen)
			continue
		}
		idx = append(idx, i)
	}
	m := len(idx)
	if m == 0 {
		return errs
	}
	pb, sb, st := make([]byte, pl*m), make([]byte, sigLen*m), make([]byte, m)
	offs := make([]C.uint32_t, m+1)
	var blob []byte
	for k, i := range idx {
		if len(pubs[i]) == pl {
			copy(pb[pl*k:], pubs[i])
		} // else: zeros, which do not decode
		copy(sb[sigLen*k:], sigs[i])
		blob = append(blob, msgs[i]...)
		offs[k+1] = C.uint32_t(len(blob))
	}
	if len(blob) == 0 {
		blob = []byte{0}
	}
	with(func(e *engine) {
		if pl == 48 {
			e.check(C.b2k_bls12381_g1_schnorr_verify(e.ctx, C.size_t(m), ptr(pb), ptr(blob), &offs[0], ptr(sb), ptr(st)))
		} else {
			e.check(C.b2k_bls12381_g2_schnorr_verify(e.ctx, C.size_t(m), ptr(pb), ptr(blob), &offs[0], ptr(sb), ptr(st)))
		}
	})
	for k, i := range idx {
		switch st[k] {
		case C.B2K_SCHNORR_OK:
		case C.B2K_SCHNORR_R, C.B2K_SCHNORR_S:
			errs[i] = schnorr.VerifyWithChecks(g, pubs[i], msgs[i], sigs[i])
			if errs[i] == nil {
				panic("b200: the device refused a signature the reference accepts")
			}
		case C.B2K_SCHNORR_PK:
			errs[i] = errSchnorrPK
		default:
			errs[i] = errSchnorrInvalid
		}
	}
	return errs
}

// SchnorrVerifyBatch is the batch twin of schnorr.Verify (schnorr.go:171-178): keys are marshalled first, and a key that does
// not marshal gets the reference's wrapped error.
func SchnorrVerifyBatch(g kyber.Group, pubs []kyber.Point, msgs, sigs [][]byte) []error {
	if len(pubs) != len(sigs) {
		panic("b200: SchnorrVerifyBatch: pubs, msgs and sigs must have the same length")
	}
	pb := make([][]byte, len(pubs))
	bad := make([]error, len(pubs))
	for i, p := range pubs {
		b, err := p.MarshalBinary()
		if err != nil {
			bad[i] = fmt.Errorf("error unmarshalling public key: %w", err)
		}
		pb[i] = b
	}
	errs := SchnorrVerifyWithChecksBatch(g, pb, msgs, sigs)
	for i := range errs {
		if bad[i] != nil {
			errs[i] = bad[i]
		}
	}
	return errs
}
