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
)

// sign/bdn for the verifier's workload: many aggregate signatures over one roster, each with its own participation mask.
// BDNTerms caches NewMask's terms (c_i + 1) PK_i (sign/bdn/mask.go:34-64) once per roster; AggregatePublicKeysBatch is
// AggregatePublicKeys (bdn.go:166-181) for every mask and VerifyBatch is bls.Verify (sign/bls/bls.go:82-96) under each of them,
// each one call to the device.  Masks are Mask.Mask() bytes, (n + 7) / 8 each; the sign.Policy check stays with the caller.

// BDNRoster holds the terms of one roster for one scheme: keys on G2 (bdn.NewSchemeOnG1) or keys on G1 (bdn.NewSchemeOnG2).
type BDNRoster struct {
	n       int
	keysG2  bool
	terms   []byte
	operand int
}

var (
	errBDNSig     = errors.New("bls: unmarshalling signature point")
	errBDNInvalid = errors.New("bls: invalid signature")
)

// BDNTerms computes the roster's terms.  Every key must be a *G2Elt (keys on G2) or every key a *G1Elt (keys on G1).
func BDNTerms(publics []kyber.Point) (*BDNRoster, error) {
	n := len(publics)
	if n == 0 {
		return nil, errors.New("b200: empty roster")
	}
	_, keysG2 := publics[0].(*G2Elt)
	wire, operand := 48, 96
	if keysG2 {
		wire, operand = 96, 192
	}
	pubs := make([]byte, wire*n)
	for i, p := range publics {
		b := marshal(p)
		if len(b) != wire {
			return nil, fmt.Errorf("b200: key %d is not on the roster's group", i)
		}
		copy(pubs[wire*i:], b)
	}
	r := &BDNRoster{n: n, keysG2: keysG2, terms: make([]byte, operand*n), operand: operand}
	var rc C.int
	with(func(e *engine) {
		if keysG2 {
			rc = C.b2k_bls12381_g2_bdn_terms(e.ctx, C.size_t(n), ptr(pubs), ptr(r.terms))
		} else {
			rc = C.b2k_bls12381_g1_bdn_terms(e.ctx, C.size_t(n), ptr(pubs), ptr(r.terms))
		}
	})
	if rc == C.B2K_ERR_POINT {
		return nil, errors.New("b200: a roster key does not decode")
	}
	if rc != 0 {
		return nil, fmt.Errorf("b200: bdn terms failed (%d)", int(rc))
	}
	return r, nil
}

func (r *BDNRoster) packMasks(masks [][]byte) ([]byte, error) {
	stride := (r.n + 7) / 8
	mb := make([]byte, stride*len(masks))
	for k, m := range masks {
		if len(m) != stride {
			return nil, fmt.Errorf("b200: mask %d has %d bytes, the roster needs %d", k, len(m), stride)
		}
		copy(mb[stride*k:], m)
	}
	return mb, nil
}

// AggregatePublicKeysBatch returns AggregatePublicKeys for every mask: *G2Elt or *G1Elt like the roster's keys.
func AggregatePublicKeysBatch(r *BDNRoster, masks [][]byte) ([]kyber.Point, error) {
	m := len(masks)
	if m == 0 {
		return nil, nil
	}
	mb, err := r.packMasks(masks)
	if err != nil {
		return nil, err
	}
	out := make([]byte, r.operand*m)
	with(func(e *engine) {
		if r.keysG2 {
			e.check(C.b2k_bls12381_g2_bdn_aggregate_keys(e.ctx, C.size_t(r.n), ptr(r.terms), C.size_t(m), ptr(mb), ptr(out)))
		} else {
			e.check(C.b2k_bls12381_g1_bdn_aggregate_keys(e.ctx, C.size_t(r.n), ptr(r.terms), C.size_t(m), ptr(mb), ptr(out)))
		}
	})
	keys := make([]kyber.Point, m)
	for k := range keys {
		if r.keysG2 {
			p := &G2Elt{}
			copy(p.aff[:], out[192*k:])
			keys[k] = p
		} else {
			p := &G1Elt{}
			copy(p.aff[:], out[96*k:])
			keys[k] = p
		}
	}
	return keys, nil
}

// VerifyBatch is bls.Verify(aggregate key of masks[k], msgs[k], sigs[k]) for every k, with the default domain separation tag of
// the signature group; errs[k] is nil or the reference's error.  A signature of the wrong length does not unmarshal either.
func VerifyBatch(r *BDNRoster, masks [][]byte, msgs [][]byte, sigs [][]byte) ([]error, error) {
	m := len(masks)
	if len(msgs) != m || len(sigs) != m {
		return nil, errors.New("b200: masks, messages and signatures differ in number")
	}
	if m == 0 {
		return nil, nil
	}
	mb, err := r.packMasks(masks)
	if err != nil {
		return nil, err
	}
	sigLen, dst := 48, domainG1 // keys on G2: signatures on G1
	if !r.keysG2 {
		sigLen, dst = 96, domainG2
	}
	sb := make([]byte, sigLen*m)
	offs := make([]C.uint32_t, m+1)
	var blob []byte
	for k := range sigs {
		if len(sigs[k]) == sigLen {
			copy(sb[sigLen*k:], sigs[k])
		} else {
			for j := 0; j < sigLen; j++ {
				sb[sigLen*k+j] = 0xff // no valid encoding: the device reports B2K_BDN_SIG
			}
		}
		blob = append(blob, msgs[k]...)
		offs[k+1] = C.uint32_t(len(blob))
	}
	if len(blob) == 0 {
		blob = []byte{0}
	}
	status := make([]byte, m)
	with(func(e *engine) {
		if r.keysG2 {
			e.check(C.b2k_bls12381_bdn_verify_g1sig(e.ctx, C.size_t(r.n), ptr(r.terms), C.size_t(m), ptr(mb), ptr(blob), &offs[0],
				ptr(dst), C.uint32_t(len(dst)), ptr(sb), ptr(status)))
		} else {
			e.check(C.b2k_bls12381_bdn_verify_g2sig(e.ctx, C.size_t(r.n), ptr(r.terms), C.size_t(m), ptr(mb), ptr(blob), &offs[0],
				ptr(dst), C.uint32_t(len(dst)), ptr(sb), ptr(status)))
		}
	})
	errs := make([]error, m)
	for k, st := range status {
		switch st {
		case C.B2K_BDN_OK:
		case C.B2K_BDN_SIG:
			errs[k] = errBDNSig
		default:
			errs[k] = errBDNInvalid
		}
	}
	return errs, nil
}
