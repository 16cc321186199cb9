//go:build b200

package b200

/*
#include <b2kyber.h>
*/
import "C"

import (
	"crypto/sha256"
	"errors"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/encrypt/ecies"
	"go.dedis.ch/kyber/v4/util/random"
)

// Batch form of ECIES on BLS12-381 with keys on G1 or on G2 and SHA-256 (encrypt/ecies/ecies.go:23-131), the Pedersen DKG's
// share encryption when its key group is BLS12-381:
//   ECIESDecryptBatch   ecies.Decrypt(g, private, ctxts[i], sha256.New) for many ciphertexts under one key
//                       (ProcessDeals, share/dkg/pedersen/dkg.go:478; b2k_bls12381_g{1,2}_ecies_decrypt)
//   ECIESEncryptBatch   ecies.Encrypt(g, publics[i], msgs[i], sha256.New) (Deals, dkg.go:377; b2k_bls12381_g{1,2}_ecies_encrypt)
// g is the suite's G1 or G2.  The device path is constant time in the key, r, dh, the derived keys and the plaintext.  Elements
// are grouped by length, one device call per length; lengths above B2K_ECIES_MAX_LEN go to the reference.

var (
	errECIESInvalid = errors.New("invalid ecies cipher")
	errECIESOpen    = errors.New("cipher: message authentication failed")
)

func eciesPointLen(g kyber.Group, who string) int {
	pl := g.PointLen()
	if pl != 48 && pl != 96 {
		panic("b200: " + who + ": g must be the G1 or the G2 of BLS12-381")
	}
	return pl
}

// ECIESDecryptBatch returns, for every ciphertext, what ecies.Decrypt(g, private, ctxts[i], sha256.New) returns: the message,
// or nil and the reference's error, checked in the reference's order: "invalid ecies cipher" below g.PointLen() bytes, then
// R's UnmarshalBinary error (kilic's own text: the reference's UnmarshalBinary is run here on the R the device refused), then
// "cipher: message authentication failed" for a body shorter than a tag or a tag that does not match.  Ciphertexts shorter
// than a point and a tag never reach the device: R is decoded here, and the short body fails Open.
func ECIESDecryptBatch(g kyber.Group, private kyber.Scalar, ctxts [][]byte) ([][]byte, []error) {
	pl := eciesPointLen(g, "ECIESDecryptBatch")
	n := len(ctxts)
	msgs, errs := make([][]byte, n), make([]error, n)
	priv, err := private.MarshalBinary()
	if err != nil {
		panic("b200: ECIESDecryptBatch: " + err.Error())
	}
	groups := map[int][]int{} // body length (incl. tag) -> indices
	for i, c := range ctxts {
		switch {
		case len(c) < pl:
			errs[i] = errECIESInvalid
		case len(c) < pl+16:
			if err := g.Point().UnmarshalBinary(c[:pl]); err != nil {
				errs[i] = err
			} else {
				errs[i] = errECIESOpen
			}
		case len(c)-pl > int(C.B2K_ECIES_MAX_LEN)+16:
			msgs[i], errs[i] = ecies.Decrypt(g, private, c, sha256.New)
		default:
			groups[len(c)-pl] = append(groups[len(c)-pl], i)
		}
	}
	for ln, idx := range groups {
		k := len(idx)
		cb, mb, st := make([]byte, 0, k*(pl+ln)), make([]byte, k*(ln-16)+1), make([]byte, k)
		for _, i := range idx {
			cb = append(cb, ctxts[i]...)
		}
		with(func(e *engine) {
			if pl == 48 {
				e.check(C.b2k_bls12381_g1_ecies_decrypt(e.ctx, ptr(priv), C.size_t(k), C.size_t(ln), ptr(cb), ptr(mb), ptr(st)))
			} else {
				e.check(C.b2k_bls12381_g2_ecies_decrypt(e.ctx, ptr(priv), C.size_t(k), C.size_t(ln), ptr(cb), ptr(mb), ptr(st)))
			}
		})
		for q, i := range idx {
			switch st[q] {
			case C.B2K_ECIES_OK:
				msgs[i] = append([]byte{}, mb[q*(ln-16):(q+1)*(ln-16)]...)
			case C.B2K_ECIES_POINT:
				errs[i] = g.Point().UnmarshalBinary(ctxts[i][:pl])
				if errs[i] == nil {
					panic("b200: the device refused an R the reference accepts")
				}
			case C.B2K_ECIES_AUTH:
				errs[i] = errECIESOpen
			}
		}
		for j := range mb {
			mb[j] = 0
		}
	}
	for j := range priv {
		priv[j] = 0
	}
	return msgs, errs
}

// ECIESEncryptBatch returns ecies.Encrypt(g, publics[i], msgs[i], sha256.New) for every i: R || ciphertext || tag, with a
// fresh r = g.Scalar().Pick(random.New()) per message, picked here as the reference picks it.
func ECIESEncryptBatch(g kyber.Group, publics []kyber.Point, msgs [][]byte) ([][]byte, error) {
	pl := eciesPointLen(g, "ECIESEncryptBatch")
	n := len(msgs)
	if len(publics) != n {
		panic("b200: ECIESEncryptBatch: publics and msgs must have the same length")
	}
	out := make([][]byte, n)
	groups := map[int][]int{}
	for i, m := range msgs {
		if len(m) > int(C.B2K_ECIES_MAX_LEN) {
			c, err := ecies.Encrypt(g, publics[i], m, sha256.New)
			if err != nil {
				return nil, err
			}
			out[i] = c
			continue
		}
		groups[len(m)] = append(groups[len(m)], i)
	}
	rnd := random.New()
	for ln, idx := range groups {
		k := len(idx)
		pb, rb := make([]byte, 0, pl*k), make([]byte, 0, 32*k)
		mb, cb, st := make([]byte, 0, k*ln+1), make([]byte, k*(pl+ln+16)), make([]byte, k)
		for _, i := range idx {
			p, err := publics[i].MarshalBinary()
			if err != nil {
				return nil, err
			}
			r, err := g.Scalar().Pick(rnd).MarshalBinary()
			if err != nil {
				return nil, err
			}
			pb, rb, mb = append(pb, p...), append(rb, r...), append(mb, msgs[i]...)
		}
		if len(mb) == 0 {
			mb = append(mb, 0)
		}
		with(func(e *engine) {
			if pl == 48 {
				e.check(C.b2k_bls12381_g1_ecies_encrypt(e.ctx, C.size_t(k), ptr(pb), ptr(rb), C.size_t(ln), ptr(mb), ptr(cb), ptr(st)))
			} else {
				e.check(C.b2k_bls12381_g2_ecies_encrypt(e.ctx, C.size_t(k), ptr(pb), ptr(rb), C.size_t(ln), ptr(mb), ptr(cb), ptr(st)))
			}
		})
		for j := range rb {
			rb[j] = 0
		}
		for j := range mb {
			mb[j] = 0
		}
		for q, i := range idx {
			if st[q] != C.B2K_ECIES_OK {
				// a kyber.Point of the group always marshals to an encoding that decodes: not reached
				return nil, errors.New("b200: ECIESEncryptBatch: a public key did not decode")
			}
			out[i] = append([]byte{}, cb[q*(pl+ln+16):(q+1)*(pl+ln+16)]...)
		}
	}
	return out, nil
}
