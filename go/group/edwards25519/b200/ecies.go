//go:build b200

// Batch form of ECIES on edwards25519 with SHA-256 (encrypt/ecies/ecies.go:23-112), the Pedersen DKG's share encryption:
//   ECIESDecryptBatch   ecies.Decrypt(suite, private, ctxts[i], sha256.New) for many ciphertexts under one key
//                       (ProcessDeals, share/dkg/pedersen/dkg.go:470-494; b2k_ed25519_ecies_decrypt)
//   ECIESEncryptBatch   ecies.Encrypt(suite, publics[i], msgs[i], sha256.New) (Deals, dkg.go:364-385; b2k_ed25519_ecies_encrypt)
// The device path is constant time in the key, r, the derived keys and the plaintext.  Elements are grouped by length, one
// device call per length; lengths above B2K_ECIES_MAX_LEN go to the reference.  UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"crypto/sha256"
	"errors"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/encrypt/ecies"
	"go.dedis.ch/kyber/v4/group/edwards25519"
	"go.dedis.ch/kyber/v4/util/random"
)

var (
	errInvalidECIES = errors.New("invalid ecies cipher")
	errOpen         = errors.New("cipher: message authentication failed")
	eciesSuite      = edwards25519.NewBlakeSHA256Ed25519()
)

// ECIESDecryptBatch returns, for every ciphertext, what ecies.Decrypt returns: the message, or nil and the reference's error
// ("invalid ecies cipher" below 32 bytes, "invalid Ed25519 curve point" for an R that does not decode,
// "cipher: message authentication failed" for a body shorter than a tag or a tag that does not match), checked in the
// reference's order: the length, then R, then the tag.  Ciphertexts of 32 to 47 bytes never reach the device: R is decoded
// here, and a body shorter than a tag fails Open.
func ECIESDecryptBatch(private kyber.Scalar, ctxts [][]byte) ([][]byte, []error) {
	n := len(ctxts)
	msgs, errs := make([][]byte, n), make([]error, n)
	priv, err := private.MarshalBinary()
	if err != nil {
		panic("b200: ECIESDecryptBatch: " + err.Error())
	}
	groups := map[int][]int{} // body length (incl. tag) -> indices
	for i, c := range ctxts {
		switch {
		case len(c) < 32:
			errs[i] = errInvalidECIES
		case len(c) < 48:
			if err := eciesSuite.Point().UnmarshalBinary(c[:32]); err != nil {
				errs[i] = err
			} else {
				errs[i] = errOpen
			}
		case len(c)-32 > int(C.B2K_ECIES_MAX_LEN)+16:
			msgs[i], errs[i] = ecies.Decrypt(eciesSuite, private, c, sha256.New)
		default:
			groups[len(c)-32] = append(groups[len(c)-32], i)
		}
	}
	for ln, idx := range groups {
		k := len(idx)
		cb, mb, st := make([]byte, 0, k*(32+ln)), make([]byte, k*(ln-16)+1), make([]byte, k)
		for _, i := range idx {
			cb = append(cb, ctxts[i]...)
		}
		run(func(c *C.b2k_ctx) C.int {
			return C.b2k_ed25519_ecies_decrypt(c, ptr(priv), C.size_t(k), C.size_t(ln), ptr(cb), ptr(mb), ptr(st))
		})
		for q, i := range idx {
			switch st[q] {
			case C.B2K_ECIES_OK:
				msgs[i] = append([]byte{}, mb[q*(ln-16):(q+1)*(ln-16)]...)
			case C.B2K_ECIES_POINT:
				errs[i] = errInvalidPoint
			case C.B2K_ECIES_AUTH:
				errs[i] = errOpen
			}
		}
		for j := range mb {
			mb[j] = 0
		}
	}
	return msgs, errs
}

// ECIESEncryptBatch returns ecies.Encrypt(suite, publics[i], msgs[i], sha256.New) for every i: R || ciphertext || tag, with
// a fresh r = suite.Scalar().Pick(random.New()) per message.
func ECIESEncryptBatch(publics []kyber.Point, msgs [][]byte) ([][]byte, error) {
	n := len(msgs)
	if len(publics) != n {
		panic("b200: ECIESEncryptBatch: publics and msgs must have the same length")
	}
	out := make([][]byte, n)
	groups := map[int][]int{}
	for i, m := range msgs {
		if len(m) > int(C.B2K_ECIES_MAX_LEN) {
			c, err := ecies.Encrypt(eciesSuite, un(publics[i]), m, sha256.New)
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
		pb, rb := make([]byte, 0, 32*k), make([]byte, 0, 32*k)
		mb, cb, st := make([]byte, 0, k*ln+1), make([]byte, k*(ln+48)), make([]byte, k)
		for _, i := range idx {
			p, err := un(publics[i]).MarshalBinary()
			if err != nil {
				return nil, err
			}
			r, err := eciesSuite.Scalar().Pick(rnd).MarshalBinary()
			if err != nil {
				return nil, err
			}
			pb, rb, mb = append(pb, p...), append(rb, r...), append(mb, msgs[i]...)
		}
		if len(mb) == 0 {
			mb = append(mb, 0)
		}
		run(func(c *C.b2k_ctx) C.int {
			return C.b2k_ed25519_ecies_encrypt(c, C.size_t(k), ptr(pb), ptr(rb), C.size_t(ln), ptr(mb), ptr(cb), ptr(st))
		})
		for j := range rb {
			rb[j] = 0
		}
		for j := range mb {
			mb[j] = 0
		}
		for q, i := range idx {
			if st[q] != C.B2K_ECIES_OK {
				return nil, errInvalidPoint // a kyber.Point always encodes to a decodable point: not reached
			}
			out[i] = append([]byte{}, cb[q*(ln+48):(q+1)*(ln+48)]...)
		}
	}
	return out, nil
}
