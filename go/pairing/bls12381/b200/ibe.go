//go:build b200

package b200

/*
#include <b2kyber.h>
*/
import "C"

import (
	"crypto/rand"
	"errors"
	"fmt"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/encrypt/ibe"
)

// Batch forms of encrypt/ibe's CCA functions (ibe.go:51-231) for many ciphertexts under one key, or many messages to one
// identity: the case of a timelock round whose key has just been published.  Results and error strings are the reference's.

const ibeMaxLen = 32 // s.Hash().Size(), SHA-256

// ptrOrNil is ptr for buffers that may be empty (a zero-length message).
func ptrOrNil(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return ptr(b)
}

func marshal(p kyber.Point) []byte {
	b, err := p.MarshalBinary()
	if err != nil {
		panic(err)
	}
	return b
}

// DecryptCCAonG1Batch is DecryptCCAonG1 for every ciphertext (U on G1, private on G2).
func DecryptCCAonG1Batch(s *Suite, private kyber.Point, cs []*ibe.Ciphertext) ([][]byte, []error) {
	return decryptBatch(s, 1, private, cs)
}

// DecryptCCAonG2Batch is DecryptCCAonG2 for every ciphertext (U on G2, private on G1).
func DecryptCCAonG2Batch(s *Suite, private kyber.Point, cs []*ibe.Ciphertext) ([][]byte, []error) {
	return decryptBatch(s, 2, private, cs)
}

func decryptBatch(s *Suite, on int, private kyber.Point, cs []*ibe.Ciphertext) ([][]byte, []error) {
	msgs, errs := make([][]byte, len(cs)), make([]error, len(cs))
	groups := map[int][]int{} // ciphertexts by length, after the reference's host-side length checks
	for i, c := range cs {
		if len(c.W) > ibeMaxLen {
			errs[i] = errors.New("ciphertext too long for the hash function provided")
			continue
		}
		if len(c.V) != len(c.W) {
			errs[i] = fmt.Errorf("XorSigma is of invalid length: exp %d vs got %d", len(c.W), len(c.V))
			continue
		}
		groups[len(c.W)] = append(groups[len(c.W)], i)
	}
	key := marshal(private)
	ub := 48 * on
	for n, idx := range groups {
		k := len(idx)
		u, v, w := make([]byte, ub*k), make([]byte, n*k), make([]byte, n*k)
		for j, i := range idx {
			copy(u[ub*j:], marshal(cs[i].U))
			copy(v[n*j:], cs[i].V)
			copy(w[n*j:], cs[i].W)
		}
		out, status := make([]byte, n*k), make([]byte, k)
		with(func(e *engine) {
			if on == 1 {
				e.check(C.b2k_bls12381_ibe_decrypt_cca_g1(e.ctx, ptr(key), C.size_t(k), ptr(u), C.size_t(n), ptrOrNil(v), ptrOrNil(w),
					ptrOrNil(out), ptr(status)))
			} else {
				e.check(C.b2k_bls12381_ibe_decrypt_cca_g2(e.ctx, ptr(key), C.size_t(k), ptr(u), C.size_t(n), ptrOrNil(v), ptrOrNil(w),
					ptrOrNil(out), ptr(status)))
			}
		})
		for j, i := range idx {
			switch status[j] {
			case C.B2K_IBE_OK:
				msgs[i] = append([]byte{}, out[n*j:n*j+n]...)
			case C.B2K_IBE_PROOF:
				errs[i] = errors.New("invalid proof: rP check failed")
			default:
				errs[i] = errors.New("malformed point U")
			}
		}
	}
	return msgs, errs
}

// EncryptCCAonG1Batch is EncryptCCAonG1 for every message (master on G1, identity on G2, U on G1); sigma from crypto/rand.
func EncryptCCAonG1Batch(s *Suite, master kyber.Point, id []byte, msgs [][]byte) ([]*ibe.Ciphertext, error) {
	return encryptBatch(s, 1, master, id, msgs)
}

// EncryptCCAonG2Batch is EncryptCCAonG2 for every message (master on G2, identity on G1, U on G2); sigma from crypto/rand.
func EncryptCCAonG2Batch(s *Suite, master kyber.Point, id []byte, msgs [][]byte) ([]*ibe.Ciphertext, error) {
	return encryptBatch(s, 2, master, id, msgs)
}

func encryptBatch(s *Suite, on int, master kyber.Point, id []byte, msgs [][]byte) ([]*ibe.Ciphertext, error) {
	out := make([]*ibe.Ciphertext, len(msgs))
	groups := map[int][]int{}
	for i, m := range msgs {
		if len(m) > ibeMaxLen {
			return nil, errors.New("plaintext too long for the hash function provided")
		}
		groups[len(m)] = append(groups[len(m)], i)
	}
	dst := s.domainG1 // the suite's DST of the identity's hash; nil = the default
	if on == 1 {
		dst = s.domainG2
	}
	key := marshal(master)
	ub := 48 * on
	for n, idx := range groups {
		k := len(idx)
		m, sigma := make([]byte, n*k), make([]byte, n*k)
		for j, i := range idx {
			copy(m[n*j:], msgs[i])
		}
		if _, err := rand.Read(sigma); err != nil {
			return nil, fmt.Errorf("err reading rand sigma: %w", err)
		}
		u, v, w := make([]byte, ub*k), make([]byte, n*k), make([]byte, n*k)
		var rc C.int
		with(func(e *engine) {
			if on == 1 {
				rc = C.b2k_bls12381_ibe_encrypt_cca_g1(e.ctx, ptr(key), ptrOrNil(id), C.size_t(len(id)), ptrOrNil(dst), C.size_t(len(dst)),
					C.size_t(k), C.size_t(n), ptrOrNil(m), ptrOrNil(sigma), ptr(u), ptrOrNil(v), ptrOrNil(w))
			} else {
				rc = C.b2k_bls12381_ibe_encrypt_cca_g2(e.ctx, ptr(key), ptrOrNil(id), C.size_t(len(id)), ptrOrNil(dst), C.size_t(len(dst)),
					C.size_t(k), C.size_t(n), ptrOrNil(m), ptrOrNil(sigma), ptr(u), ptrOrNil(v), ptrOrNil(w))
			}
		})
		if rc != C.B2K_OK {
			return nil, fmt.Errorf("b2kyber: IBE encryption failed (%d)", int(rc))
		}
		for j, i := range idx {
			var U kyber.Point
			if on == 1 {
				U = s.G1().Point()
			} else {
				U = s.G2().Point()
			}
			if err := U.UnmarshalBinary(u[ub*j : ub*j+ub]); err != nil {
				return nil, err
			}
			out[i] = &ibe.Ciphertext{U: U, V: append([]byte{}, v[n*j:n*j+n]...), W: append([]byte{}, w[n*j:n*j+n]...)}
		}
	}
	return out, nil
}
