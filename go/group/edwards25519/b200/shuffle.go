//go:build b200

// Batch form of Neff's shuffle verification on edwards25519:
//   HashVerifyShuffles      proof.HashVerify(suite, protocolName, shuffle.Verifier(suite, G, H, X, Y, Xbar, Ybar), proof) for m
//                           shuffles of k pairs in one call (proof/hash.go:168-175, shuffle/pair.go:239-312, shuffle/simple.go:186-254;
//                           b2k_ed25519_shuffle_verify)
//   GetSequenceVerifiable   shuffle.GetSequenceVerifiable (shuffle/sequences.go:155-190; b2k_ed25519_shuffle_sequence_verifiable)
// The per-shuffle errors carry the reference's messages.  The suite is edwards25519.NewBlakeSHA256Ed25519: the transcript is
// blake2xb, run inside the library.  UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"errors"
	"fmt"
	"io"

	"go.dedis.ch/kyber/v4"
)

// ShuffleProof is one shuffle to check: the pairs before (X, Y) and after (Xbar, Ybar) and the bytes of proof.HashProve
type ShuffleProof struct {
	X, Y, Xbar, Ybar []kyber.Point
	Proof            []byte
}

var (
	errSimpleShuffle = errors.New("incorrect SimpleShuffleProof")
	errPairShuffle   = errors.New("invalid PairShuffleProof")
)

// HashVerifyShuffles returns errs[s] = proof.HashVerify(suite, protocolName, shuffle.Verifier(suite, G, H, X, Y, Xbar, Ybar),
// Proof) for every shuffle (nil when it holds).  G or H nil is the base point, as in shuffle.Verifier.  Every shuffle has the
// same k >= 2.  A proof shorter than 32 (12k + 3) bytes fails as the reference's Get does (io.ErrUnexpectedEOF); bytes beyond
// that length are never read, as in the reference.
func HashVerifyShuffles(protocolName string, G, H kyber.Point, shuffles []ShuffleProof) ([]error, error) {
	m := len(shuffles)
	errs := make([]error, m)
	if m == 0 {
		return errs, nil
	}
	k := len(shuffles[0].X)
	if k < 2 {
		return nil, errors.New("can't shuffle permutation of size <= 1")
	}
	plen := 32 * (12*k + 3)
	var idx []int
	var x, y, xb, yb, pb []byte
	for s, sh := range shuffles {
		if len(sh.X) != k || len(sh.Y) != k || len(sh.Xbar) != k || len(sh.Ybar) != k {
			return nil, fmt.Errorf("shuffle %d: mismatched vector lengths", s)
		}
		if len(sh.Proof) < plen {
			errs[s] = io.ErrUnexpectedEOF
			continue
		}
		idx = append(idx, s)
		x = append(x, packPoints(sh.X)...)
		y = append(y, packPoints(sh.Y)...)
		xb = append(xb, packPoints(sh.Xbar)...)
		yb = append(yb, packPoints(sh.Ybar)...)
		pb = append(pb, sh.Proof[:plen]...)
	}
	n := len(idx)
	if n == 0 {
		return errs, nil
	}
	var gb, hb []byte
	if G != nil {
		gb = packPoints(repeat(G, n))
	}
	if H != nil {
		hb = packPoints(repeat(H, n))
	}
	proto := []byte(protocolName)
	st := make([]byte, n)
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_shuffle_verify(c, C.size_t(n), C.size_t(k), optPtr(gb), optPtr(hb), ptr(x), ptr(y), ptr(xb), ptr(yb),
			ptr(pb), optPtr(proto), C.uint32_t(len(proto)), ptr(st))
	})
	for j, s := range idx {
		switch st[j] {
		case C.B2K_SHUFFLE_OK:
		case C.B2K_SHUFFLE_SIMPLE:
			errs[s] = errSimpleShuffle
		case C.B2K_SHUFFLE_PAIR:
			errs[s] = errPairShuffle
		default:
			errs[s] = errInvalidPoint
		}
	}
	return errs, nil
}

// GetSequenceVerifiable is shuffle.GetSequenceVerifiable: xUp[i] = sum_j e[j] X[j][i], and likewise yUp, xDown and yDown
func GetSequenceVerifiable(X, Y, Xbar, Ybar [][]kyber.Point, e []kyber.Scalar) (xUp, yUp, xDown, yDown []kyber.Point) {
	nq := len(X)
	if nq == 0 || len(X[0]) == 0 || len(Y) != nq || len(Xbar) != nq || len(Ybar) != nq || len(e) != nq {
		panic("b200: GetSequenceVerifiable: mismatched dimensions")
	}
	k := len(X[0])
	var x, y, xb, yb []byte
	for j := 0; j < nq; j++ {
		if len(X[j]) != k || len(Y[j]) != k || len(Xbar[j]) != k || len(Ybar[j]) != k {
			panic("b200: GetSequenceVerifiable: mismatched dimensions")
		}
		x = append(x, packPoints(X[j])...)
		y = append(y, packPoints(Y[j])...)
		xb = append(xb, packPoints(Xbar[j])...)
		yb = append(yb, packPoints(Ybar[j])...)
	}
	eb := packScalars(e)
	out := [4][]byte{make([]byte, 32*k), make([]byte, 32*k), make([]byte, 32*k), make([]byte, 32*k)}
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_shuffle_sequence_verifiable(c, C.size_t(nq), C.size_t(k), ptr(x), ptr(y), ptr(xb), ptr(yb), ptr(eb),
			ptr(out[0]), ptr(out[1]), ptr(out[2]), ptr(out[3]))
	})
	res := [4][]kyber.Point{}
	for q := range out {
		res[q] = make([]kyber.Point, k)
		for i := 0; i < k; i++ {
			res[q][i] = unpackPoint(out[q][32*i : 32*i+32])
		}
	}
	return res[0], res[1], res[2], res[3]
}

func repeat(p kyber.Point, n int) []kyber.Point {
	out := make([]kyber.Point, n)
	for i := range out {
		out[i] = p
	}
	return out
}

// optPtr is ptr, or NULL for an empty slice
func optPtr(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return ptr(b)
}
