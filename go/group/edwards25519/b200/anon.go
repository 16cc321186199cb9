//go:build b200

// Batch form of ring signature verification on edwards25519:
//   AnonVerifyBatch   anon.Verify(suite, msgs[j], anonymitySet, linkScope, sigs[j]) for many signatures over one anonymity set and
//                     one link scope (sign/anon/sig.go:192-248; b2k_ed25519_anon_verify).  Named apart from
//                     VerifyBatch, the eddsa form in this package.
// The suite is edwards25519.NewBlakeSHA256Ed25519 (XOF = blake2xb).  One signature is one device thread's n-step chain, far
// slower than a CPU core on its own: the batch is the use.  UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"errors"
	"io"
	"math"
	"unsafe"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/sign/anon"
)

var errInvalidSignature = errors.New("invalid signature")

// AnonVerifyBatch returns, for every signature, what anon.Verify returns: the canonical linkage tag of a valid linkable signature
// (linkScope != nil; an empty non-nil scope is linkable), an empty non-nil slice for a valid unlinkable one, and a nil tag
// with errors.New("invalid signature"), or errors.New("invalid Ed25519 curve point") for a Tag that does not decode.
// n = len(anonymitySet) sizes every signature, as in the reference: 32 (n + 1) bytes, plus 32 for the Tag when linkable.
// Bytes beyond that are never read.  A shorter signature is answered here as fixbuf's io.ReadFull would cut it: io.EOF when it
// ends on an item boundary, io.ErrUnexpectedEOF inside an item (fixbuf is not vendored in the reference, so how it wraps the
// io.ReadFull error is not visible; these are io.ReadFull's own errors).
func AnonVerifyBatch(msgs [][]byte, anonymitySet anon.Set, linkScope []byte, sigs [][]byte) (tags [][]byte, errs []error) {
	m := len(sigs)
	if len(msgs) != m {
		panic("b200: AnonVerifyBatch: msgs and sigs must have the same length")
	}
	tags, errs = make([][]byte, m), make([]error, m)
	n := len(anonymitySet)
	linkable := linkScope != nil
	siglen := 32 * (n + 1)
	if linkable {
		siglen += 32
	}
	var idx []int // the signatures that go to the device
	total := 0
	for j, s := range sigs {
		if len(s) < siglen {
			if len(s)%32 == 0 {
				errs[j] = io.EOF
			} else {
				errs[j] = io.ErrUnexpectedEOF
			}
			continue
		}
		idx = append(idx, j)
		total += len(msgs[j])
	}
	k := len(idx)
	if k == 0 {
		return tags, errs
	}
	if total > math.MaxUint32 {
		panic("b200: AnonVerifyBatch: more than 4 GiB of messages in one batch")
	}
	var ring []byte
	if n > 0 {
		ring = packPoints([]kyber.Point(anonymitySet))
	}
	sb, st, tb := make([]byte, 0, k*siglen), make([]byte, k), make([]byte, 32*k)
	mb := make([]byte, 0, total+1)
	offs := make([]uint32, k+1)
	for q, j := range idx {
		sb = append(sb, sigs[j][:siglen]...)
		mb = append(mb, msgs[j]...)
		offs[q+1] = uint32(len(mb))
	}
	if len(mb) == 0 {
		mb = append(mb, 0)
	}
	lk := C.int(0)
	if linkable {
		lk = 1
	}
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_anon_verify(c, C.size_t(n), optPtr(ring), lk, optPtr(linkScope), C.size_t(len(linkScope)),
			C.size_t(k), ptr(mb), (*C.uint32_t)(unsafe.Pointer(&offs[0])), ptr(sb), ptr(st), ptr(tb))
	})
	for q, j := range idx {
		switch st[q] {
		case C.B2K_ANON_OK:
			if linkable {
				tags[j] = append([]byte(nil), tb[32*q:32*q+32]...)
			} else {
				tags[j] = []byte{}
			}
		case C.B2K_ANON_INVALID:
			errs[j] = errInvalidSignature
		case C.B2K_ANON_POINT:
			errs[j] = errInvalidPoint
		}
	}
	return tags, errs
}
