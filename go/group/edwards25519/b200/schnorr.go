//go:build b200

// Batch form of schnorr.VerifyWithChecks / schnorr.Verify (sign/schnorr/schnorr.go:89-183) on edwards25519.  On this group
// sign/schnorr and sign/eddsa accept exactly the same signatures: the checks are the same set (decode, canonical and small
// order for R and the key, s canonical) in another order, the hash is the same SHA-512, and the digest over re-encodings
// equals eddsa's over the raw bytes once R and the key passed "canonical" and "not small order".  So the device path is
// b2k_ed25519_verify, and its statuses map as: 0 -> nil, 8 (encode(s B) != encode(R + h A)) -> "schnorr: invalid signature",
// 1-7 -> the reference's schnorr.VerifyWithChecks for that signature on the host, which then fails before any scalar
// multiplication and returns its own first error (at most two decodes).
// UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"errors"
	"fmt"
	"math"
	"unsafe"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/sign/schnorr"
)

var errSchnorrInvalid = errors.New("schnorr: invalid signature")

// SchnorrVerifyWithChecksBatch returns errs[i] = schnorr.VerifyWithChecks(g, pubs[i], msgs[i], sigs[i]) for every i, with g
// the edwards25519 group, in one device call.  A signature that is not 64 bytes gets the reference's length error on the
// host; a key that is not 32 bytes travels as 32 bytes of 0xff (no valid encoding) and its error comes from the host re-run.
func SchnorrVerifyWithChecksBatch(g kyber.Group, pubs, msgs, sigs [][]byte) []error {
	n := len(sigs)
	if len(pubs) != n || len(msgs) != n {
		panic("b200: SchnorrVerifyWithChecksBatch: pubs, msgs and sigs must have the same length")
	}
	errs := make([]error, n)
	idx := make([]int, 0, n) // the signatures that go to the device
	total := 0
	for i := range sigs {
		if len(sigs[i]) != 64 {
			errs[i] = fmt.Errorf("schnorr: signature of invalid length %d instead of %d", len(sigs[i]), 64)
			continue
		}
		idx = append(idx, i)
		total += len(msgs[i])
	}
	m := len(idx)
	if m == 0 {
		return errs
	}
	if total > math.MaxUint32 {
		panic("b200: SchnorrVerifyWithChecksBatch: more than 4 GiB of messages in one batch")
	}
	pb, sb, st := make([]byte, 32*m), make([]byte, 64*m), make([]byte, m)
	mb := make([]byte, 0, total+1)
	offs := make([]uint32, m+1)
	for k, i := range idx {
		if len(pubs[i]) == 32 {
			copy(pb[32*k:], pubs[i])
		} else {
			for j := 0; j < 32; j++ {
				pb[32*k+j] = 0xff
			}
		}
		copy(sb[64*k:], sigs[i])
		mb = append(mb, msgs[i]...)
		offs[k+1] = uint32(len(mb))
	}
	if len(mb) == 0 {
		mb = append(mb, 0)
	}
	c := acquire()
	rc := C.b2k_ed25519_verify(c, C.size_t(m), ptr(pb), ptr(mb), (*C.uint32_t)(unsafe.Pointer(&offs[0])), ptr(sb), ptr(st))
	msg := C.GoString(C.b2k_last_error(c))
	ctxPool <- c
	if rc != 0 {
		panic("b200: " + msg)
	}
	for k, i := range idx {
		switch st[k] {
		case C.B2K_ED_OK:
		case C.B2K_ED_NOT_EQUAL:
			errs[i] = errSchnorrInvalid
		default:
			errs[i] = schnorr.VerifyWithChecks(g, pubs[i], msgs[i], sigs[i])
			if errs[i] == nil {
				panic("b200: the device refused a signature the reference accepts")
			}
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
