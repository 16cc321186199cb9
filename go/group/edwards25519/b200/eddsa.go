//go:build b200

// Batch form of eddsa.VerifyWithChecks / eddsa.Verify (sign/eddsa/eddsa.go:149-239): every signature of the batch is checked
// on the device in one call (b2k_ed25519_verify), with the reference's checks in the reference's order, and gets the error
// the reference would return for it, wrapped the same way (errors.Is holds for the eddsa.Err* values).
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
	"go.dedis.ch/kyber/v4/sign/eddsa"
)

// the error of point.UnmarshalBinary (group/edwards25519/point.go:65-70), which the reference wraps for R and the key
var errInvalidPoint = errors.New("invalid Ed25519 curve point")

// statusError turns the B2K_ED_* status of one signature into the error VerifyWithChecks returns for it
func statusError(st byte) error {
	switch st {
	case C.B2K_ED_OK:
		return nil
	case C.B2K_ED_SIG_NOT_CANONICAL:
		return fmt.Errorf("error: %w", eddsa.ErrSignatureNotCanonical)
	case C.B2K_ED_R_NOT_CANONICAL:
		return fmt.Errorf("error: %w", eddsa.ErrPointRNotCanonical)
	case C.B2K_ED_R_INVALID:
		return fmt.Errorf("error: %w: %w", eddsa.ErrPointRInvalid, errInvalidPoint)
	case C.B2K_ED_R_SMALL_ORDER:
		return fmt.Errorf("error: %w", eddsa.ErrPointRSmallOrder)
	case C.B2K_ED_PK_NOT_CANONICAL:
		return fmt.Errorf("error: %w", eddsa.ErrPKNotCanonical)
	case C.B2K_ED_PK_INVALID:
		return fmt.Errorf("error: %w: %w", eddsa.ErrPKInvalid, errInvalidPoint)
	case C.B2K_ED_PK_SMALL_ORDER:
		return fmt.Errorf("error: %w", eddsa.ErrPKSmallOrder)
	case C.B2K_ED_NOT_EQUAL:
		return fmt.Errorf("error: %w", eddsa.ErrSignatureRecNotEqual)
	}
	panic("b200: unknown verification status")
}

// VerifyWithChecksBatch returns errs[i] = eddsa.VerifyWithChecks(pubs[i], msgs[i], sigs[i]) for every i, computed on the
// device in one call.  Lengths keep the reference's order: a signature that is not 64 bytes gets ErrSignatureLength on the
// host and never reaches the device; a key that is not 32 bytes travels as 32 bytes of 0xff, which point.IsCanonical
// rejects, so it fails with ErrPKNotCanonical only after the signature's own checks (point.IsCanonical returns false
// for any other length, point.go:308-311).
func VerifyWithChecksBatch(pubs, msgs, sigs [][]byte) []error {
	n := len(sigs)
	if len(pubs) != n || len(msgs) != n {
		panic("b200: VerifyWithChecksBatch: pubs, msgs and sigs must have the same length")
	}
	errs := make([]error, n)
	idx := make([]int, 0, n) // the signatures that go to the device
	total := 0
	for i := range sigs {
		if len(sigs[i]) != 64 {
			errs[i] = fmt.Errorf("error: %w: expect 64 but got %v", eddsa.ErrSignatureLength, len(sigs[i]))
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
		panic("b200: VerifyWithChecksBatch: more than 4 GiB of messages in one batch")
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
		errs[i] = statusError(st[k])
	}
	return errs
}

// VerifyBatch is the batch twin of eddsa.Verify (eddsa.go:231-239): the keys are marshalled first, and a key that does not
// marshal gets ErrPKMarshalling like in the reference.
func VerifyBatch(pubs []kyber.Point, msgs, sigs [][]byte) []error {
	if len(pubs) != len(sigs) {
		panic("b200: VerifyBatch: pubs, msgs and sigs must have the same length")
	}
	pb := make([][]byte, len(pubs))
	bad := make([]error, len(pubs))
	for i, p := range pubs {
		b, err := un(p).MarshalBinary()
		if err != nil {
			bad[i] = fmt.Errorf("error: %w: %w", eddsa.ErrPKMarshalling, err)
		}
		pb[i] = b
	}
	errs := VerifyWithChecksBatch(pb, msgs, sigs)
	for i := range errs {
		if bad[i] != nil {
			errs[i] = bad[i]
		}
	}
	return errs
}
