//go:build b200

// Package b200 puts the GPU engine under kyber's edwards25519 group (group/edwards25519): Point.Mul -- the curve's hot
// operation, point.go:235-258 / geScalarMult ge.go:443-502 -- and its batch form run in libb2kyber.so
// (b2k_ed25519_mul_batch); everything else (Add, Sub, Neg, Embed, Pick, marshalling: single cheap host operations in the
// reference too) is the reference's own point, which this type wraps.  UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"crypto/cipher"
	"errors"
	"io"
	"sync"
	"unsafe"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/group/edwards25519"
)

var (
	ctxOnce sync.Once
	ctxPool chan *C.b2k_ctx
	ctxErr  error
)

func acquire() *C.b2k_ctx {
	ctxOnce.Do(func() {
		ctxPool = make(chan *C.b2k_ctx, 4)
		for i := 0; i < 4; i++ {
			var c *C.b2k_ctx
			if rc := C.b2k_create(0, &c); rc != 0 {
				ctxErr = errors.New("b200: no sm_90 device available (there is no CPU fallback)")
				return
			}
			ctxPool <- c
		}
	})
	if ctxErr != nil {
		panic(ctxErr)
	}
	return <-ctxPool
}

func ptr(b []byte) *C.uint8_t { return (*C.uint8_t)(unsafe.Pointer(&b[0])) }

// Point wraps the reference's point; methods that take points unwrap their arguments first (the reference's methods
// type-assert their own concrete type, point.go:81-83,195-197).
type Point struct {
	p kyber.Point
}

var base = new(edwards25519.Curve)

func newPoint() *Point { return &Point{p: base.Point()} }

func un(q kyber.Point) kyber.Point {
	if w, ok := q.(*Point); ok {
		return w.p
	}
	return q
}

func (P *Point) String() string                 { return P.p.String() }
func (P *Point) MarshalSize() int               { return P.p.MarshalSize() }
func (P *Point) MarshalBinary() ([]byte, error) { return P.p.MarshalBinary() }
func (P *Point) UnmarshalBinary(b []byte) error { return P.p.UnmarshalBinary(b) }
func (P *Point) MarshalTo(w io.Writer) (int, error) {
	return P.p.MarshalTo(w)
}
func (P *Point) UnmarshalFrom(r io.Reader) (int, error) { return P.p.UnmarshalFrom(r) }
func (P *Point) Equal(P2 kyber.Point) bool              { return P.p.Equal(un(P2)) }
func (P *Point) Set(P2 kyber.Point) kyber.Point         { P.p.Set(un(P2)); return P }
func (P *Point) Clone() kyber.Point                     { return &Point{p: P.p.Clone()} }
func (P *Point) Null() kyber.Point                      { P.p.Null(); return P }
func (P *Point) Base() kyber.Point                      { P.p.Base(); return P }
func (P *Point) EmbedLen() int                          { return P.p.EmbedLen() }
func (P *Point) Embed(data []byte, rand cipher.Stream) kyber.Point {
	P.p.Embed(data, rand)
	return P
}
func (P *Point) Pick(rand cipher.Stream) kyber.Point  { P.p.Pick(rand); return P }
func (P *Point) Data() ([]byte, error)                { return P.p.Data() }
func (P *Point) Add(P1, P2 kyber.Point) kyber.Point   { P.p.Add(un(P1), un(P2)); return P }
func (P *Point) Sub(P1, P2 kyber.Point) kyber.Point   { P.p.Sub(un(P1), un(P2)); return P }
func (P *Point) Neg(A kyber.Point) kyber.Point        { P.p.Neg(un(A)); return P }

// Mul replaces point.Mul (group/edwards25519/point.go:235-258): s*A, or s*B for a nil A, on the device.
// Scalars travel as their 32 little-endian bytes (scalar.go:187-189: raw, unreduced on UnmarshalBinary). The kernel
// reads them as geScalarMult does: 64 signed nibbles, a top nibble above 8 (only from 2^255 on) selecting nothing, with
// no reduction mod l, so torsion components behave as in the reference. Points travel as 32-byte compressed encodings
// (ge.go:99-150).
func (P *Point) Mul(s kyber.Scalar, A kyber.Point) kyber.Point {
	src := A
	if src == nil {
		src = base.Point().Base()
	}
	out := MulBatch([]kyber.Scalar{s}, []kyber.Point{src})
	P.p.Set(un(out[0]))
	return P
}

// MulBatch: out[i] = s[i]*A[i] in one launch (BASELINE.json configs[0]: 1024 Point.Mul; the loop of
// util/test/group.go:118-122 and benchmark/ on this group).
func MulBatch(s []kyber.Scalar, A []kyber.Point) []kyber.Point {
	n := len(s)
	out := make([]kyber.Point, n)
	if n == 0 {
		return out
	}
	sb, pb, ob := make([]byte, 32*n), make([]byte, 32*n), make([]byte, 32*n)
	for i := 0; i < n; i++ {
		b, _ := s[i].MarshalBinary() // 32 B little-endian
		copy(sb[32*i:], b)
		q, _ := un(A[i]).MarshalBinary()
		copy(pb[32*i:], q)
	}
	c := acquire()
	rc := C.b2k_ed25519_mul_batch(c, C.size_t(n), ptr(sb), ptr(pb), ptr(ob))
	msg := C.GoString(C.b2k_last_error(c))
	ctxPool <- c
	if rc != 0 {
		panic("b200: " + msg)
	}
	for i := 0; i < n; i++ {
		q := newPoint()
		if err := q.p.UnmarshalBinary(ob[32*i : 32*i+32]); err != nil {
			panic("b200: engine returned an undecodable point")
		}
		out[i] = q
	}
	return out
}

// Curve is the kyber.Group: the reference's Curve with Point() returning the engine-backed wrapper.
type Curve struct {
	edwards25519.Curve
}

func (c *Curve) Point() kyber.Point { return newPoint() }

// SuiteEd25519 mirrors group/edwards25519/suite.go:22-60 with the group swapped.
type SuiteEd25519 struct {
	*edwards25519.SuiteEd25519
	curve Curve
}

func (s *SuiteEd25519) Point() kyber.Point { return s.curve.Point() }

func NewBlakeSHA256Ed25519() *SuiteEd25519 {
	return &SuiteEd25519{SuiteEd25519: edwards25519.NewBlakeSHA256Ed25519()}
}
func NewBlakeSHA256Ed25519WithRand(r cipher.Stream) *SuiteEd25519 {
	return &SuiteEd25519{SuiteEd25519: edwards25519.NewBlakeSHA256Ed25519WithRand(r)}
}
