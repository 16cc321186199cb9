//go:build b200

// Batch forms of the share/poly operations on edwards25519, the group kyber's secret-sharing protocols run on
// (share/vss/pedersen, share/dkg/pedersen, share/pvss, sign/dss, sign/cosi):
//   MSM            sum s_i P_i in one call (b2k_ed25519_msm): the Mul + Add loops
//   RecoverCommit  share.RecoverCommit (share/poly.go:449-476) with the Lagrange weights and the MSM on the device
//   PubPolyCheck   share.PubPoly.Check (share/poly.go:405-409) for a batch of deals, as vss.go:636-645 and dkg.go:489-494,
//                  826-834 run it once per deal, response and justification
// Scalars travel as their 32 little-endian bytes and are read like the reference's Point.Mul reads them (geScalarMult);
// points as 32-byte compressed encodings.  UNCOMPILED: no Go toolchain in the build image.
package b200

/*
#cgo LDFLAGS: -lb2kyber
#include <b2kyber.h>
*/
import "C"

import (
	"errors"
	"sort"
	"unsafe"

	"go.dedis.ch/kyber/v4"
	"go.dedis.ch/kyber/v4/share"
)

func u32ptr(b []uint32) *C.uint32_t { return (*C.uint32_t)(unsafe.Pointer(&b[0])) }

// run calls f with a pooled context and panics with the library's message if it fails
func run(f func(c *C.b2k_ctx) C.int) {
	c := acquire()
	rc := f(c)
	msg := C.GoString(C.b2k_last_error(c))
	ctxPool <- c
	if rc != 0 {
		panic("b200: " + msg)
	}
}

func packScalars(s []kyber.Scalar) []byte {
	b := make([]byte, 32*len(s))
	for i, x := range s {
		v, _ := x.MarshalBinary() // 32 B little-endian, unreduced (scalar.go:226-233)
		copy(b[32*i:], v)
	}
	return b
}

func packPoints(p []kyber.Point) []byte {
	b := make([]byte, 32*len(p))
	for i, x := range p {
		v, _ := un(x).MarshalBinary()
		copy(b[32*i:], v)
	}
	return b
}

func unpackPoint(b []byte) kyber.Point {
	q := newPoint()
	if err := q.p.UnmarshalBinary(b); err != nil {
		panic("b200: engine returned an undecodable point")
	}
	return q
}

// MSM returns sum_i s[i] * p[i]; the identity for an empty input
func MSM(s []kyber.Scalar, p []kyber.Point) kyber.Point {
	n := len(s)
	if len(p) != n {
		panic("b200: MSM: scalars and points must have the same length")
	}
	if n == 0 {
		return newPoint().Null()
	}
	sb, pb, out := packScalars(s), packPoints(p), make([]byte, 32)
	run(func(c *C.b2k_ctx) C.int { return C.b2k_ed25519_msm(c, C.size_t(n), ptr(sb), ptr(pb), ptr(out)) })
	return unpackPoint(out)
}

// RecoverCommit is share.RecoverCommit: xyCommit's selection (poly.go:418-445: non-nil shares sorted by index, the first t
// kept) on the host, the Lagrange weights at zero and the t-term MSM on the device
func RecoverCommit(shares []*share.PubShare, t, n uint32) (kyber.Point, error) {
	sorted := make([]*share.PubShare, 0, len(shares))
	for _, s := range shares {
		if s != nil {
			sorted = append(sorted, s)
		}
	}
	sort.Slice(sorted, func(i, j int) bool { return sorted[i].I < sorted[j].I })
	if uint32(len(sorted)) > t {
		sorted = sorted[:t]
	}
	if uint32(len(sorted)) < t || t == 0 {
		return nil, errors.New("share: not enough good public shares to reconstruct secret commitment")
	}
	idx := make([]uint32, t)
	pts := make([]kyber.Point, t)
	for i, s := range sorted {
		idx[i] = s.I
		pts[i] = s.V
	}
	pb, out := packPoints(pts), make([]byte, 32)
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_recover_commit(c, C.size_t(t), u32ptr(idx), ptr(pb), ptr(out))
	})
	return unpackPoint(out), nil
}

// PubPolyCheck returns ok[d][k] = share.NewPubPoly(g, nil, commits[d]).Check(shares[d][k]) for m deals that share one
// threshold t (every commits[d] has t entries) and hold the same number of shares, in one call
func PubPolyCheck(commits [][]kyber.Point, shares [][]*share.PriShare) [][]bool {
	m := len(commits)
	if len(shares) != m {
		panic("b200: PubPolyCheck: one row of shares per deal")
	}
	ok := make([][]bool, m)
	if m == 0 || len(commits[0]) == 0 || len(shares[0]) == 0 {
		return ok
	}
	t, n := len(commits[0]), len(shares[0])
	cb := make([]byte, 0, 32*m*t)
	idx := make([]uint32, 0, m*n)
	var sv []kyber.Scalar
	for d := 0; d < m; d++ {
		if len(commits[d]) != t || len(shares[d]) != n {
			panic("b200: PubPolyCheck: every deal needs the same threshold and share count")
		}
		cb = append(cb, packPoints(commits[d])...)
		for _, s := range shares[d] {
			idx = append(idx, s.I)
			sv = append(sv, s.V)
		}
	}
	sb, res := packScalars(sv), make([]byte, m*n)
	run(func(c *C.b2k_ctx) C.int {
		return C.b2k_ed25519_pubpoly_check(c, C.size_t(m), C.size_t(t), ptr(cb), C.size_t(n), u32ptr(idx), ptr(sb), ptr(res))
	})
	for d := 0; d < m; d++ {
		ok[d] = make([]bool, n)
		for k := 0; k < n; k++ {
			ok[d][k] = res[d*n+k] == 1
		}
	}
	return ok
}
