//go:build cgo && cuda

package identity

/*
#include "afcrypto.h"
*/
import "C"

import (
	"net/http"
	"sync"
	"unsafe"
)

// ResolveCUDA serves a batch of DID requests in one afc_did_resolve_batch call on ctx (an afc_ctx*).  The snapshot lives on the device as
// one afc_did_directory with identities, built at the first call after New / SetSnapshot: each DID once, its first holder in the
// snapshot's order.  Any non-zero return code sends the whole batch through ResolveStdlib, and so does each request the device marks
// AFC_DIDRES_HOST.  The snapshot passed to Serve serves that fallback; it must be the one SetSnapshot installed.
type ResolveCUDA struct {
	ctx      unsafe.Pointer
	fallback ResolveStdlib
	mu       sync.Mutex
	snap     *Snapshot
	dir      *C.afc_did_directory
}

func NewResolveCUDA(ctx unsafe.Pointer, snap *Snapshot) *ResolveCUDA { return &ResolveCUDA{ctx: ctx, snap: snap} }

// SetSnapshot installs a new registry snapshot after a registration; the directory is rebuilt at its next use.
func (s *ResolveCUDA) SetSnapshot(snap *Snapshot) {
	s.mu.Lock()
	defer s.mu.Unlock()
	if s.dir != nil {
		C.afc_did_directory_free(s.dir)
	}
	s.snap, s.dir = snap, nil
}

func (s *ResolveCUDA) directory() *C.afc_did_directory {
	if s.dir != nil {
		return s.dir
	}
	var dids, cols []byte
	var kinds []byte
	off, coff := []uint64{0}, []uint64{0}
	seen := map[string]bool{}
	add := func(did string, kind byte, path, fn, jwk string) {
		if seen[did] {
			return
		}
		seen[did] = true
		dids = append(dids, did...)
		off = append(off, uint64(len(dids)))
		kinds = append(kinds, kind)
		for _, v := range []string{path, fn, jwk} {
			cols = append(cols, v...)
			coff = append(coff, uint64(len(cols)))
		}
	}
	root, _ := lookup(s.snap, s.snap.RootDID)
	add(root.DID, C.AFC_DID_KIND_SERVER, root.DerivationPath, "", root.PublicKeyJWK)
	for _, a := range s.snap.Agents {
		add(a.DID, C.AFC_DID_KIND_AGENT, a.DerivationPath, "", a.PublicKeyJWK)
		for _, c := range a.Reasoners {
			add(c.DID, C.AFC_DID_KIND_REASONER, c.DerivationPath, c.FunctionName, c.PublicKeyJWK)
		}
		for _, c := range a.Skills {
			add(c.DID, C.AFC_DID_KIND_SKILL, c.DerivationPath, c.FunctionName, c.PublicKeyJWK)
		}
	}
	n := len(off) - 1
	pks := make([]byte, 32*n+32) // afc_did_resolve_batch reads no key
	dids, cols, kinds = append(dids, 0), append(cols, 0), append(kinds, 0)
	var d *C.afc_did_directory
	if C.afc_did_directory_new((*C.afc_ctx)(s.ctx), u8(pks), u8(dids), (*C.uint64_t)(unsafe.Pointer(&off[0])), C.uint32_t(n), &d) != 0 {
		return nil
	}
	if C.afc_did_directory_set_identities(d, u8(kinds), u8(cols), (*C.uint64_t)(unsafe.Pointer(&coff[0]))) != 0 {
		C.afc_did_directory_free(d)
		return nil
	}
	s.dir = d
	return d
}

func (s *ResolveCUDA) Serve(snap *Snapshot, reqs []ResolveReq) ([]ResolveResp, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	s.mu.Lock()
	defer s.mu.Unlock()
	dir := s.directory()
	if dir == nil {
		return s.fallback.Serve(snap, reqs)
	}
	kinds := make([]byte, n+1)
	var buf []byte
	off := make([]uint64, n+1)
	for i, r := range reqs {
		kinds[i] = byte(r.Kind)
		buf = append(buf, r.DID...)
		off[i+1] = uint64(len(buf))
	}
	buf = append(buf, 0)
	capacity := uint64(C.afc_did_resolve_bound(dir, (*C.uint64_t)(unsafe.Pointer(&off[0])), C.uint32_t(n)))
	bodies := make([]byte, capacity+1)
	bodyOff := make([]uint64, n+1)
	state := make([]byte, n)
	if C.afc_did_resolve_batch((*C.afc_ctx)(s.ctx), dir, u8(kinds), u8(buf), (*C.uint64_t)(unsafe.Pointer(&off[0])), C.uint32_t(n), u8(bodies),
		C.uint64_t(capacity), (*C.uint64_t)(unsafe.Pointer(&bodyOff[0])), u8(state)) != 0 {
		return s.fallback.Serve(snap, reqs)
	}
	status := map[byte]int{C.AFC_DIDRES_FOUND: http.StatusOK, C.AFC_DIDRES_NOT_FOUND: http.StatusNotFound, C.AFC_DIDRES_BAD_REQUEST: http.StatusBadRequest}
	out := make([]ResolveResp, n)
	for i := range reqs {
		if state[i] == C.AFC_DIDRES_HOST {
			out[i] = serveOne(snap, reqs[i])
			continue
		}
		out[i] = ResolveResp{status[state[i]], append([]byte(nil), bodies[bodyOff[i]:bodyOff[i+1]]...)}
	}
	return out, nil
}
