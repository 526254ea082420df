//go:build cgo && cuda

package identity

/*
#cgo LDFLAGS: -lafcrypto
#include "afcrypto.h"
*/
import "C"

import (
	"strings"
	"unsafe"
)

// RegisterCUDA registers a batch of new agents in one afc_did_register_batch call on ctx (an afc_ctx*).  A master seed of any length but
// 32 bytes, or any non-zero return code, sends the whole batch through RegisterStdlib.  The expanded keys it returns feed
// afc_ed25519_sign_expanded* and both credential issue calls; the caller wipes them when it is done.
type RegisterCUDA struct {
	ctx      unsafe.Pointer
	fallback RegisterStdlib
}

func NewRegisterCUDA(ctx unsafe.Pointer) *RegisterCUDA { return &RegisterCUDA{ctx: ctx} }

func u8(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&b[0]))
}

func (r *RegisterCUDA) Register(masterSeed []byte, serverID string, reqs []Request) ([]Result, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	if len(masterSeed) != 32 {
		return r.fallback.Register(masterSeed, serverID, reqs)
	}
	var nodes, ids []byte
	nodeOff := make([]uint64, n+1)
	idIdx := make([]uint64, 2*n+1)
	idOff := []uint64{0}
	agentIndex := make([]uint32, n)
	for i, q := range reqs {
		nodes = append(nodes, q.AgentNodeID...)
		nodeOff[i+1] = uint64(len(nodes))
		agentIndex[i] = q.AgentIndex
		for k, list := range [2][]string{q.Reasoners, q.Skills} {
			for _, id := range list {
				ids = append(ids, id...)
				idOff = append(idOff, uint64(len(ids)))
			}
			idIdx[2*i+k+1] = uint64(len(idOff) - 1)
		}
	}
	nodes = append(nodes, 0) // never empty, so &nodes[0] exists
	ids = append(ids, 0)
	slots := n + len(idOff) - 1
	sid := []byte(serverID + "\x00")
	bound := uint64(C.afc_did_register_bound((*C.uint64_t)(&nodeOff[0]), (*C.uint64_t)(&idIdx[0]), (*C.uint64_t)(&idOff[0]), C.uint32_t(n),
		C.uint64_t(len(serverID))))
	compOff := make([]uint64, n+1)
	bodyOff := make([]uint64, n+1)
	expanded := make([]byte, 96*slots)
	pks := make([]byte, 32*slots)
	dids := make([]byte, C.AFC_DID_CHARS*slots)
	paths := make([]byte, C.AFC_DID_PATH_SLOT*slots)
	flags := make([]byte, slots)
	body := make([]byte, bound+1)
	rc := C.afc_did_register_batch((*C.afc_ctx)(r.ctx), u8(masterSeed), u8(sid), C.uint64_t(len(serverID)), u8(nodes), (*C.uint64_t)(&nodeOff[0]),
		(*C.uint32_t)(&agentIndex[0]), (*C.uint64_t)(&idIdx[0]), u8(ids), (*C.uint64_t)(&idOff[0]), C.uint32_t(n), (*C.uint64_t)(&compOff[0]),
		u8(expanded), u8(pks), u8(dids), u8(paths), u8(flags), u8(body), C.uint64_t(bound), (*C.uint64_t)(&bodyOff[0]))
	wipe := func() {
		for i := range expanded {
			expanded[i] = 0
		}
		for i := range body {
			body[i] = 0 // every private JWK
		}
	}
	defer wipe()
	if rc != 0 {
		return r.fallback.Register(masterSeed, serverID, reqs)
	}
	out := make([]Result, n)
	for i := range reqs {
		c0, c1 := int(compOff[i]), int(compOff[i+1])
		comps := make([]Component, 0, c1-c0)
		for c := c0; c < c1; c++ {
			comp := Component{
				Path: strings.TrimRight(string(paths[C.AFC_DID_PATH_SLOT*c:C.AFC_DID_PATH_SLOT*(c+1)]), "\x00"),
				DID:  string(dids[C.AFC_DID_CHARS*c : C.AFC_DID_CHARS*(c+1)]),
				Kept: flags[c]&C.AFC_DID_KEPT != 0,
			}
			copy(comp.Key[:], expanded[96*c:96*c+96])
			comps = append(comps, comp)
		}
		out[i] = Result{Components: comps, Body: append([]byte(nil), body[bodyOff[i]:bodyOff[i+1]]...)}
	}
	return out, nil
}
