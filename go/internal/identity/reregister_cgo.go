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

// ReregisterCUDA re-registers a batch of known agents in one afc_did_reregister_batch call on ctx (an afc_ctx*).  A master seed of any
// length but 32 bytes, or any non-zero return code, sends the whole batch through ReregisterStdlib.  The slots' expanded keys feed
// afc_ed25519_sign_expanded* and both credential issue calls; the caller wipes them when it is done.
type ReregisterCUDA struct {
	ctx      unsafe.Pointer
	fallback ReregisterStdlib
}

func NewReregisterCUDA(ctx unsafe.Pointer) *ReregisterCUDA { return &ReregisterCUDA{ctx: ctx} }

func (r *ReregisterCUDA) Reregister(masterSeed []byte, serverID string, reqs []ReRequest) ([]ReResult, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	if len(masterSeed) != 32 {
		return r.fallback.Reregister(masterSeed, serverID, reqs)
	}
	var agentCols, ids, regCols []byte
	agentOff := []uint64{0}
	idIdx := make([]uint64, 2*n+1)
	idOff := []uint64{0}
	regIdx := make([]uint64, 2*n+1)
	regOff := []uint64{0}
	agentIndex := make([]uint32, n)
	for i, q := range reqs {
		for _, s := range [3][]byte{[]byte(q.Agent.DID), q.Agent.PublicKeyJWK, []byte(q.Agent.DerivationPath)} {
			agentCols = append(agentCols, s...)
			agentOff = append(agentOff, uint64(len(agentCols)))
		}
		agentIndex[i] = q.AgentIndex
		for k, list := range [2][]string{q.Reasoners, q.Skills} {
			for _, id := range list {
				ids = append(ids, id...)
				idOff = append(idOff, uint64(len(ids)))
			}
			idIdx[2*i+k+1] = uint64(len(idOff) - 1)
			for _, c := range [2][]StoredComponent{q.Agent.Reasoners, q.Agent.Skills}[k] {
				for _, s := range [5][]byte{[]byte(c.Key), []byte(c.DID), c.PublicKeyJWK, []byte(c.DerivationPath), []byte(c.FunctionName)} {
					regCols = append(regCols, s...)
					regOff = append(regOff, uint64(len(regCols)))
				}
			}
			regIdx[2*i+k+1] = uint64((len(regOff) - 1) / 5)
		}
	}
	agentCols, ids, regCols = append(agentCols, 0), append(ids, 0), append(regCols, 0) // never empty, so &x[0] exists
	m, g := len(idOff)-1, (len(regOff)-1)/5
	sid := []byte(serverID + "\x00")
	bound := uint64(C.afc_did_reregister_bound((*C.uint64_t)(&agentOff[0]), (*C.uint64_t)(&idIdx[0]), (*C.uint64_t)(&idOff[0]),
		(*C.uint64_t)(&regIdx[0]), (*C.uint64_t)(&regOff[0]), C.uint32_t(n), C.uint64_t(len(serverID))))
	state := make([]byte, n)
	counts := make([]uint32, 4*n)
	expanded := make([]byte, 96*2*n)
	pks := make([]byte, 32*2*n)
	dids := make([]byte, C.AFC_DID_CHARS*2*n)
	paths := make([]byte, C.AFC_DID_PATH_SLOT*2*n)
	regFlags := make([]byte, g+1)
	idFlags := make([]byte, m+1)
	body := make([]byte, bound+1)
	bodyOff := make([]uint64, n+1)
	rc := C.afc_did_reregister_batch((*C.afc_ctx)(r.ctx), u8(masterSeed), u8(sid), C.uint64_t(len(serverID)), u8(agentCols), (*C.uint64_t)(&agentOff[0]),
		(*C.uint32_t)(&agentIndex[0]), (*C.uint64_t)(&idIdx[0]), u8(ids), (*C.uint64_t)(&idOff[0]), (*C.uint64_t)(&regIdx[0]), u8(regCols),
		(*C.uint64_t)(&regOff[0]), C.uint32_t(n), u8(state), (*C.uint32_t)(&counts[0]), u8(expanded), u8(pks), u8(dids), u8(paths), u8(regFlags),
		u8(idFlags), u8(body), C.uint64_t(bound), (*C.uint64_t)(&bodyOff[0]))
	wipe := func() {
		for i := range expanded {
			expanded[i] = 0
		}
		for i := range body {
			body[i] = 0 // the new components' private JWKs
		}
	}
	defer wipe()
	if rc != 0 {
		return r.fallback.Reregister(masterSeed, serverID, reqs)
	}
	out := make([]ReResult, n)
	gi, ii := 0, 0
	for i, q := range reqs {
		res := &out[i]
		res.State = int(state[i])
		for k := 0; k < 4; k++ {
			res.Counts[k] = int(counts[4*i+k])
		}
		res.Body = append([]byte(nil), body[bodyOff[i]:bodyOff[i+1]]...)
		for kind, list := range [2][]string{q.Reasoners, q.Skills} {
			stored := [2][]StoredComponent{q.Agent.Reasoners, q.Agent.Skills}[kind]
			res.Gone[kind] = make([]bool, len(stored))
			for k := range stored {
				res.Gone[kind][k] = regFlags[gi]&C.AFC_DIDRR_GONE != 0
				gi++
			}
			for _, id := range list {
				if idFlags[ii] == C.AFC_DIDRR_NEW|C.AFC_DID_KEPT {
					res.New[kind] = append(res.New[kind], id)
				}
				ii++
			}
			if res.State == RePartial && res.Counts[kind] > 0 {
				t := 2*i + kind
				c := &Component{Path: strings.TrimRight(string(paths[C.AFC_DID_PATH_SLOT*t:C.AFC_DID_PATH_SLOT*(t+1)]), "\x00"),
					DID: string(dids[C.AFC_DID_CHARS*t : C.AFC_DID_CHARS*(t+1)]), Kept: true}
				copy(c.Key[:], expanded[96*t:96*t+96])
				res.Slots[kind] = c
			}
		}
	}
	return out, nil
}
