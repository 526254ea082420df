//go:build cgo && cuda

package crypto

/*
#include "afcrypto.h"
*/
import "C"

import (
	"sync"
	"unsafe"
)

// ChainCUDA serves a batch of workflow chains in one afc_vc_workflow_chain_batch call.  The registry's public half lives on the device
// as one afc_did_directory per context, built from the keys map at the first call on that context (SetKeys replaces it after a
// registration).  Any non-zero return code sends the whole batch through ChainStdlib, and so does each workflow the device marks
// AFC_CHAIN_HOST.  keys passed to WorkflowChainBatch serve that fallback; they must be the map the directories hold.
type ChainCUDA struct {
	c        *CUDA
	fallback ChainStdlib
	mu       sync.Mutex
	keys     map[string][]byte
	dirs     map[*C.afc_ctx]*C.afc_did_directory
}

func NewChainCUDA(c *CUDA, keys map[string][]byte) *ChainCUDA {
	return &ChainCUDA{c: c, keys: keys, dirs: map[*C.afc_ctx]*C.afc_did_directory{}}
}

// SetKeys installs a new registry snapshot; the device directories are rebuilt at their next use.
func (s *ChainCUDA) SetKeys(keys map[string][]byte) {
	s.mu.Lock()
	defer s.mu.Unlock()
	for _, d := range s.dirs {
		C.afc_did_directory_free(d)
	}
	s.keys, s.dirs = keys, map[*C.afc_ctx]*C.afc_did_directory{}
}

func (s *ChainCUDA) directory(ctx *C.afc_ctx) *C.afc_did_directory {
	s.mu.Lock()
	defer s.mu.Unlock()
	if d, ok := s.dirs[ctx]; ok {
		return d
	}
	var dids, pks []byte
	off := []uint64{0}
	for did, pk := range s.keys {
		if len(pk) != 32 {
			return nil
		}
		dids = append(dids, did...)
		off = append(off, uint64(len(dids)))
		pks = append(pks, pk...)
	}
	dids, pks = append(dids, 0), append(pks, make([]byte, 32)...)
	var d *C.afc_did_directory
	if C.afc_did_directory_new(ctx, (*C.uint8_t)(unsafe.Pointer(&pks[0])), (*C.uint8_t)(unsafe.Pointer(&dids[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])),
		C.uint32_t(len(off)-1), &d) != 0 {
		return nil
	}
	s.dirs[ctx] = d
	return d
}

// chainPacking holds the call's host arrays, in include/afcrypto.h's layout
type chainPacking struct {
	cols, rcols, ccols, crcols []byte
	colOff, recOff, rcolOff, ccolOff, crcolOff []uint64
	created, clock, size []int64
	zone []int32
	flags []uint8
	ki []uint32
}

func (s *ChainCUDA) WorkflowChainBatch(reqs []ChainRequest, keys map[string][]byte) ([][]byte, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	keyOf := map[string]uint32{}
	var seeds []byte
	p := chainPacking{colOff: []uint64{0}, recOff: []uint64{0}, rcolOff: []uint64{0}, ccolOff: []uint64{0}, crcolOff: []uint64{0}}
	add := func(buf *[]byte, off *[]uint64, v string) { *buf = append(*buf, v...); *off = append(*off, uint64(len(*buf))) }
	for i := range reqs {
		r := &reqs[i]
		k := string(r.Key.Seed())
		j, ok := keyOf[k]
		if !ok {
			j = uint32(len(keyOf))
			keyOf[k] = j
			seeds = append(seeds, k...)
		}
		p.ki = append(p.ki, j)
		session := ""
		if len(r.Records) > 0 {
			session = r.Records[0].SessionID
		}
		for _, v := range [C.AFC_WORKFLOW_COLUMNS]string{r.WorkflowID, session, workflowIssuer(&r.WorkflowRequest), r.VCID, r.IssuanceDate, r.SnapshotText, r.ProofCreated} {
			add(&p.cols, &p.colOff, v)
		}
		add(&p.ccols, &p.ccolOff, r.WorkflowVCID)
		add(&p.ccols, &p.ccolOff, r.ResolvedAt)
		_, zoff := r.SnapshotTime.Zone()
		p.clock = append(p.clock, r.SnapshotTime.Unix(), int64(r.SnapshotTime.Nanosecond()), int64(zoff))
		for _, vc := range r.Records {
			add(&p.rcols, &p.rcolOff, vc.VCID)
			add(&p.rcols, &p.rcolOff, vc.Status)
			var f uint8
			agent, name := "", ""
			if vc.AgentNodeID == nil {
				f |= C.AFC_CHAIN_AGENT_NODE_ID_NIL
			} else {
				agent = *vc.AgentNodeID
			}
			if vc.WorkflowName == nil {
				f |= C.AFC_CHAIN_WORKFLOW_NAME_NIL
			} else {
				name = *vc.WorkflowName
			}
			if vc.VCDocument == nil {
				f |= C.AFC_CHAIN_VC_DOCUMENT_NIL
			}
			for _, v := range [C.AFC_CHAIN_RECORD_COLUMNS]string{vc.ExecutionID, vc.WorkflowID, vc.SessionID, agent, name, vc.IssuerDID, vc.TargetDID,
				vc.CallerDID, string(vc.VCDocument), vc.Signature, vc.StorageURI, vc.InputHash, vc.OutputHash} {
				add(&p.crcols, &p.crcolOff, v)
			}
			_, zc := vc.CreatedAt.Zone()
			p.created = append(p.created, vc.CreatedAt.Unix(), int64(vc.CreatedAt.Nanosecond()))
			p.zone = append(p.zone, int32(zc))
			p.flags = append(p.flags, f)
			p.size = append(p.size, vc.DocumentSize)
		}
		p.recOff = append(p.recOff, uint64(len(p.rcolOff)-1)/2)
	}
	// every array non-empty, so that &x[0] is valid
	p.cols, p.rcols, p.ccols, p.crcols = append(p.cols, 0), append(p.rcols, 0), append(p.ccols, 0), append(p.crcols, 0)
	p.created, p.size, p.zone, p.flags = append(p.created, 0, 0), append(p.size, 0), append(p.zone, 0), append(p.flags, 0)
	d := s.c.pick()
	dir := s.directory(d.ctx)
	if dir == nil {
		return s.fallback.WorkflowChainBatch(reqs, keys)
	}
	exp := make([]byte, 96*len(keyOf))
	if C.afc_ed25519_expand_batch(d.ctx, (*C.uint8_t)(unsafe.Pointer(&seeds[0])), C.uint32_t(len(keyOf)), (*C.uint8_t)(unsafe.Pointer(&exp[0]))) != 0 {
		return s.fallback.WorkflowChainBatch(reqs, keys)
	}
	defer func() {
		for i := range exp {
			exp[i] = 0
		}
	}()
	u8 := func(b []byte) *C.uint8_t { return (*C.uint8_t)(unsafe.Pointer(&b[0])) }
	u64 := func(b []uint64) *C.uint64_t { return (*C.uint64_t)(unsafe.Pointer(&b[0])) }
	i64 := func(b []int64) *C.int64_t { return (*C.int64_t)(unsafe.Pointer(&b[0])) }
	bound := int(C.afc_vc_workflow_chain_bound(u64(p.colOff), u64(p.recOff), u64(p.rcolOff), u64(p.ccolOff), u64(p.crcolOff), C.uint32_t(n)))
	bodies := make([]byte, bound+1)
	bodyOff := make([]uint64, n+1)
	state := make([]uint8, n)
	rc := C.afc_vc_workflow_chain_batch(d.ctx, u8(exp), C.uint32_t(len(keyOf)), (*C.uint32_t)(unsafe.Pointer(&p.ki[0])), u8(p.cols), u64(p.colOff),
		u64(p.recOff), u8(p.rcols), u64(p.rcolOff), i64(p.created), u8(p.ccols), u64(p.ccolOff), i64(p.clock), u8(p.crcols), u64(p.crcolOff),
		u8(p.flags), i64(p.size), (*C.int32_t)(unsafe.Pointer(&p.zone[0])), dir, C.uint32_t(n), u8(bodies), C.uint64_t(bound), u64(bodyOff),
		u8(state))
	if rc != 0 {
		return s.fallback.WorkflowChainBatch(reqs, keys)
	}
	out := make([][]byte, n)
	for i := range reqs {
		if state[i] != C.AFC_CHAIN_BUILT {
			b, err := chainOne(&reqs[i], keys)
			if err != nil {
				return nil, err
			}
			out[i] = b
			continue
		}
		out[i] = bodies[bodyOff[i]:bodyOff[i+1]:bodyOff[i+1]]
	}
	return out, nil
}

var _ ChainIssuer = (*ChainCUDA)(nil)
