//go:build cgo && cuda

package crypto

/*
#include "afcrypto.h"
*/
import "C"

import (
	"unsafe"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// IssueCUDA issues a batch in one afc_vc_issue_execution_batch call: hashes, documents and signatures on the GPU.  The columns,
// payloads and results share one pooled pinned buffer.  Any non-zero return code sends the whole batch through IssueStdlib.
type IssueCUDA struct {
	c        *CUDA
	fallback IssueStdlib
}

func NewIssueCUDA(c *CUDA) *IssueCUDA { return &IssueCUDA{c: c} }

func (s *IssueCUDA) IssueExecutionBatch(reqs []IssueRequest, hashData bool) ([]types.ExecutionVC, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	// distinct signing keys -> expanded keys (seed || prefix || pk, afc_ed25519_expand_batch)
	keyOf := map[string]uint32{}
	var seeds []byte
	ki := make([]uint32, n)
	for i := range reqs {
		k := string(reqs[i].Key.Seed())
		j, ok := keyOf[k]
		if !ok {
			j = uint32(len(keyOf))
			keyOf[k] = j
			seeds = append(seeds, k...)
		}
		ki[i] = j
	}
	d := s.c.pick()
	exp := make([]byte, 96*len(keyOf))
	if C.afc_ed25519_expand_batch(d.ctx, (*C.uint8_t)(unsafe.Pointer(&seeds[0])), C.uint32_t(len(keyOf)), (*C.uint8_t)(unsafe.Pointer(&exp[0]))) != 0 {
		return s.fallback.IssueExecutionBatch(reqs, hashData)
	}
	defer func() {
		for i := range exp {
			exp[i] = 0
		}
	}()
	const nc = C.AFC_ISSUE_COLUMNS
	colBytes, payBytes := 0, 0
	for i := range reqs {
		r := &reqs[i]
		colBytes += len(r.VCID) + len(r.CallerDID) + len(r.IssuanceDate) + len(r.ExecutionID) + len(r.WorkflowID) + len(r.SessionID) +
			len(r.CallerType) + len(r.AgentNodeDID) + len(r.TargetDID) + len(r.FunctionName) + len(r.Timestamp) + len(r.Status) +
			len(r.ErrorMessage) + len(r.ProofCreated)
		payBytes += len(r.Input) + len(r.Output)
	}
	// layout: [col_off][pay_off][duration][key_index][nil][cols][payloads][doc_off][hashes][proof values][documents]
	oColOff := 0
	oPayOff := oColOff + align16(8*(n*nc+1))
	oDur := oPayOff + align16(8*(2*n+1))
	oKi := oDur + align16(8*n)
	oNil := oKi + align16(4*n)
	oCols := oNil + align16(2*n)
	oPay := oCols + align16(colBytes+1)
	oDocOff := oPay + align16(payBytes+1)
	oHash := oDocOff + align16(8*(n+1))
	oPV := oHash + align16(86*n)
	oDocs := oPV + align16(86*n)
	bound := 0
	{ // afc_vc_issue_bound reads only col_off[0] and col_off[14 n]: a sum over requests, so n-1 empty ones plus one of all the bytes
		one := make([]uint64, nc+1)
		fixed := int(C.afc_vc_issue_bound((*C.uint64_t)(unsafe.Pointer(&one[0])), 1))
		one[nc] = uint64(colBytes)
		bound = int(C.afc_vc_issue_bound((*C.uint64_t)(unsafe.Pointer(&one[0])), 1)) + (n-1)*fixed
	}
	p, class := d.get(oDocs + bound)
	if p == nil {
		return s.fallback.IssueExecutionBatch(reqs, hashData)
	}
	defer d.put(p, class)
	base := unsafe.Slice((*byte)(p), oDocs+bound)
	colOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oColOff])), n*nc+1)
	payOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oPayOff])), 2*n+1)
	dur := unsafe.Slice((*int64)(unsafe.Pointer(&base[oDur])), n)
	kis := unsafe.Slice((*uint32)(unsafe.Pointer(&base[oKi])), n)
	nil_ := base[oNil : oNil+2*n]
	cpos, ppos := 0, 0
	for i := range reqs {
		r := &reqs[i]
		for k, v := range [nc]string{r.VCID, r.CallerDID, r.IssuanceDate, r.ExecutionID, r.WorkflowID, r.SessionID, r.CallerType, r.AgentNodeDID,
			r.TargetDID, r.FunctionName, r.Timestamp, r.Status, r.ErrorMessage, r.ProofCreated} {
			colOff[i*nc+k] = uint64(cpos)
			cpos += copy(base[oCols+cpos:], v)
		}
		for k, pl := range [2][]byte{r.Input, r.Output} {
			payOff[2*i+k] = uint64(ppos)
			ppos += copy(base[oPay+ppos:], pl)
			nil_[2*i+k] = 0
			if pl == nil {
				nil_[2*i+k] = 1
			}
		}
		dur[i] = int64(r.DurationMS)
		kis[i] = ki[i]
	}
	colOff[n*nc] = uint64(cpos)
	payOff[2*n] = uint64(ppos)
	flags := C.uint32_t(0)
	if hashData {
		flags = C.AFC_ISSUE_HASH_DATA
	}
	u8 := func(o int) *C.uint8_t { return (*C.uint8_t)(unsafe.Pointer(&base[o])) }
	u64 := func(o int) *C.uint64_t { return (*C.uint64_t)(unsafe.Pointer(&base[o])) }
	rc := C.afc_vc_issue_execution_batch(d.ctx, (*C.uint8_t)(unsafe.Pointer(&exp[0])), C.uint32_t(len(keyOf)), (*C.uint32_t)(unsafe.Pointer(&base[oKi])),
		u8(oCols), u64(oColOff), (*C.int64_t)(unsafe.Pointer(&base[oDur])), u8(oPay), u64(oPayOff), u8(oNil), flags, C.uint32_t(n), nil,
		u8(oDocs), C.uint64_t(bound), u64(oDocOff), u8(oHash), u8(oPV))
	if rc != 0 {
		return s.fallback.IssueExecutionBatch(reqs, hashData)
	}
	docOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oDocOff])), n+1)
	out := make([]types.ExecutionVC, n)
	for i := range reqs {
		var ih, oh string
		if hashData {
			ih, oh = string(base[oHash+86*i:oHash+86*i+43]), string(base[oHash+86*i+43:oHash+86*i+86])
		}
		doc := append([]byte(nil), base[oDocs+int(docOff[i]):oDocs+int(docOff[i+1])]...)
		out[i] = storedRecord(&reqs[i], doc, string(base[oPV+86*i:oPV+86*i+86]), ih, oh)
	}
	return out, nil
}

var _ Issuer = (*IssueCUDA)(nil)
