//go:build cgo && cuda

package crypto

/*
#include "afcrypto.h"
*/
import "C"

import (
	"time"
	"unsafe"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// WorkflowCUDA issues a batch of workflow credentials in one afc_vc_issue_workflow_batch call.  Any non-zero return code sends the whole
// batch through WorkflowStdlib, and so does each workflow the device marks AFC_WORKFLOW_HOST (a status that is not printable ASCII, a
// time RFC 3339 cannot write in four digits).
type WorkflowCUDA struct {
	c        *CUDA
	fallback WorkflowStdlib
}

func NewWorkflowCUDA(c *CUDA) *WorkflowCUDA { return &WorkflowCUDA{c: c} }

var workflowStatusNames = [8]string{"unknown", "pending", "queued", "running", "succeeded", "failed", "cancelled", "timeout"}

func (s *WorkflowCUDA) IssueWorkflowBatch(reqs []WorkflowRequest) ([]types.WorkflowVC, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	keyOf := map[string]uint32{}
	var seeds []byte
	ki := make([]uint32, n)
	m, colBytes, recBytes := 0, 0, 0
	for i := range reqs {
		r := &reqs[i]
		k := string(r.Key.Seed())
		j, ok := keyOf[k]
		if !ok {
			j = uint32(len(keyOf))
			keyOf[k] = j
			seeds = append(seeds, k...)
		}
		ki[i] = j
		session := ""
		if len(r.Records) > 0 {
			session = r.Records[0].SessionID
		}
		colBytes += len(r.WorkflowID) + len(session) + len(workflowIssuer(r)) + len(r.VCID) + len(r.IssuanceDate) + len(r.SnapshotText) + len(r.ProofCreated)
		for _, vc := range r.Records {
			recBytes += len(vc.VCID) + len(vc.Status)
		}
		m += len(r.Records)
	}
	d := s.c.pick()
	exp := make([]byte, 96*len(keyOf))
	if C.afc_ed25519_expand_batch(d.ctx, (*C.uint8_t)(unsafe.Pointer(&seeds[0])), C.uint32_t(len(keyOf)), (*C.uint8_t)(unsafe.Pointer(&exp[0]))) != 0 {
		return s.fallback.IssueWorkflowBatch(reqs)
	}
	defer func() {
		for i := range exp {
			exp[i] = 0
		}
	}()
	const nc = C.AFC_WORKFLOW_COLUMNS
	// layout: [col_off][rec_off][rec_col_off][created_at][key_index][state][summary][cols][rec_cols][doc_off][proof values][documents]
	oColOff := 0
	oRecOff := oColOff + align16(8*(n*nc+1))
	oRecColOff := oRecOff + align16(8*(n+1))
	oCreated := oRecColOff + align16(8*(2*m+1))
	oKi := oCreated + align16(16*m)
	oState := oKi + align16(4*n)
	oSum := oState + align16(n)
	oCols := oSum + align16(16*n)
	oRecCols := oCols + align16(colBytes+1)
	oDocOff := oRecCols + align16(recBytes+1)
	oPV := oDocOff + align16(8*(n+1))
	oDocs := oPV + align16(86*n)
	// afc_vc_workflow_bound is linear in the workflow count, column bytes, records and record bytes: read its coefficients off one workflow
	bound := 0
	{
		co := make([]uint64, nc+1)
		ro := []uint64{0, 0}
		rco := []uint64{0, 0, 0}
		f := func() int {
			return int(C.afc_vc_workflow_bound((*C.uint64_t)(unsafe.Pointer(&co[0])), (*C.uint64_t)(unsafe.Pointer(&ro[0])),
				(*C.uint64_t)(unsafe.Pointer(&rco[0])), 1))
		}
		fixed := f()
		co[nc] = 1
		perCol := f() - fixed
		co[nc], ro[1] = 0, 1
		perRec := f() - fixed
		rco[2] = 1
		perRecByte := f() - fixed - perRec
		bound = n*fixed + perCol*colBytes + perRec*m + perRecByte*recBytes
	}
	p, class := d.get(oDocs + bound)
	if p == nil {
		return s.fallback.IssueWorkflowBatch(reqs)
	}
	defer d.put(p, class)
	base := unsafe.Slice((*byte)(p), oDocs+bound)
	colOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oColOff])), n*nc+1)
	recOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oRecOff])), n+1)
	recColOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oRecColOff])), 2*m+1)
	created := unsafe.Slice((*int64)(unsafe.Pointer(&base[oCreated])), 2*m)
	kis := unsafe.Slice((*uint32)(unsafe.Pointer(&base[oKi])), n)
	cpos, rpos, r := 0, 0, 0
	for i := range reqs {
		q := &reqs[i]
		session := ""
		if len(q.Records) > 0 {
			session = q.Records[0].SessionID
		}
		for k, v := range [nc]string{q.WorkflowID, session, workflowIssuer(q), q.VCID, q.IssuanceDate, q.SnapshotText, q.ProofCreated} {
			colOff[i*nc+k] = uint64(cpos)
			cpos += copy(base[oCols+cpos:], v)
		}
		recOff[i] = uint64(r)
		for _, vc := range q.Records {
			recColOff[2*r] = uint64(rpos)
			rpos += copy(base[oRecCols+rpos:], vc.VCID)
			recColOff[2*r+1] = uint64(rpos)
			rpos += copy(base[oRecCols+rpos:], vc.Status)
			created[2*r], created[2*r+1] = vc.CreatedAt.Unix(), int64(vc.CreatedAt.Nanosecond())
			r++
		}
		kis[i] = ki[i]
	}
	colOff[n*nc] = uint64(cpos)
	recOff[n] = uint64(r)
	recColOff[2*m] = uint64(rpos)
	u8 := func(o int) *C.uint8_t { return (*C.uint8_t)(unsafe.Pointer(&base[o])) }
	u64 := func(o int) *C.uint64_t { return (*C.uint64_t)(unsafe.Pointer(&base[o])) }
	rc := C.afc_vc_issue_workflow_batch(d.ctx, (*C.uint8_t)(unsafe.Pointer(&exp[0])), C.uint32_t(len(keyOf)), (*C.uint32_t)(unsafe.Pointer(&base[oKi])),
		u8(oCols), u64(oColOff), u64(oRecOff), u8(oRecCols), u64(oRecColOff), (*C.int64_t)(unsafe.Pointer(&base[oCreated])), C.uint32_t(n),
		u8(oDocs), C.uint64_t(bound), u64(oDocOff), u8(oPV), u8(oState), (*C.uint32_t)(unsafe.Pointer(&base[oSum])))
	if rc != 0 {
		return s.fallback.IssueWorkflowBatch(reqs)
	}
	docOff := unsafe.Slice((*uint64)(unsafe.Pointer(&base[oDocOff])), n+1)
	summary := unsafe.Slice((*uint32)(unsafe.Pointer(&base[oSum])), 4*n)
	out := make([]types.WorkflowVC, n)
	for i := range reqs {
		q := &reqs[i]
		if base[oState+i] != C.AFC_WORKFLOW_BUILT {
			vc, err := workflowOne(q)
			if err != nil {
				return nil, err
			}
			out[i] = vc
			continue
		}
		start := q.SnapshotTime // the full-precision times come from the records the call names
		var end *time.Time
		if len(q.Records) > 0 {
			start = q.Records[summary[4*i+2]].CreatedAt
		}
		if e := summary[4*i+3]; e != 0xFFFFFFFF {
			t := q.Records[e].CreatedAt
			end = &t
		}
		doc := append([]byte(nil), base[oDocs+int(docOff[i]):oDocs+int(docOff[i+1])]...)
		out[i] = workflowRecord(q, workflowStatusNames[summary[4*i]&7], start, end, doc, string(base[oPV+86*i:oPV+86*i+86]))
	}
	return out, nil
}

var _ WorkflowIssuer = (*WorkflowCUDA)(nil)
