//go:build cgo && cuda

package crypto

/*
#include <stdlib.h>
#include "afcrypto.h"
*/
import "C"

import (
	"crypto/ed25519"
	"encoding/json"
	"fmt"
	"unsafe"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// StoredCUDA verifies stored documents on the GPU against a key set that knows its issuers' DIDs
// (afc_keyset_new_named).  Documents the device cannot prove to be in json.Marshal's exact form (AFC_VC_HOST), and every
// document of a batch whose call fails, go through StoredStdlib: the answers never differ from the reference's.
type StoredCUDA struct {
	ctx  *C.afc_ctx
	ks   *C.afc_keyset
	dids []string
	keys map[string]ed25519.PublicKey
}

// NewStoredCUDA registers the issuers (DID -> public key) on the context's GPU.
func NewStoredCUDA(c *CUDA, issuers map[string]ed25519.PublicKey) (*StoredCUDA, error) {
	if len(c.devs) == 0 || len(issuers) == 0 {
		return nil, fmt.Errorf("crypto: no device or no issuers")
	}
	s := &StoredCUDA{ctx: c.devs[0].ctx, keys: issuers}
	pks := make([]byte, 0, 32*len(issuers))
	var dids []byte
	off := []uint64{0}
	for did, pk := range issuers {
		if len(pk) != ed25519.PublicKeySize {
			return nil, fmt.Errorf("crypto: bad public key length for %s", did)
		}
		s.dids = append(s.dids, did)
		pks = append(pks, pk...)
		dids = append(dids, did...)
		off = append(off, uint64(len(dids)))
	}
	dids = append(dids, 0)
	rc := C.afc_keyset_new_named(s.ctx, (*C.uint8_t)(unsafe.Pointer(&pks[0])), (*C.uint8_t)(unsafe.Pointer(&dids[0])),
		(*C.uint64_t)(unsafe.Pointer(&off[0])), C.uint32_t(len(issuers)), &s.ks)
	if rc != 0 {
		return nil, fmt.Errorf("crypto: afc_keyset_new_named: %s", C.GoString(C.afc_strerror(rc)))
	}
	return s, nil
}

func (s *StoredCUDA) Close() { C.afc_keyset_free(s.ks) }

func (s *StoredCUDA) VerifyStoredBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error) {
	return s.verifyBatch(kind, docs, resolve, false)
}

// VerifyJSONBatch is VerifyVC for documents as clients send them (request bodies of POST /api/v1/did/verify, files given to
// `af vc verify`), in any JSON spelling: the device re-marshals them (afc_vc_verify_json_batch).  Documents it leaves to the
// host go through verifyStoredOne, which handles any spelling.
func (s *StoredCUDA) VerifyJSONBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error) {
	return s.verifyBatch(kind, docs, resolve, true)
}

func (s *StoredCUDA) verifyBatch(kind DocKind, docs []json.RawMessage, resolve Resolver, anySpelling bool) ([]types.VCVerificationResponse, error) {
	n := len(docs)
	if n == 0 {
		return nil, nil
	}
	total := 0
	for _, d := range docs {
		total += len(d)
	}
	buf := C.malloc(C.size_t(total + 1))
	off := C.malloc(C.size_t(8 * (n + 1)))
	status := C.malloc(C.size_t(n))
	fields := C.malloc(C.size_t(16 * n))
	defer C.free(buf)
	defer C.free(off)
	defer C.free(status)
	defer C.free(fields)
	b := unsafe.Slice((*byte)(buf), total+1)
	o := unsafe.Slice((*uint64)(off), n+1)
	pos := 0
	for i, d := range docs {
		o[i] = uint64(pos)
		pos += copy(b[pos:], d)
	}
	o[n] = uint64(pos)
	var rc C.int
	if anySpelling {
		rc = C.afc_vc_verify_json_batch(s.ctx, s.ks, C.int(kind), (*C.uint8_t)(buf), (*C.uint64_t)(off), C.uint32_t(n),
			(*C.uint8_t)(status), (*C.uint32_t)(fields))
	} else {
		rc = C.afc_vc_verify_stored_batch(s.ctx, s.ks, C.int(kind), (*C.uint8_t)(buf), (*C.uint64_t)(off), C.uint32_t(n),
			(*C.uint8_t)(status), (*C.uint32_t)(fields))
	}
	if rc != 0 {
		if anySpelling {
			observeFallback("verify_json")
		} else {
			observeFallback("verify_stored")
		}
		return StoredStdlib{}.VerifyStoredBatch(kind, docs, resolve)
	}
	st := unsafe.Slice((*byte)(status), n)
	f := unsafe.Slice((*uint32)(fields), 4*n)
	out := make([]types.VCVerificationResponse, n)
	for i, d := range docs {
		switch st[i] {
		case C.AFC_VC_VALID:
			var issued string
			_ = json.Unmarshal(d[f[4*i+2]-1:f[4*i+2]+f[4*i+3]+1], &issued) // the JSON string, quotes included
			out[i] = types.VCVerificationResponse{Valid: true, IssuerDID: string(d[f[4*i] : f[4*i]+f[4*i+1]]), IssuedAt: issued,
				Message: "VC verified successfully"}
		case C.AFC_VC_INVALID:
			out[i] = types.VCVerificationResponse{Valid: false, Message: "Invalid signature"}
		default: // HOST, and the error statuses, whose messages carry Go's own error text
			out[i] = verifyStoredOne(kind, d, resolve)
		}
	}
	return out, nil
}

// StoredAuditCUDA audits stored execution VCs on the GPU (afc_vc_audit_stored_batch) against the same named key set.
// Credentials the device leaves to the host (AFC_VC_HOST) or whose mask holds an undecided bit, and every credential of a
// batch whose call fails, go through StoredAuditStdlib.
type StoredAuditCUDA struct{ *StoredCUDA }

func (s StoredAuditCUDA) AuditStoredBatch(vcs []types.ExecutionVC, resolve Resolver) ([]AuditResult, error) {
	n := len(vcs)
	if n == 0 {
		return nil, nil
	}
	total, ctotal := 0, 0
	for i := range vcs {
		v := &vcs[i]
		total += len(v.VCDocument)
		for _, c := range auditColumns(v) {
			ctotal += len(c)
		}
	}
	buf := C.malloc(C.size_t(total + 1))
	off := C.malloc(C.size_t(8 * (n + 1)))
	cols := C.malloc(C.size_t(ctotal + 1))
	coff := C.malloc(C.size_t(8 * (C.AFC_AUDIT_COLUMNS*n + 1)))
	status := C.malloc(C.size_t(n))
	issues := C.malloc(C.size_t(4 * n))
	for _, p := range []unsafe.Pointer{buf, off, cols, coff, status, issues} {
		defer C.free(p)
	}
	b := unsafe.Slice((*byte)(buf), total+1)
	o := unsafe.Slice((*uint64)(off), n+1)
	cb := unsafe.Slice((*byte)(cols), ctotal+1)
	co := unsafe.Slice((*uint64)(coff), C.AFC_AUDIT_COLUMNS*n+1)
	pos, cpos, k := 0, 0, 0
	for i := range vcs {
		o[i] = uint64(pos)
		pos += copy(b[pos:], vcs[i].VCDocument)
		for _, c := range auditColumns(&vcs[i]) {
			co[k] = uint64(cpos)
			cpos += copy(cb[cpos:], c)
			k++
		}
	}
	o[n], co[k] = uint64(pos), uint64(cpos)
	rc := C.afc_vc_audit_stored_batch(s.ctx, s.ks, C.AFC_DOC_EXECUTION_VC, (*C.uint8_t)(buf), (*C.uint64_t)(off), (*C.uint8_t)(cols),
		(*C.uint64_t)(coff), C.uint32_t(n), (*C.uint8_t)(status), (*C.uint32_t)(issues))
	if rc != 0 {
		observeFallback("audit_stored")
		return StoredAuditStdlib{}.AuditStoredBatch(vcs, resolve)
	}
	st := unsafe.Slice((*byte)(status), n)
	is := unsafe.Slice((*uint32)(issues), n)
	out := make([]AuditResult, n)
	for i := range vcs {
		if st[i] == C.AFC_VC_HOST || is[i]&(AuditStatusUndecided|AuditTimestampUndecided) != 0 {
			out[i] = auditStoredOne(&vcs[i], resolve)
			continue
		}
		out[i] = AuditResult{Status: st[i], Issues: is[i]}
	}
	return out, nil
}

// the record's columns in the order of AFC_AUDIT_COLUMNS
func auditColumns(v *types.ExecutionVC) [10]string {
	return [10]string{v.IssuerDID, v.ExecutionID, v.WorkflowID, v.SessionID, v.CallerDID, v.TargetDID, v.Status, v.InputHash, v.OutputHash, v.Signature}
}
