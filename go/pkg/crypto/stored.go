package crypto

import (
	"crypto/ed25519"
	"encoding/base64"
	"encoding/json"
	"fmt"
	"strings"
	"time"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// DocKind names the struct a stored document is the json.Marshal of.
type DocKind int

const (
	ExecutionVC DocKind = 0 // types.VCDocument
	WorkflowVC  DocKind = 1 // types.WorkflowVCDocument
)

// Resolver returns the issuer's public key, or an error worded as DIDService.ResolveDID words it.
type Resolver func(did string) (ed25519.PublicKey, error)

// StoredVerifier verifies stored credential documents from their bytes and answers exactly what VCService.VerifyVC
// (internal/services/vc_service.go:242-289) answers for each: parse, resolve the issuer, decode the signature, verify.
// VerifyStoredBatch is for documents as the control plane stores them (json.Marshal's form); VerifyJSONBatch for documents in
// any JSON spelling (request bodies, files).  Both answer the same; they differ in which documents the GPU form can take.
type StoredVerifier interface {
	VerifyStoredBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error)
	VerifyJSONBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error)
}

// StoredStdlib is the reference's own path, one document at a time: Unmarshal, zero the proof, Marshal, Verify.
type StoredStdlib struct{}

func (StoredStdlib) VerifyStoredBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error) {
	out := make([]types.VCVerificationResponse, len(docs))
	for i, d := range docs {
		out[i] = verifyStoredOne(kind, d, resolve)
	}
	return out, nil
}

// VerifyJSONBatch is VerifyVC for documents as clients send them, in any JSON spelling; the stdlib path is the same
// Unmarshal -> Marshal -> Verify, which does not depend on the spelling.
func (StoredStdlib) VerifyJSONBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error) {
	return StoredStdlib{}.VerifyStoredBatch(kind, docs, resolve)
}

func verifyStoredOne(kind DocKind, doc json.RawMessage, resolve Resolver) types.VCVerificationResponse {
	var issuer, issued, proofValue string
	var canonical []byte
	var err error
	switch kind {
	case ExecutionVC:
		var v types.VCDocument
		if err = json.Unmarshal(doc, &v); err != nil {
			return types.VCVerificationResponse{Valid: false, Error: fmt.Sprintf("failed to parse VC document: %v", err)}
		}
		issuer, issued, proofValue = v.Issuer, v.IssuanceDate, v.Proof.ProofValue
		v.Proof = types.VCProof{}
		canonical, err = json.Marshal(v)
	case WorkflowVC:
		var v types.WorkflowVCDocument
		if err = json.Unmarshal(doc, &v); err != nil {
			return types.VCVerificationResponse{Valid: false, Error: fmt.Sprintf("failed to parse VC document: %v", err)}
		}
		issuer, issued, proofValue = v.Issuer, v.IssuanceDate, v.Proof.ProofValue
		v.Proof = types.VCProof{}
		canonical, err = json.Marshal(v)
	default:
		return types.VCVerificationResponse{Valid: false, Error: "unknown document kind"}
	}
	pk, rerr := resolve(issuer)
	if rerr != nil {
		return types.VCVerificationResponse{Valid: false, Error: fmt.Sprintf("failed to resolve issuer DID: %v", rerr)}
	}
	if err != nil {
		return types.VCVerificationResponse{Valid: false, Error: fmt.Sprintf("failed to verify signature: failed to marshal VC for verification: %v", err)}
	}
	sig, err := base64.RawURLEncoding.DecodeString(proofValue)
	if err != nil {
		return types.VCVerificationResponse{Valid: false, Error: fmt.Sprintf("failed to verify signature: failed to decode signature: %v", err)}
	}
	if !ed25519.Verify(pk, canonical, sig) {
		return types.VCVerificationResponse{Valid: false, Message: "Invalid signature"}
	}
	return types.VCVerificationResponse{Valid: true, IssuerDID: issuer, IssuedAt: issued, Message: "VC verified successfully"}
}

// Audit bits of one credential against its record (include/afcrypto.h AFC_AUDIT_*).  Bits 0-9: the record's column differs
// from the document's member, in the order of auditColumns.
const (
	AuditIssuerMismatch uint32 = 1 << iota
	AuditExecutionIDMismatch
	AuditWorkflowIDMismatch
	AuditSessionIDMismatch
	AuditCallerDIDMismatch
	AuditTargetDIDMismatch
	AuditStatusMismatch
	AuditInputHashMismatch
	AuditOutputHashMismatch
	AuditSignatureMismatch
	AuditInvalidTimestamp
	AuditMissingContext
	AuditMissingType
	AuditMissingID
	AuditMissingIssuer
	AuditMissingIssuanceDate
	AuditNotW3C
	AuditNotAgentField
	AuditStatusUndecided    // device only: the status comparison is left to the stdlib form
	AuditTimestampUndecided // device only: the timestamp rule is left to the stdlib form
)

// Audit statuses: those of afc_vc_verify_stored_batch (AFC_VC_*), plus AuditParseError where json.Unmarshal fails (the
// reference's early parse_error result, vc_service.go:966-977).
const (
	AuditInvalid     uint8 = 0
	AuditValid       uint8 = 1
	AuditHost        uint8 = 2 // device only: not provably canonical, finished by the stdlib form
	AuditUnresolved  uint8 = 3
	AuditBadEncoding uint8 = 4
	AuditParseError  uint8 = 5
)

// AuditResult is what VerifyExecutionVCComprehensive decides for one credential, before it builds the VerificationIssues:
// the signature check (Status) and the mismatches and rule failures (Issues).
type AuditResult struct {
	Status uint8
	Issues uint32
}

// StoredAuditor audits stored execution VCs against their records: the checks of performIntegrityChecks,
// performSecurityAnalysis and performComplianceChecks (internal/services/vc_service.go:1008-1359) for each credential.
type StoredAuditor interface {
	AuditStoredBatch(vcs []types.ExecutionVC, resolve Resolver) ([]AuditResult, error)
}

// StoredAuditStdlib is the reference's own path, one credential at a time.
type StoredAuditStdlib struct{}

func (StoredAuditStdlib) AuditStoredBatch(vcs []types.ExecutionVC, resolve Resolver) ([]AuditResult, error) {
	out := make([]AuditResult, len(vcs))
	for i := range vcs {
		out[i] = auditStoredOne(&vcs[i], resolve)
	}
	return out, nil
}

func auditStoredOne(vc *types.ExecutionVC, resolve Resolver) AuditResult {
	var d types.VCDocument
	if err := json.Unmarshal(vc.VCDocument, &d); err != nil {
		return AuditResult{Status: AuditParseError}
	}
	var r AuditResult
	cs := d.CredentialSubject
	for k, p := range [10][2]string{{vc.IssuerDID, d.Issuer}, {vc.ExecutionID, cs.ExecutionID}, {vc.WorkflowID, cs.WorkflowID},
		{vc.SessionID, cs.SessionID}, {vc.CallerDID, cs.Caller.DID}, {vc.TargetDID, cs.Target.DID}, {"", ""},
		{vc.InputHash, cs.Execution.InputHash}, {vc.OutputHash, cs.Execution.OutputHash}, {vc.Signature, d.Proof.ProofValue}} {
		if p[0] != p[1] {
			r.Issues |= 1 << k
		}
	}
	if types.NormalizeExecutionStatus(vc.Status) != types.NormalizeExecutionStatus(cs.Execution.Status) {
		r.Issues |= AuditStatusMismatch
	}
	if _, err := time.Parse(time.RFC3339, d.IssuanceDate); err != nil {
		r.Issues |= AuditInvalidTimestamp
	}
	for _, m := range []struct {
		missing bool
		bit     uint32
	}{{len(d.Context) == 0, AuditMissingContext}, {len(d.Type) == 0, AuditMissingType}, {d.ID == "", AuditMissingID},
		{d.Issuer == "", AuditMissingIssuer}, {d.IssuanceDate == "", AuditMissingIssuanceDate}} {
		if m.missing {
			r.Issues |= m.bit
		}
	}
	if !contains(d.Context, "https://www.w3.org/2018/credentials/v1") {
		r.Issues |= AuditNotW3C
	}
	if !contains(d.Type, "VerifiableCredential") || !contains(d.Type, "AgentFieldExecutionCredential") {
		r.Issues |= AuditNotAgentField
	}
	v := verifyStoredOne(ExecutionVC, vc.VCDocument, resolve)
	switch {
	case v.Valid:
		r.Status = AuditValid
	case v.Error == "":
		r.Status = AuditInvalid
	case strings.HasPrefix(v.Error, "failed to resolve issuer DID"):
		r.Status = AuditUnresolved
	default:
		r.Status = AuditBadEncoding
	}
	return r
}

func contains(list []string, s string) bool {
	for _, x := range list {
		if x == s {
			return true
		}
	}
	return false
}
