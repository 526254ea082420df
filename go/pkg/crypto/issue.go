package crypto

import (
	"crypto/ed25519"
	"crypto/sha256"
	"encoding/base64"
	"encoding/json"
	"fmt"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// IssueRequest is one GenerateExecutionVC call (internal/services/vc_service.go:138-239) with the values the reference reads from a
// clock or makes up passed in: the VC id, issuanceDate, the proof's created and the execution timestamp (RFC 3339 strings).
type IssueRequest struct {
	VCID, CallerDID, IssuanceDate, ExecutionID, WorkflowID, SessionID string
	CallerType, AgentNodeDID, TargetDID, FunctionName, Timestamp      string
	Status, ErrorMessage, ProofCreated                                string // ErrorMessage: untruncated, "" = none
	DurationMS                                                         int
	Input, Output                                                      []byte // nil hashes as null
	Key                                                                ed25519.PrivateKey
}

// Issuer issues execution credentials: the stored document, its signature and both hashes, exactly as GenerateExecutionVC
// computes and stores them.  hashData: VCRequirements.HashSensitiveData (without it both hashes are "").
type Issuer interface {
	IssueExecutionBatch(reqs []IssueRequest, hashData bool) ([]types.ExecutionVC, error)
}

var _ Issuer = IssueStdlib{}

// IssueStdlib is the reference's own path, one request at a time: createVCDocument, signVC, json.Marshal.
type IssueStdlib struct{}

func (IssueStdlib) IssueExecutionBatch(reqs []IssueRequest, hashData bool) ([]types.ExecutionVC, error) {
	out := make([]types.ExecutionVC, len(reqs))
	for i := range reqs {
		vc, err := issueOne(&reqs[i], hashData)
		if err != nil {
			return nil, err
		}
		out[i] = vc
	}
	return out, nil
}

func hashDataOf(data []byte) string { // hashData(marshalDataOrNull(data)), vc_service.go:508-515, 1297-1306
	b, _ := json.Marshal(data) // nil -> null, else the std-base64 text in quotes
	h := sha256.Sum256(b)
	return base64.RawURLEncoding.EncodeToString(h[:])
}

func issueOne(r *IssueRequest, hashData bool) (types.ExecutionVC, error) {
	var ih, oh string
	if hashData {
		ih, oh = hashDataOf(r.Input), hashDataOf(r.Output)
	}
	msg := r.ErrorMessage
	if len(msg) > 500 {
		msg = msg[:500] + "...[truncated]"
	}
	doc := types.VCDocument{
		Context: []string{"https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/execution/v1"},
		Type:    []string{"VerifiableCredential", "AgentFieldExecutionCredential"},
		ID:      fmt.Sprintf("urn:agentfield:vc:%s", r.VCID), Issuer: r.CallerDID, IssuanceDate: r.IssuanceDate,
		CredentialSubject: types.VCCredentialSubject{
			ExecutionID: r.ExecutionID, WorkflowID: r.WorkflowID, SessionID: r.SessionID,
			Caller:      types.VCCaller{DID: r.CallerDID, Type: r.CallerType, AgentNodeDID: r.AgentNodeDID},
			Target:      types.VCTarget{DID: r.TargetDID, AgentNodeDID: r.AgentNodeDID, FunctionName: r.FunctionName},
			Execution: types.VCExecution{InputHash: ih, OutputHash: oh, Timestamp: r.Timestamp, DurationMS: r.DurationMS, Status: r.Status,
				ErrorMessage: msg},
			Audit: types.VCAudit{InputDataHash: ih, OutputDataHash: oh,
				Metadata: map[string]interface{}{"agentfield_version": "1.0.0", "vc_version": "1.0"}},
		},
	}
	canonical, err := json.Marshal(doc) // signVC: the zero-valued proof
	if err != nil {
		return types.ExecutionVC{}, err
	}
	sig := base64.RawURLEncoding.EncodeToString(ed25519.Sign(r.Key, canonical))
	doc.Proof = types.VCProof{Type: "Ed25519Signature2020", Created: r.ProofCreated, VerificationMethod: r.CallerDID + "#key-1",
		ProofPurpose: "assertionMethod", ProofValue: sig}
	stored, err := json.Marshal(doc)
	if err != nil {
		return types.ExecutionVC{}, err
	}
	return storedRecord(r, stored, sig, ih, oh), nil
}

// the ExecutionVC record GenerateExecutionVC stores (vc_service.go:206-227); CreatedAt and the status normalisation are the caller's
func storedRecord(r *IssueRequest, doc []byte, sig, ih, oh string) types.ExecutionVC {
	return types.ExecutionVC{VCID: r.VCID, ExecutionID: r.ExecutionID, WorkflowID: r.WorkflowID, SessionID: r.SessionID, IssuerDID: r.CallerDID,
		TargetDID: r.TargetDID, CallerDID: r.CallerDID, VCDocument: json.RawMessage(doc), Signature: sig, DocumentSize: int64(len(doc)),
		InputHash: ih, OutputHash: oh, Status: r.Status}
}
