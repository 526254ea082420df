package crypto

import (
	"crypto/ed25519"
	"encoding/base64"
	"encoding/json"
	"fmt"
	"time"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// WorkflowRequest is one generateWorkflowVCDocument call (internal/services/vc_service.go:525-632) with the values the reference reads
// from a clock or makes up passed in: the document's VC id, issuanceDate, snapshotTime, the proof's created, the WorkflowVC record's id
// and SnapshotTime.  Records are the workflow's ExecutionVCs in GetExecutionVCsByWorkflow order; RootDID is the issuer when there are
// none.  Key is the issuer's signing key (records[0].IssuerDID's, or RootDID's).
type WorkflowRequest struct {
	WorkflowID                                     string
	Records                                        []types.ExecutionVC
	RootDID                                        string
	VCID, IssuanceDate, SnapshotText, ProofCreated string // SnapshotText: time.Now().UTC().Format(time.RFC3339), also startTime without records
	WorkflowVCID                                   string
	SnapshotTime                                   time.Time
	Key                                            ed25519.PrivateKey
}

// WorkflowIssuer issues workflow credentials exactly as generateWorkflowVCDocument builds and signs them.
type WorkflowIssuer interface {
	IssueWorkflowBatch(reqs []WorkflowRequest) ([]types.WorkflowVC, error)
}

var _ WorkflowIssuer = WorkflowStdlib{}

// WorkflowStdlib is the reference's own path, one workflow at a time.
type WorkflowStdlib struct{}

func (WorkflowStdlib) IssueWorkflowBatch(reqs []WorkflowRequest) ([]types.WorkflowVC, error) {
	out := make([]types.WorkflowVC, len(reqs))
	for i := range reqs {
		vc, err := workflowOne(&reqs[i])
		if err != nil {
			return nil, err
		}
		out[i] = vc
	}
	return out, nil
}

func workflowIssuer(r *WorkflowRequest) string {
	if len(r.Records) > 0 {
		return r.Records[0].IssuerDID
	}
	return r.RootDID
}

// workflowStatus is determineWorkflowStatus (vc_service.go:721-772)
func workflowStatus(recs []types.ExecutionVC) string {
	if len(recs) == 0 {
		return string(types.ExecutionStatusPending)
	}
	seen := map[string]bool{}
	for _, vc := range recs {
		seen[types.NormalizeExecutionStatus(vc.Status)] = true
	}
	for _, s := range []types.ExecutionStatus{types.ExecutionStatusFailed, types.ExecutionStatusTimeout, types.ExecutionStatusCancelled,
		types.ExecutionStatusRunning, types.ExecutionStatusQueued, types.ExecutionStatusPending, types.ExecutionStatusUnknown} {
		if seen[string(s)] {
			return string(s)
		}
	}
	return string(types.ExecutionStatusSucceeded)
}

func completedSteps(recs []types.ExecutionVC) int { // countCompletedSteps (vc_service.go:775-787)
	n := 0
	for _, vc := range recs {
		if types.NormalizeExecutionStatus(vc.Status) == string(types.ExecutionStatusSucceeded) {
			n++
		}
	}
	return n
}

// workflowRecord is the WorkflowVC generateWorkflowVCDocument returns (vc_service.go:613-629), its times taken from the records
func workflowRecord(r *WorkflowRequest, status string, start time.Time, end *time.Time, doc []byte, sig string) types.WorkflowVC {
	ids := make([]string, len(r.Records))
	for i, vc := range r.Records {
		ids[i] = vc.VCID
	}
	session := ""
	if len(r.Records) > 0 {
		session = r.Records[0].SessionID
	}
	return types.WorkflowVC{WorkflowID: r.WorkflowID, SessionID: session, ComponentVCs: ids, WorkflowVCID: r.WorkflowVCID, Status: status,
		StartTime: start, EndTime: end, TotalSteps: len(r.Records), CompletedSteps: completedSteps(r.Records), VCDocument: json.RawMessage(doc),
		Signature: sig, IssuerDID: workflowIssuer(r), SnapshotTime: r.SnapshotTime, DocumentSize: int64(len(doc))}
}

// workflowOne is generateWorkflowVCDocument with the clock values passed in.  Without records startTime is SnapshotText (the reference
// reads time.Now() there); StartTime in the record is then SnapshotTime.
func workflowOne(r *WorkflowRequest) (types.WorkflowVC, error) {
	status := workflowStatus(r.Records)
	ids := make([]string, len(r.Records))
	for i, vc := range r.Records {
		ids[i] = vc.VCID
	}
	session := ""
	start, startText := r.SnapshotTime, r.SnapshotText
	var end *time.Time
	if len(r.Records) > 0 {
		session = r.Records[0].SessionID
		start = r.Records[0].CreatedAt
		latest := r.Records[0].CreatedAt
		for _, vc := range r.Records {
			if vc.CreatedAt.Before(start) {
				start = vc.CreatedAt
			}
			if vc.CreatedAt.After(latest) {
				latest = vc.CreatedAt
			}
		}
		if types.IsTerminalExecutionStatus(status) {
			end = &latest
		}
		startText = start.UTC().Format(time.RFC3339)
	}
	issuer := workflowIssuer(r)
	cs := types.WorkflowVCCredentialSubject{WorkflowID: r.WorkflowID, SessionID: session, ComponentVCIDs: ids, TotalSteps: len(ids),
		CompletedSteps: len(ids), Status: status, StartTime: startText, SnapshotTime: r.SnapshotText,
		Orchestrator: types.VCCaller{DID: issuer, Type: "agentfield_server", AgentNodeDID: issuer},
		Audit: types.VCAudit{Metadata: map[string]interface{}{"agentfield_version": "1.0.0", "vc_version": "1.0",
			"workflow_type": "agent_execution_chain", "total_executions": len(ids)}}}
	if end != nil {
		e := end.UTC().Format(time.RFC3339)
		cs.EndTime = &e
	}
	doc := types.WorkflowVCDocument{
		Context: []string{"https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/workflow/v1"},
		Type:    []string{"VerifiableCredential", "AgentFieldWorkflowCredential"},
		ID:      fmt.Sprintf("urn:agentfield:workflow-vc:%s", r.VCID), Issuer: issuer, IssuanceDate: r.IssuanceDate, CredentialSubject: cs,
	}
	canonical, err := json.Marshal(doc) // signWorkflowVC: the zero-valued proof
	if err != nil {
		return types.WorkflowVC{}, err
	}
	sig := base64.RawURLEncoding.EncodeToString(ed25519.Sign(r.Key, canonical))
	doc.Proof = types.VCProof{Type: "Ed25519Signature2020", Created: r.ProofCreated, VerificationMethod: issuer + "#key-1",
		ProofPurpose: "assertionMethod", ProofValue: sig}
	stored, err := json.Marshal(doc)
	if err != nil {
		return types.WorkflowVC{}, err
	}
	return workflowRecord(r, status, start, end, stored, sig), nil
}
