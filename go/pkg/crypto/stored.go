package crypto

import (
	"crypto/ed25519"
	"encoding/base64"
	"encoding/json"
	"fmt"

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
type StoredVerifier interface {
	VerifyStoredBatch(kind DocKind, docs []json.RawMessage, resolve Resolver) ([]types.VCVerificationResponse, error)
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
