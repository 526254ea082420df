package crypto

import (
	"encoding/base64"
	"encoding/json"
	"strings"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// ChainRequest is one GetWorkflowVCChain (internal/services/vc_service.go:292-338) after the storage read: the workflow credential's
// inputs, and ResolvedAt, the text collectDIDResolutionBundle (:810-870) reads from the clock (time.Now().UTC().Format(time.RFC3339)).
type ChainRequest struct {
	WorkflowRequest
	ResolvedAt string
}

// PublicJWK is ed25519PublicKeyToJWK's text of a public key: what the registry stores for every DID the reference registers, and so
// what collectDIDResolutionBundle embeds (after the compaction json.Marshal applies to a RawMessage, which leaves it as it is).
func PublicJWK(pk []byte) string {
	return `{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"` + base64.RawURLEncoding.EncodeToString(pk) + `"}`
}

// ChainIssuer returns, per request, the body the chain endpoint's c.JSON writes for types.WorkflowVCChainResponse.  keys is the
// registry's public half, DID -> 32-byte public key, for every DID ResolveDID resolves: registry.RootDID (the key at m/44'/0', issuer of
// every workflow without records) and every agent's and component's DID.
type ChainIssuer interface {
	WorkflowChainBatch(reqs []ChainRequest, keys map[string][]byte) ([][]byte, error)
}

var _ ChainIssuer = ChainStdlib{}

// ChainStdlib is the reference's path, one workflow at a time: generateWorkflowVCDocument (WorkflowStdlib), the bundle, json.Marshal.
type ChainStdlib struct{}

func (ChainStdlib) WorkflowChainBatch(reqs []ChainRequest, keys map[string][]byte) ([][]byte, error) {
	out := make([][]byte, len(reqs))
	for i := range reqs {
		b, err := chainOne(&reqs[i], keys)
		if err != nil {
			return nil, err
		}
		out[i] = b
	}
	return out, nil
}

func chainOne(r *ChainRequest, keys map[string][]byte) ([]byte, error) {
	wvc, err := workflowOne(&r.WorkflowRequest)
	if err != nil {
		return nil, err
	}
	records := r.Records
	if records == nil {
		records = []types.ExecutionVC{} // GetExecutionVCsByWorkflow returns an empty slice, never nil (vc_storage.go:298)
	}
	return json.Marshal(types.WorkflowVCChainResponse{WorkflowID: r.WorkflowID, ComponentVCs: records, WorkflowVC: wvc, TotalSteps: len(records),
		Status: wvc.Status, DIDResolutionBundle: chainBundle(records, wvc.IssuerDID, keys, r.ResolvedAt)})
}

// chainBundle is collectDIDResolutionBundle with ResolveDID replaced by the registry's stored public JWK
func chainBundle(records []types.ExecutionVC, issuer string, keys map[string][]byte, resolvedAt string) map[string]types.DIDResolutionEntry {
	unique := map[string]bool{}
	for _, vc := range records {
		for _, d := range []string{vc.IssuerDID, vc.CallerDID, vc.TargetDID} {
			if d != "" && d != "did:key:" {
				unique[d] = true
			}
		}
	}
	if issuer != "" && issuer != "did:key:" {
		unique[issuer] = true
	}
	bundle := map[string]types.DIDResolutionEntry{}
	for did := range unique {
		pk, ok := keys[did]
		if !ok || len(strings.TrimSpace(did)) == 0 {
			continue
		}
		method := "key"
		if len(did) > 4 && did[:4] == "did:" {
			if parts := strings.Split(did, ":"); len(parts) >= 2 {
				method = parts[1]
			}
		}
		bundle[did] = types.DIDResolutionEntry{Method: method, PublicKeyJWK: json.RawMessage(PublicJWK(pk)), ResolvedFrom: "bundled", ResolvedAt: resolvedAt}
	}
	return bundle
}
