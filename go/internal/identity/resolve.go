package identity

import (
	"encoding/base64"
	"encoding/json"
	"fmt"
	"net/http"
)

// Request kinds of a Resolver: the two DID handlers of internal/handlers/did_handlers.go.
const (
	ResolveRequest  = 0 // GET /api/v1/did/resolve/:did (:73-94)
	DocumentRequest = 1 // GET /api/v1/did/document/:did (:368-429)
)

// ResolveReq is one request to either handler: its kind and c.Param("did").
type ResolveReq struct {
	Kind int
	DID  string
}

// ResolveResp is what the handler writes: the HTTP status and the body c.JSON writes.
type ResolveResp struct {
	Status int
	Body   []byte
}

// SnapshotComponent is a reasoner or skill as the registry stores it.
type SnapshotComponent struct {
	FunctionName, DID, DerivationPath, PublicKeyJWK string
}

// SnapshotAgent is an agent node as the registry stores it, its reasoners and skills in insertion order.
type SnapshotAgent struct {
	DID, DerivationPath, PublicKeyJWK string
	Reasoners, Skills                 []SnapshotComponent
}

// Snapshot is the part of the server's DID registry ResolveDID (internal/services/did_service.go:368-473) reads: the root DID with its
// public key, and the agents in registration order.  The registry keeps agents and components in Go maps, whose iteration order is
// random, so the reference may return any holder of a DID the registry holds twice (re-registration gives every new component of one
// kind the same DID); a Snapshot fixes one order, and both resolvers return the first holder in it.
type Snapshot struct {
	RootDID string
	RootPub []byte
	Agents  []SnapshotAgent
}

// Resolver serves a batch of DID requests against a registry snapshot.  The handlers' registry checks (DID system disabled, missing
// server registry) stay with the caller.
type Resolver interface {
	Serve(snap *Snapshot, reqs []ResolveReq) ([]ResolveResp, error)
}

var _ Resolver = ResolveStdlib{}

// ResolveStdlib is the reference's path, one request at a time: ResolveDID's scan, then the handler's c.JSON (json.Marshal of a map:
// keys sorted, HTML escaping on).  It does not rebuild the private JWK ResolveDID regenerates, which both handlers discard.
type ResolveStdlib struct{}

type resolved struct {
	DID, PublicKeyJWK, DerivationPath, ComponentType, FunctionName string
}

func lookup(snap *Snapshot, did string) (resolved, bool) {
	if snap.RootDID == did {
		jwk, _ := json.Marshal(map[string]interface{}{"kty": "OKP", "crv": "Ed25519", "x": base64.RawURLEncoding.EncodeToString(snap.RootPub),
			"use": "sig", "alg": "EdDSA"})
		return resolved{did, string(jwk), "m/44'/0'", "agentfield_server", ""}, true
	}
	for _, a := range snap.Agents {
		if a.DID == did {
			return resolved{a.DID, a.PublicKeyJWK, a.DerivationPath, "agent", ""}, true
		}
		for _, c := range a.Reasoners {
			if c.DID == did {
				return resolved{c.DID, c.PublicKeyJWK, c.DerivationPath, "reasoner", c.FunctionName}, true
			}
		}
		for _, c := range a.Skills {
			if c.DID == did {
				return resolved{c.DID, c.PublicKeyJWK, c.DerivationPath, "skill", c.FunctionName}, true
			}
		}
	}
	return resolved{}, false
}

func respond(status int, v interface{}) ResolveResp {
	b, _ := json.Marshal(v)
	return ResolveResp{status, b}
}

func serveOne(snap *Snapshot, r ResolveReq) ResolveResp {
	if r.DID == "" {
		return respond(http.StatusBadRequest, map[string]interface{}{"error": "DID parameter is required"})
	}
	id, ok := lookup(snap, r.DID)
	if r.Kind == ResolveRequest {
		if !ok {
			return respond(http.StatusNotFound, map[string]interface{}{"error": "DID not found"})
		}
		return respond(http.StatusOK, map[string]interface{}{"did": id.DID, "public_key_jwk": id.PublicKeyJWK, "component_type": id.ComponentType,
			"function_name": id.FunctionName, "derivation_path": id.DerivationPath})
	}
	if !ok {
		return respond(http.StatusNotFound, map[string]interface{}{"error": "DID not found", "details": fmt.Sprintf("DID not found: %s", r.DID)})
	}
	var publicKeyJWK map[string]interface{}
	if err := json.Unmarshal([]byte(id.PublicKeyJWK), &publicKeyJWK); err != nil {
		return respond(http.StatusInternalServerError, map[string]interface{}{"error": "Failed to parse public key", "details": err.Error()})
	}
	did := r.DID
	return respond(http.StatusOK, map[string]interface{}{
		"@context":           []string{"https://www.w3.org/ns/did/v1", "https://w3id.org/security/suites/ed25519-2020/v1"},
		"id":                 did,
		"verificationMethod": []map[string]interface{}{{"id": did + "#key-1", "type": "Ed25519VerificationKey2020", "controller": did, "publicKeyJwk": publicKeyJWK}},
		"authentication":     []string{did + "#key-1"},
		"assertionMethod":    []string{did + "#key-1"},
		"service": []map[string]interface{}{{"id": did + "#agentfield-service", "type": "AgentFieldAgentService",
			"serviceEndpoint": "https://agentfield.example.com/api/v1", "description": "AgentField Agent Platform Service"}},
	})
}

func (ResolveStdlib) Serve(snap *Snapshot, reqs []ResolveReq) ([]ResolveResp, error) {
	out := make([]ResolveResp, len(reqs))
	for i, r := range reqs {
		out[i] = serveOne(snap, r)
	}
	return out, nil
}
