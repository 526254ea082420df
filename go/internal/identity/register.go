package identity

import (
	"crypto/ed25519"
	"crypto/sha512"
	"encoding/base64"
	"encoding/json"
	"fmt"
	"hash/fnv"
)

// Request is one new agent: types.DIDRegistrationRequest's node id and the ids of its reasoners and skills, and the agent index the
// registry assigns it (len(registry.AgentNodes) when the request is handled).
type Request struct {
	AgentNodeID string
	Reasoners   []string
	Skills      []string
	AgentIndex  uint32
}

// Identity mirrors types.DIDIdentity (pkg/types/did_types.go:114-121).
type Identity struct {
	DID            string `json:"did"`
	PrivateKeyJWK  string `json:"private_key_jwk"`
	PublicKeyJWK   string `json:"public_key_jwk"`
	DerivationPath string `json:"derivation_path"`
	ComponentType  string `json:"component_type"`
	FunctionName   string `json:"function_name,omitempty"`
}

// Package mirrors types.DIDIdentityPackage; Response mirrors types.DIDRegistrationResponse (did_types.go:106-111, 253-265).
type Package struct {
	AgentDID           Identity            `json:"agent_did"`
	ReasonerDIDs       map[string]Identity `json:"reasoner_dids"`
	SkillDIDs          map[string]Identity `json:"skill_dids"`
	AgentFieldServerID string              `json:"agentfield_server_id"`
}
type Response struct {
	Success         bool    `json:"success"`
	IdentityPackage Package `json:"identity_package"`
	Message         string  `json:"message,omitempty"`
	Error           string  `json:"error,omitempty"`
}

// Component is one derived key: the agent, then each non-empty reasoner id, then each non-empty skill id, in request order.  Key is the
// expanded form afc_ed25519_expand_batch writes (clamped scalar || prefix || public key, from SHA-512 of the derived seed): what
// afc_ed25519_sign_expanded* and both credential issue calls take.  Kept is false for an id repeated later in its list (the map keeps the
// later one).  Key is secret: the caller wipes it when it is done.
type Component struct {
	Path string
	Key  [96]byte
	DID  string
	Kept bool
}

// Pub is the component's public key (the last 32 bytes of Key).
func (c *Component) Pub() ed25519.PublicKey { return ed25519.PublicKey(c.Key[64:]) }

// Result is what handleNewRegistration computes for one request: its components and the response body c.JSON writes.
type Result struct {
	Components []Component
	Body       []byte
}

// Registrar registers new agents in bulk (handleNewRegistration, internal/services/did_service.go:186-365, and BackfillExistingNodes'
// loop, :653-723).
type Registrar interface {
	Register(masterSeed []byte, serverID string, reqs []Request) ([]Result, error)
}

// ServerHash is hashAgentFieldServerID (:578-582).
func ServerHash(serverID string) uint32 {
	h := fnv.New32a()
	h.Write([]byte(serverID))
	return h.Sum32() % (1 << 31)
}

// RegisterStdlib is the reference's loop: SHA-256 and ed25519.NewKeyFromSeed on the CPU, one component at a time.
type RegisterStdlib struct{}

func jwk(pub ed25519.PublicKey, seed []byte) string {
	m := map[string]interface{}{"kty": "OKP", "crv": "Ed25519", "x": base64.RawURLEncoding.EncodeToString(pub), "use": "sig", "alg": "EdDSA"}
	if seed != nil {
		m["d"] = base64.RawURLEncoding.EncodeToString(seed)
	}
	b, _ := json.Marshal(m)
	return string(b)
}

func stdlibComponent(masterSeed []byte, path, ctype, fn string) (Component, Identity) {
	e := Derive(masterSeed, path)
	pub := ed25519.PublicKey(e.Pub[:])
	did := "did:key:z" + base64.RawURLEncoding.EncodeToString(append([]byte{0xed, 0x01}, pub...))
	c := Component{Path: path, DID: did, Kept: true}
	h := sha512.Sum512(e.Seed[:]) // ed25519.NewKeyFromSeed's expansion
	h[0] &= 248
	h[31] &= 127
	h[31] |= 64
	copy(c.Key[:64], h[:])
	copy(c.Key[64:], pub)
	ident := Identity{DID: did, PrivateKeyJWK: jwk(pub, e.Seed[:]), PublicKeyJWK: jwk(pub, nil), DerivationPath: path, ComponentType: ctype, FunctionName: fn}
	for i := range h {
		h[i] = 0
	}
	for i := range e.Seed {
		e.Seed[i] = 0
	}
	return c, ident
}

func (RegisterStdlib) Register(masterSeed []byte, serverID string, reqs []Request) ([]Result, error) {
	h := ServerHash(serverID)
	out := make([]Result, len(reqs))
	for i, r := range reqs {
		agentPath := fmt.Sprintf("m/44'/%d'/%d'", h, r.AgentIndex)
		ac, aid := stdlibComponent(masterSeed, agentPath, "agent", "")
		comps := []Component{ac}
		maps := [2]map[string]Identity{{}, {}}
		for kind, list := range [2][]string{r.Reasoners, r.Skills} {
			at := map[string]int{}
			j := 0
			for _, id := range list {
				if id == "" {
					continue
				}
				ctype := [2]string{"reasoner", "skill"}[kind]
				c, ident := stdlibComponent(masterSeed, fmt.Sprintf("m/44'/%d'/%d'/%d'/%d'", h, r.AgentIndex, kind, j), ctype, id)
				if k, ok := at[id]; ok {
					comps[k].Kept = false
				}
				at[id] = len(comps)
				comps = append(comps, c)
				maps[kind][id] = ident
				j++
			}
		}
		resp := Response{Success: true, IdentityPackage: Package{AgentDID: aid, ReasonerDIDs: maps[0], SkillDIDs: maps[1], AgentFieldServerID: serverID},
			Message: fmt.Sprintf("Successfully registered agent %s with %d reasoners and %d skills", r.AgentNodeID, len(maps[0]), len(maps[1]))}
		body, err := json.Marshal(resp)
		if err != nil {
			return nil, err
		}
		out[i] = Result{Components: comps, Body: body}
	}
	return out, nil
}
