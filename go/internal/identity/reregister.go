package identity

import (
	"encoding/json"
	"fmt"
	"strconv"
	"strings"
)

// StoredComponent is what the registry holds for one reasoner or skill (types.ReasonerDIDInfo / SkillDIDInfo) and the existing identity
// package needs: its map key, DID, stored public JWK (a json.RawMessage, copied as stored), derivation path and function name.
type StoredComponent struct {
	Key            string
	DID            string
	PublicKeyJWK   []byte
	DerivationPath string
	FunctionName   string
}

// KnownAgent is a registry record (types.AgentDIDInfo): the agent's own DID, stored public JWK and path, and its components in any order.
type KnownAgent struct {
	DID            string
	PublicKeyJWK   []byte
	DerivationPath string
	Reasoners      []StoredComponent
	Skills         []StoredComponent
}

// ReRequest is a registration request for an agent the registry already holds.  AgentIndex is the <a> of the new components' paths;
// AgentIndexOf(Agent.DerivationPath) is the stable choice (the reference uses the agent's place in Go's randomised map iteration).
type ReRequest struct {
	Agent      KnownAgent
	Reasoners  []string
	Skills     []string
	AgentIndex uint32
}

// The states of a re-registration (AFC_DIDRR_*).
const (
	ReUnchanged = 0 // nothing new or removed: the existing identity package
	ReRemoved   = 1 // removals only: the package of what remains
	RePartial   = 2 // new components: only they are in the body, with their private JWKs
	ReInvalid   = 3 // a stored list repeats a key, which no Go map can: refused, empty body
)

// ReResult is what RegisterAgent's branch for a known agent returns and changes.  Gone[kind][k] marks Agent.Reasoners / .Skills [k] for
// deletion; New[kind] lists the ids to add (each once), all with the key of Slots[kind], whose Key is secret (the caller wipes it).
// Counts: new reasoners, new skills, removed reasoners, removed skills.
type ReResult struct {
	State  int
	Counts [4]int
	Body   []byte
	Gone   [2][]bool
	New    [2][]string
	Slots  [2]*Component
}

// Reregistrar re-registers known agents in bulk (RegisterAgent, internal/services/did_service.go:154-179: PerformDifferentialAnalysis,
// DeregisterComponents, PartialRegisterAgent or buildExistingIdentityPackage).  Requests must name distinct agents.
type Reregistrar interface {
	Reregister(masterSeed []byte, serverID string, reqs []ReRequest) ([]ReResult, error)
}

// AgentIndexOf reads <a> from an agent path m/44'/<h>'/<a>'.
func AgentIndexOf(path string) (uint32, error) {
	p := strings.Split(path, "/")
	if len(p) != 4 || p[0] != "m" || p[1] != "44'" || !strings.HasSuffix(p[3], "'") {
		return 0, fmt.Errorf("not an agent derivation path: %q", path)
	}
	a, err := strconv.ParseUint(strings.TrimSuffix(p[3], "'"), 10, 32)
	return uint32(a), err
}

// ReregisterStdlib is the reference's branch on the CPU, request by request.
type ReregisterStdlib struct{}

func storedIdentity(c StoredComponent, ctype string) Identity {
	return Identity{DID: c.DID, PublicKeyJWK: string(c.PublicKeyJWK), DerivationPath: c.DerivationPath, ComponentType: ctype, FunctionName: c.FunctionName}
}

func (ReregisterStdlib) Reregister(masterSeed []byte, serverID string, reqs []ReRequest) ([]ReResult, error) {
	h := ServerHash(serverID)
	out := make([]ReResult, len(reqs))
	for i, r := range reqs {
		res := &out[i]
		stored := [2][]StoredComponent{r.Agent.Reasoners, r.Agent.Skills}
		res.Gone = [2][]bool{make([]bool, len(stored[0])), make([]bool, len(stored[1]))}
		invalid := false
		for kind := range stored {
			seen := map[string]bool{}
			for _, c := range stored[kind] {
				invalid = invalid || seen[c.Key]
				seen[c.Key] = true
			}
		}
		if invalid {
			res.State = ReInvalid
			res.Gone = [2][]bool{make([]bool, len(stored[0])), make([]bool, len(stored[1]))}
			continue
		}
		var newIDs [2][]string
		left := [2]int{}
		for kind, list := range [2][]string{r.Reasoners, r.Skills} {
			given, have := map[string]bool{}, map[string]bool{}
			for _, id := range list {
				if id != "" { // extractReasonerIDs / extractSkillIDs
					given[id] = true
				}
			}
			for k, c := range stored[kind] {
				have[c.Key] = true
				res.Gone[kind][k] = !given[c.Key] // setDifference(existing, new)
				if res.Gone[kind][k] {
					res.Counts[2+kind]++
				} else {
					left[kind]++
				}
			}
			for _, id := range list {
				if id != "" && !have[id] {
					newIDs[kind] = append(newIDs[kind], id) // setDifference(new, existing): duplicates kept
				}
			}
		}
		agent := Identity{DID: r.Agent.DID, PublicKeyJWK: string(r.Agent.PublicKeyJWK), DerivationPath: r.Agent.DerivationPath, ComponentType: "agent"}
		maps := [2]map[string]Identity{{}, {}}
		var msg string
		switch {
		case len(newIDs[0])+len(newIDs[1]) > 0: // PartialRegisterAgent: one path per kind, j = the map's size after the removals
			res.State = RePartial
			for kind := range newIDs {
				if len(newIDs[kind]) == 0 {
					continue
				}
				ctype := [2]string{"reasoner", "skill"}[kind]
				path := fmt.Sprintf("m/44'/%d'/%d'/%d'/%d'", h, r.AgentIndex, kind, left[kind])
				for _, id := range newIDs[kind] {
					c, ident := stdlibComponent(masterSeed, path, ctype, id)
					if res.Slots[kind] == nil {
						cc := c
						res.Slots[kind] = &cc
					}
					for k := range c.Key {
						c.Key[k] = 0
					}
					if _, dup := maps[kind][id]; !dup {
						res.New[kind] = append(res.New[kind], id)
					}
					maps[kind][id] = ident
				}
				res.Counts[kind] = len(maps[kind])
			}
			msg = fmt.Sprintf("Partial registration successful: %d new reasoners, %d new skills", len(maps[0]), len(maps[1]))
		default:
			for kind, ctype := range [2]string{"reasoner", "skill"} {
				for k, c := range stored[kind] {
					if !res.Gone[kind][k] {
						maps[kind][c.Key] = storedIdentity(c, ctype)
					}
				}
			}
			if res.Counts[2]+res.Counts[3] > 0 {
				res.State = ReRemoved
				msg = fmt.Sprintf("Registration updated: removed %d reasoners, %d skills", res.Counts[2], res.Counts[3])
			} else {
				res.State = ReUnchanged
				msg = "No changes detected, registration skipped"
			}
		}
		body, err := json.Marshal(Response{Success: true, IdentityPackage: Package{AgentDID: agent, ReasonerDIDs: maps[0], SkillDIDs: maps[1],
			AgentFieldServerID: serverID}, Message: msg})
		if err != nil {
			return nil, err
		}
		res.Body = body
	}
	return out, nil
}
