// gen_golden_test.go — pins every expectation under tests/golden/ to the Go standard library and the reference's own structs.
//
// SOURCE ONLY in this repository (the build image has no Go toolchain).  Run it wherever Go 1.24 and the reference exist:
//
//	REF=/path/to/agentfield/control-plane ; REPO=/path/to/this/repo
//	mkdir -p $REF/tools/afcgolden && cp $REPO/baseline/go/gen_golden_test.go $REF/tools/afcgolden/
//	cd $REF && AFC_GOLDEN_DIR=$REPO/tests/golden go test ./tools/afcgolden -run TestPinGolden -v
//
// It (1) recomputes every expectation with exactly the calls the reference makes on this path —
//
//	ed25519.NewKeyFromSeed / Sign / Verify   internal/services/vc_service.go:460-463,504,712-715,1624
//	json.Marshal(types.VCDocument{..., Proof: zero})            :436-439, :471-474      (canonical bytes)
//	json.Marshal(types.WorkflowVCDocument{..., Proof: zero})    :686-693, :1589-1597
//	json.Unmarshal into the struct before re-marshalling        :250-251 (metadata -> float64)
//	msg[:500] + "...[truncated]"                               :153-160
//	hmac.New(sha256.New, secret) + "sha256="+hex               internal/services/webhook_dispatcher.go:470-474
//	json.Marshal(types.ExecutionWebhookPayload)                 :299, pkg/types/webhook.go:42-53
//	sha256.Sum256 + base64.RawURLEncoding                       vc_service.go:508-515
//	sha256(masterSeed || path), "did:key:z"+base64url(0xED01||pk)   internal/services/did_service.go:515-536
//
// — (2) FAILS on the first difference from the committed expectation, so `go test` alone turns parity green or red, and
// (3) writes $AFC_GOLDEN_DIR/go_pinned.json, which tests/test_oracle.py::test_go_pinned_vectors_when_present compares with the
// fixtures again from the Python side.  RFC 6962 has no stdlib implementation: it is restated below from the RFC with sha256.
package afcgolden

import (
	"bytes"
	"crypto/ed25519"
	"crypto/hmac"
	"crypto/sha256"
	"crypto/sha512"
	"encoding/base64"
	"encoding/binary"
	"encoding/hex"
	"encoding/json"
	"fmt"
	"math"
	"os"
	"path/filepath"
	"runtime"
	"testing"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

func goldenDir(t *testing.T) string {
	if d := os.Getenv("AFC_GOLDEN_DIR"); d != "" {
		return d
	}
	t.Fatal("set AFC_GOLDEN_DIR to <repo>/tests/golden")
	return ""
}

func load(t *testing.T, name string, v interface{}) {
	b, err := os.ReadFile(filepath.Join(goldenDir(t), name))
	if err != nil {
		t.Fatalf("%s: %v", name, err)
	}
	if err := json.Unmarshal(b, v); err != nil {
		t.Fatalf("%s: %v", name, err)
	}
}

func unhex(t *testing.T, s string) []byte {
	b, err := hex.DecodeString(s)
	if err != nil {
		t.Fatalf("bad hex %q", s)
	}
	return b
}

type pinned struct {
	File, Case, Field, Value string
}

var out []pinned

func check(t *testing.T, file, id, field, got, want string) {
	out = append(out, pinned{file, id, field, got})
	if got != want {
		t.Errorf("%s [%s] %s:\n   go: %s\n want: %s", file, id, field, got, want)
	}
}

func boolStr(b bool) string {
	if b {
		return "true"
	}
	return "false"
}

// ---- RFC 6962 §2.1 (no stdlib implementation)
func mth(leaves [][]byte) [32]byte {
	switch len(leaves) {
	case 0:
		return sha256.Sum256(nil)
	case 1:
		return sha256.Sum256(append([]byte{0}, leaves[0]...))
	}
	k := 1
	for k*2 < len(leaves) {
		k *= 2
	}
	l, r := mth(leaves[:k]), mth(leaves[k:])
	return sha256.Sum256(append(append([]byte{1}, l[:]...), r[:]...))
}

func verifyRecover(pk, msg, sig []byte) (ok bool) {
	// ed25519.Verify panics on len(pk) != 32 (the adapter re-panics): none of the fixtures has such a key
	return ed25519.Verify(ed25519.PublicKey(pk), msg, sig)
}

func TestPinGolden(t *testing.T) {
	out = nil
	// ---------------- rfc8032.json: NewKeyFromSeed, Sign, Verify
	var r8032 []struct{ Name, Seed, Pk, Msg, Sig string }
	load(t, "rfc8032.json", &r8032)
	for _, e := range r8032 {
		priv := ed25519.NewKeyFromSeed(unhex(t, e.Seed))
		check(t, "rfc8032.json", e.Name, "pk", hex.EncodeToString(priv.Public().(ed25519.PublicKey)), e.Pk)
		check(t, "rfc8032.json", e.Name, "sig", hex.EncodeToString(ed25519.Sign(priv, unhex(t, e.Msg))), e.Sig)
		check(t, "rfc8032.json", e.Name, "valid", boolStr(verifyRecover(unhex(t, e.Pk), unhex(t, e.Msg), unhex(t, e.Sig))), "true")
	}
	// ---------------- ed25519_edge.json: Go's accept / reject decision on every edge case
	var edge []struct {
		Name, Pk, Msg, Sig string
		Valid              bool
	}
	load(t, "ed25519_edge.json", &edge)
	for _, e := range edge {
		check(t, "ed25519_edge.json", e.Name, "valid", boolStr(verifyRecover(unhex(t, e.Pk), unhex(t, e.Msg), unhex(t, e.Sig))), boolStr(e.Valid))
	}
	// ---------------- rfc4231.json, fips180.json
	var r4231 []struct{ Name, Key, Msg, Tag string }
	load(t, "rfc4231.json", &r4231)
	for _, e := range r4231 {
		m := hmac.New(sha256.New, unhex(t, e.Key))
		m.Write(unhex(t, e.Msg))
		check(t, "rfc4231.json", e.Name, "tag", hex.EncodeToString(m.Sum(nil)), e.Tag)
	}
	var fips []struct{ Alg, Msg, Digest string }
	load(t, "fips180.json", &fips)
	for i, e := range fips {
		id := e.Alg + "#" + string(rune('0'+i/10)) + string(rune('0'+i%10))
		if e.Alg == "sha256" {
			d := sha256.Sum256(unhex(t, e.Msg))
			check(t, "fips180.json", id, "digest", hex.EncodeToString(d[:]), e.Digest)
		} else {
			d := sha512.Sum512(unhex(t, e.Msg))
			check(t, "fips180.json", id, "digest", hex.EncodeToString(d[:]), e.Digest)
		}
	}
	// ---------------- rfc6962.json: roots of the CT reference tree and of the synthetic logs
	var ct struct {
		EmptyRoot string `json:"empty_root"`
		Leaves    []string
		Roots     []string
		Synthetic []struct {
			N      int
			Leaves []string
			Root   string
		}
	}
	load(t, "rfc6962.json", &ct)
	er := mth(nil)
	check(t, "rfc6962.json", "empty", "root", hex.EncodeToString(er[:]), ct.EmptyRoot)
	var lv [][]byte
	for i, l := range ct.Leaves {
		lv = append(lv, unhex(t, l))
		r := mth(lv)
		check(t, "rfc6962.json", "ct-"+string(rune('1'+i)), "root", hex.EncodeToString(r[:]), ct.Roots[i])
	}
	for _, s := range ct.Synthetic {
		if len(s.Leaves) != s.N {
			continue // large logs carry a digest of their leaves instead of the leaves
		}
		var ls [][]byte
		for _, l := range s.Leaves {
			ls = append(ls, unhex(t, l))
		}
		r := mth(ls)
		check(t, "rfc6962.json", "synthetic", "root", hex.EncodeToString(r[:]), s.Root)
	}
	// ---------------- reference_flow.json: derivePrivateKey, did:key, hashData, one signed VC-shaped message
	var flow struct {
		MasterSeed  string `json:"master_seed"`
		Derivations []struct{ Path, Seed, Pk, Did string }
		HashData    []struct {
			Payload    *string
			Marshalled string
			Hash       string
		} `json:"hash_data"`
		Vc struct{ Canonical, Seed, Pk, Sig, ProofValue string }
	}
	load(t, "reference_flow.json", &flow)
	master := unhex(t, flow.MasterSeed)
	for _, d := range flow.Derivations {
		h := sha256.New() // did_service.go:517-521
		h.Write(master)
		h.Write([]byte(d.Path))
		seed := h.Sum(nil)
		priv := ed25519.NewKeyFromSeed(seed)
		pk := priv.Public().(ed25519.PublicKey)
		check(t, "reference_flow.json", d.Path, "seed", hex.EncodeToString(seed), d.Seed)
		check(t, "reference_flow.json", d.Path, "pk", hex.EncodeToString(pk), d.Pk)
		check(t, "reference_flow.json", d.Path, "did", "did:key:z"+base64.RawURLEncoding.EncodeToString(append([]byte{0xed, 0x01}, pk...)), d.Did)
	}
	for i, hd := range flow.HashData {
		var marshalled []byte
		if hd.Payload == nil {
			marshalled = []byte("null") // marshalDataOrNull(nil), vc_service.go:1298-1306
		} else {
			marshalled, _ = json.Marshal(unhex(t, *hd.Payload)) // json.Marshal([]byte) = quoted std base64
		}
		id := "hash_data#" + string(rune('0'+i))
		check(t, "reference_flow.json", id, "marshalled", hex.EncodeToString(marshalled), hd.Marshalled)
		sum := sha256.Sum256(marshalled)
		check(t, "reference_flow.json", id, "hash", base64.RawURLEncoding.EncodeToString(sum[:]), hd.Hash)
	}
	{
		priv := ed25519.NewKeyFromSeed(unhex(t, flow.Vc.Seed))
		sig := ed25519.Sign(priv, []byte(flow.Vc.Canonical))
		check(t, "reference_flow.json", "vc", "sig", hex.EncodeToString(sig), flow.Vc.Sig)
		check(t, "reference_flow.json", "vc", "proofValue", base64.RawURLEncoding.EncodeToString(sig), flow.Vc.ProofValue)
	}
	// ---------------- go_cases.json
	type party struct {
		Did          string
		Type         string
		AgentNodeDid string `json:"agent_node_did"`
		FunctionName string `json:"function_name"`
	}
	var gc struct {
		Floats  []struct{ Bits, Expect string }
		Strings []struct{ Utf8, Expect string }
		Execs   []struct {
			Context, Type                                               []string
			Id, Issuer                                                  string
			IssuanceDate                                                string `json:"issuance_date"`
			ExecutionId                                                 string `json:"execution_id"`
			WorkflowId                                                  string `json:"workflow_id"`
			SessionId                                                   string `json:"session_id"`
			Caller, Target                                              party
			InputHash                                                   string `json:"input_hash"`
			OutputHash                                                  string `json:"output_hash"`
			InputDataHash                                               string `json:"input_data_hash"`
			OutputDataHash                                              string `json:"output_data_hash"`
			Timestamp                                                   string
			DurationMs                                                  int `json:"duration_ms"`
			Status                                                      string
			ErrorMessageInput                                           string `json:"error_message_input"`
			MetadataJson                                                string `json:"metadata_json"`
			Seed, Pk                                                    string
			ProofCreated                                                string `json:"proof_created"`
			ExpectCanonical                                             string `json:"expect_canonical"`
			ExpectSig                                                   string `json:"expect_sig"`
			ExpectStored                                                string `json:"expect_stored"`
		} `json:"execution_vcs"`
		Workflows []struct {
			WorkflowId      string   `json:"workflow_id"`
			SessionId       string   `json:"session_id"`
			ComponentVcIds  []string `json:"component_vc_ids"`
			Status          string
			StartTime       string  `json:"start_time"`
			EndTime         *string `json:"end_time"`
			SnapshotTime    string  `json:"snapshot_time"`
			IssuerDid       string  `json:"issuer_did"`
			VcId            string  `json:"vc_id"`
			IssuanceDate    string  `json:"issuance_date"`
			ProofCreated    string  `json:"proof_created"`
			Seed, Pk        string
			ExpectCanonical string `json:"expect_canonical"`
			ExpectSig       string `json:"expect_sig"`
			ExpectStored    string `json:"expect_stored"`
		} `json:"workflow_vcs"`
		Webhooks []struct {
			Event        string
			ExecutionId  string `json:"execution_id"`
			WorkflowId   string `json:"workflow_id"`
			Status       string
			Target, Type string
			DurationMs   *int64  `json:"duration_ms"`
			ResultJson   *string `json:"result_json"`
			ErrorMessage *string `json:"error_message"`
			Timestamp    string
			Secret       string
			ExpectBody   string `json:"expect_body"`
			ExpectHeader string `json:"expect_header"`
		}
	}
	load(t, "go_cases.json", &gc)
	for _, f := range gc.Floats {
		x := math.Float64frombits(binary.BigEndian.Uint64(unhex(t, f.Bits)))
		b, err := json.Marshal(x)
		if err != nil {
			t.Fatalf("float %s: %v", f.Bits, err)
		}
		check(t, "go_cases.json", "float "+f.Bits, "json", string(b), f.Expect)
	}
	for _, s := range gc.Strings {
		b, _ := json.Marshal(string(unhex(t, s.Utf8)))
		check(t, "go_cases.json", "string "+s.Utf8, "json", string(b), s.Expect)
	}
	for _, c := range gc.Execs {
		msg := c.ErrorMessageInput
		if len(msg) > 500 { // vc_service.go:153-160
			msg = msg[:500] + "...[truncated]"
		}
		var md map[string]interface{}
		if err := json.Unmarshal([]byte(c.MetadataJson), &md); err != nil {
			t.Fatalf("metadata %s: %v", c.Id, err)
		}
		doc := types.VCDocument{
			Context: c.Context, Type: c.Type, ID: c.Id, Issuer: c.Issuer, IssuanceDate: c.IssuanceDate,
			CredentialSubject: types.VCCredentialSubject{
				ExecutionID: c.ExecutionId, WorkflowID: c.WorkflowId, SessionID: c.SessionId,
				Caller:    types.VCCaller{DID: c.Caller.Did, Type: c.Caller.Type, AgentNodeDID: c.Caller.AgentNodeDid},
				Target:    types.VCTarget{DID: c.Target.Did, AgentNodeDID: c.Target.AgentNodeDid, FunctionName: c.Target.FunctionName},
				Execution: types.VCExecution{InputHash: c.InputHash, OutputHash: c.OutputHash, Timestamp: c.Timestamp, DurationMS: c.DurationMs, Status: c.Status, ErrorMessage: msg},
				Audit:     types.VCAudit{InputDataHash: c.InputDataHash, OutputDataHash: c.OutputDataHash, Metadata: md},
			},
		}
		canonical, _ := json.Marshal(doc) // zero Proof still present: what signVC signs
		check(t, "go_cases.json", c.Id, "canonical", string(canonical), c.ExpectCanonical)
		priv := ed25519.NewKeyFromSeed(unhex(t, c.Seed))
		sig := ed25519.Sign(priv, canonical)
		check(t, "go_cases.json", c.Id, "sig", hex.EncodeToString(sig), c.ExpectSig)
		doc.Proof = types.VCProof{Type: "Ed25519Signature2020", Created: c.ProofCreated, VerificationMethod: c.Issuer + "#key-1",
			ProofPurpose: "assertionMethod", ProofValue: base64.RawURLEncoding.EncodeToString(sig)}
		stored, _ := json.Marshal(doc)
		check(t, "go_cases.json", c.Id, "stored", string(stored), c.ExpectStored)
		// VerifyVC: parse the stored bytes, zero the proof, re-marshal, verify (vc_service.go:250-251, 469-505)
		var parsed types.VCDocument
		if err := json.Unmarshal(stored, &parsed); err != nil {
			t.Fatalf("unmarshal stored %s: %v", c.Id, err)
		}
		pv := parsed.Proof.ProofValue
		parsed.Proof = types.VCProof{}
		again, _ := json.Marshal(parsed)
		check(t, "go_cases.json", c.Id, "remarshalled", string(again), c.ExpectCanonical)
		sb, _ := base64.RawURLEncoding.DecodeString(pv)
		check(t, "go_cases.json", c.Id, "verify", boolStr(ed25519.Verify(unhex(t, c.Pk), again, sb)), "true")
	}
	for _, c := range gc.Workflows {
		n := len(c.ComponentVcIds)
		doc := types.WorkflowVCDocument{ // createWorkflowVCDocument, vc_service.go:635-683
			Context: []string{"https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/workflow/v1"},
			Type:    []string{"VerifiableCredential", "AgentFieldWorkflowCredential"},
			ID:      "urn:agentfield:workflow-vc:" + c.VcId, Issuer: c.IssuerDid, IssuanceDate: c.IssuanceDate,
			CredentialSubject: types.WorkflowVCCredentialSubject{
				WorkflowID: c.WorkflowId, SessionID: c.SessionId, ComponentVCIDs: c.ComponentVcIds, TotalSteps: n, CompletedSteps: n, Status: c.Status,
				StartTime: c.StartTime, EndTime: c.EndTime, SnapshotTime: c.SnapshotTime,
				Orchestrator: types.VCCaller{DID: c.IssuerDid, Type: "agentfield_server", AgentNodeDID: c.IssuerDid},
				Audit: types.VCAudit{Metadata: map[string]interface{}{"agentfield_version": "1.0.0", "vc_version": "1.0",
					"workflow_type": "agent_execution_chain", "total_executions": n}},
			},
		}
		canonical, _ := json.Marshal(doc)
		check(t, "go_cases.json", c.WorkflowId, "canonical", string(canonical), c.ExpectCanonical)
		priv := ed25519.NewKeyFromSeed(unhex(t, c.Seed))
		sig := ed25519.Sign(priv, canonical)
		check(t, "go_cases.json", c.WorkflowId, "sig", hex.EncodeToString(sig), c.ExpectSig)
		doc.Proof = types.VCProof{Type: "Ed25519Signature2020", Created: c.ProofCreated, VerificationMethod: c.IssuerDid + "#key-1",
			ProofPurpose: "assertionMethod", ProofValue: base64.RawURLEncoding.EncodeToString(sig)}
		stored, _ := json.Marshal(doc)
		check(t, "go_cases.json", c.WorkflowId, "stored", string(stored), c.ExpectStored)
		var parsed types.WorkflowVCDocument // verifyWorkflowVCSignature, :1589-1625 (total_executions comes back as float64)
		if err := json.Unmarshal(stored, &parsed); err != nil {
			t.Fatalf("unmarshal stored %s: %v", c.WorkflowId, err)
		}
		parsed.Proof = types.VCProof{}
		again, _ := json.Marshal(parsed)
		check(t, "go_cases.json", c.WorkflowId, "remarshalled", string(again), c.ExpectCanonical)
		check(t, "go_cases.json", c.WorkflowId, "verify", boolStr(ed25519.Verify(unhex(t, c.Pk), again, sig)), "true")
	}
	for _, c := range gc.Webhooks {
		p := types.ExecutionWebhookPayload{Event: c.Event, ExecutionID: c.ExecutionId, RunID: c.WorkflowId, Status: c.Status, Target: c.Target,
			TargetType: c.Type, DurationMS: c.DurationMs, ErrorMessage: c.ErrorMessage, Timestamp: c.Timestamp}
		if c.ResultJson != nil {
			var res interface{}
			if err := json.Unmarshal([]byte(*c.ResultJson), &res); err != nil {
				t.Fatalf("result %s: %v", c.ExecutionId, err)
			}
			p.Result = res
		}
		body, _ := json.Marshal(p)
		check(t, "go_cases.json", c.ExecutionId, "body", string(body), c.ExpectBody)
		m := hmac.New(sha256.New, []byte(c.Secret)) // generateWebhookSignature
		m.Write(body)
		check(t, "go_cases.json", c.ExecutionId, "header", "sha256="+hex.EncodeToString(m.Sum(nil)), c.ExpectHeader)
	}
	// ---------------- webhook_cases.json: whole deliveries, buildPayload + determineWebhookEvent + decodeExecutionPayload
	// (internal/services/webhook_dispatcher.go:394-468) restated with the reference's own types and stdlib calls
	var wc []struct {
		ExecutionId  string  `json:"execution_id"`
		RunId        string  `json:"run_id"`
		Status       string  `json:"status"`
		NodeId       string  `json:"node_id"`
		ReasonerId   string  `json:"reasoner_id"`
		TargetType   string  `json:"target_type"`
		Timestamp    string  `json:"timestamp"`
		Result       string  `json:"result"`
		DurationMs   *int64  `json:"duration_ms"`
		ErrorMessage *string `json:"error_message"`
		Secret       *string `json:"secret"`
		ExpectBody   string  `json:"expect_body"`
		ExpectHeader *string `json:"expect_header"`
	}
	load(t, "webhook_cases.json", &wc)
	for _, c := range wc {
		p := types.ExecutionWebhookPayload{Event: types.WebhookEventExecutionFailed, ExecutionID: c.ExecutionId, RunID: c.RunId, Status: c.Status,
			Target: c.NodeId + "." + c.ReasonerId, TargetType: c.TargetType, DurationMS: c.DurationMs, Timestamp: c.Timestamp}
		if types.NormalizeExecutionStatus(c.Status) == string(types.ExecutionStatusSucceeded) {
			p.Event = types.WebhookEventExecutionCompleted
			if raw := []byte(c.Result); len(raw) > 0 {
				var v interface{}
				if err := json.Unmarshal(raw, &v); err == nil {
					p.Result = v
				} else {
					p.Result = string(raw)
				}
			}
		} else {
			p.ErrorMessage = c.ErrorMessage
		}
		body, _ := json.Marshal(p)
		check(t, "webhook_cases.json", c.ExecutionId, "body", string(body), c.ExpectBody)
		if c.Secret != nil && c.ExpectHeader != nil {
			m := hmac.New(sha256.New, []byte(*c.Secret))
			m.Write(body)
			check(t, "webhook_cases.json", c.ExecutionId, "header", "sha256="+hex.EncodeToString(m.Sum(nil)), *c.ExpectHeader)
		}
	}
	// ---------------- verify_request_cases.json: POST /api/v1/did/verify on raw bodies — gin's default ShouldBindJSON
	// (json.NewDecoder(body).Decode), VCService.VerifyVC (internal/services/vc_service.go:242-289) against the fixture's registry, and
	// c.JSON's json.Marshal of the response
	var vr struct {
		Registry []struct{ Did, Pk string }
		Cases    []struct {
			Name         string `json:"name"`
			BodyHex      string `json:"body_hex"`
			ExpectStatus int    `json:"expect_status"`
			ExpectBody   string `json:"expect_body"`
		}
	}
	load(t, "verify_request_cases.json", &vr)
	vrKeys := map[string][]byte{}
	for _, r := range vr.Registry {
		vrKeys[r.Did] = unhex(t, r.Pk)
	}
	for _, c := range vr.Cases {
		status, body := 200, []byte(nil)
		var req types.VCVerificationRequest
		if err := json.NewDecoder(bytes.NewReader(unhex(t, c.BodyHex))).Decode(&req); err != nil {
			status, body = 400, []byte(`{"error":"Invalid request body"}`)
		} else {
			res := types.VCVerificationResponse{}
			var vc types.VCDocument
			if err := json.Unmarshal(req.VCDocument, &vc); err != nil {
				res.Error = fmt.Sprintf("failed to parse VC document: %v", err)
			} else if pk, ok := vrKeys[vc.Issuer]; !ok {
				res.Error = fmt.Sprintf("failed to resolve issuer DID: DID not found: %s", vc.Issuer)
			} else {
				cp := vc
				cp.Proof = types.VCProof{}
				canonical, _ := json.Marshal(cp)
				if sig, err := base64.RawURLEncoding.DecodeString(vc.Proof.ProofValue); err != nil {
					res.Error = fmt.Sprintf("failed to verify signature: failed to decode signature: %v", err)
				} else if !verifyRecover(pk, canonical, sig) {
					res.Message = "Invalid signature"
				} else {
					res = types.VCVerificationResponse{Valid: true, IssuerDID: vc.Issuer, IssuedAt: vc.IssuanceDate, Message: "VC verified successfully"}
				}
			}
			body, _ = json.Marshal(res)
		}
		check(t, "verify_request_cases.json", c.Name, "status", fmt.Sprint(status), fmt.Sprint(c.ExpectStatus))
		check(t, "verify_request_cases.json", c.Name, "body", string(body), c.ExpectBody)
	}
	// ---------------- write go_pinned.json
	doc := map[string]interface{}{"go": runtime.Version(), "failed": t.Failed(), "entries": out}
	b, _ := json.MarshalIndent(doc, "", " ")
	if err := os.WriteFile(filepath.Join(goldenDir(t), "go_pinned.json"), append(b, '\n'), 0o644); err != nil {
		t.Fatal(err)
	}
	t.Logf("%d expectations pinned with %s -> go_pinned.json", len(out), runtime.Version())
}
