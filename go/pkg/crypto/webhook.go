package crypto

import (
	"crypto/hmac"
	"crypto/sha256"
	"encoding/hex"
	"encoding/json"
	"fmt"

	"github.com/Agent-Field/agentfield/control-plane/pkg/types"
)

// WebhookDelivery is one execution webhook delivery (internal/services/webhook_dispatcher.go:294-320): the execution record's
// fields the payload reads, the target type the caller resolved (resolveTargetType), the timestamp it formatted (CompletedAt in
// RFC 3339, or now) and the webhook's secret (nil: no signature header).
type WebhookDelivery struct {
	ExecutionID, RunID, Status, NodeID, ReasonerID string
	TargetType, Timestamp                          string
	DurationMS                                     *int64
	ResultPayload                                  json.RawMessage // the stored raw result (empty: nil)
	ErrorMessage                                   *string
	Secret                                         *string
}

// SignedWebhook is a delivery's request body and its X-AgentField-Signature value ("" without a secret).
type SignedWebhook struct {
	Body      []byte
	Signature string
}

// WebhookSigner builds and signs many deliveries: exactly the body json.Marshal(buildPayload(...)) and the header
// generateWebhookSignature write.
type WebhookSigner interface {
	SignWebhookBatch(ds []WebhookDelivery) ([]SignedWebhook, error)
}

var _ WebhookSigner = WebhookStdlib{}

// WebhookStdlib is the reference's own path, one delivery at a time: buildPayload + json.Marshal + generateWebhookSignature.
type WebhookStdlib struct{}

func (WebhookStdlib) SignWebhookBatch(ds []WebhookDelivery) ([]SignedWebhook, error) {
	out := make([]SignedWebhook, len(ds))
	for i := range ds {
		s, err := signWebhookOne(&ds[i])
		if err != nil {
			return nil, err
		}
		out[i] = s
	}
	return out, nil
}

func webhookEvent(status string) string { // determineWebhookEvent, webhook_dispatcher.go:450-457
	if types.NormalizeExecutionStatus(status) == string(types.ExecutionStatusSucceeded) {
		return types.WebhookEventExecutionCompleted
	}
	return types.WebhookEventExecutionFailed
}

func decodeResult(raw json.RawMessage) interface{} { // decodeExecutionPayload, webhook_dispatcher.go:459-468
	if len(raw) == 0 {
		return nil
	}
	var v interface{}
	if err := json.Unmarshal(raw, &v); err == nil {
		return v
	}
	return string(raw)
}

func signWebhookOne(d *WebhookDelivery) (SignedWebhook, error) {
	event := webhookEvent(d.Status)
	p := types.ExecutionWebhookPayload{
		Event: event, ExecutionID: d.ExecutionID, RunID: d.RunID, Status: d.Status,
		Target: fmt.Sprintf("%s.%s", d.NodeID, d.ReasonerID), TargetType: d.TargetType, DurationMS: d.DurationMS, Timestamp: d.Timestamp,
	}
	if event == types.WebhookEventExecutionCompleted {
		p.Result = decodeResult(d.ResultPayload)
	} else {
		p.ErrorMessage = d.ErrorMessage
	}
	body, err := json.Marshal(p)
	if err != nil {
		return SignedWebhook{}, err
	}
	s := SignedWebhook{Body: body}
	if d.Secret != nil {
		mac := hmac.New(sha256.New, []byte(*d.Secret))
		mac.Write(body)
		s.Signature = "sha256=" + hex.EncodeToString(mac.Sum(nil))
	}
	return s, nil
}
