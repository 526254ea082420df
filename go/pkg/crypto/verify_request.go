package crypto

import (
	"bytes"
	"encoding/json"
	"net/http"
	"sync"
	"time"
)

// RequestVerifier answers raw request bodies of POST /api/v1/did/verify (DIDHandlers.VerifyVC, internal/handlers/did_handlers.go:97-111)
// and POST /api/ui/v1/vc/verify (internal/handlers/ui/did.go:442-469): per body the HTTP status and the exact bytes the handler's
// c.JSON writes.  The UI route adds "details": err.Error() to its 400 body; its caller builds that body itself when the status is 400.
type RequestVerifier interface {
	VerifyRequestBatch(bodies [][]byte, resolve Resolver) ([]VerifyResponse, error)
}

// VerifyResponse is one answer: Status (200 or 400) and Body, written with c.Data(Status, "application/json; charset=utf-8", Body).
type VerifyResponse struct {
	Status int
	Body   []byte
}

// verifyRequest is types.VCVerificationRequest (pkg/types/did_types.go:268-271).
type verifyRequest struct {
	VCDocument json.RawMessage `json:"vc_document"`
}

// RequestStdlib is the reference handler on one body at a time: gin's ShouldBindJSON with its default decoder
// (json.NewDecoder(body).Decode, the validator has nothing to check), VCService.VerifyVC on the raw vc_document, json.Marshal of the
// response (c.JSON, HTML escaping on).
type RequestStdlib struct{}

func (RequestStdlib) VerifyRequestBatch(bodies [][]byte, resolve Resolver) ([]VerifyResponse, error) {
	out := make([]VerifyResponse, len(bodies))
	for i, b := range bodies {
		out[i] = verifyRequestOne(b, resolve)
	}
	return out, nil
}

var badRequestBody = []byte(`{"error":"Invalid request body"}`)

func verifyRequestOne(body []byte, resolve Resolver) VerifyResponse {
	var req verifyRequest
	if err := json.NewDecoder(bytes.NewReader(body)).Decode(&req); err != nil {
		return VerifyResponse{Status: http.StatusBadRequest, Body: badRequestBody}
	}
	res := verifyStoredOne(ExecutionVC, req.VCDocument, resolve)
	b, err := json.Marshal(res)
	if err != nil {
		return VerifyResponse{Status: http.StatusInternalServerError, Body: []byte(`{"error":"Failed to verify VC"}`)}
	}
	return VerifyResponse{Status: http.StatusOK, Body: b}
}

// RequestBatcher lets concurrent handler goroutines share one VerifyRequestBatch call, in the manner of VerifyBatcher: bodies queue
// until BatchMax are pending or LingerMicros have passed since the first, then one call answers them all.
type RequestBatcher struct {
	V            RequestVerifier
	Resolve      Resolver
	BatchMax     int
	LingerMicros int

	mu      sync.Mutex
	pending []requestItem
	timer   *time.Timer
}

type requestItem struct {
	body []byte
	out  chan VerifyResponse
}

// Verify answers one request body; the handler becomes "read the body, Verify it, c.Data(status, ..., body)".
func (b *RequestBatcher) Verify(body []byte) VerifyResponse {
	r := requestItem{body: body, out: make(chan VerifyResponse, 1)}
	b.mu.Lock()
	b.pending = append(b.pending, r)
	if len(b.pending) >= b.BatchMax {
		batch := b.take()
		b.mu.Unlock()
		b.flush(batch)
	} else {
		if b.timer == nil {
			b.timer = time.AfterFunc(time.Duration(b.LingerMicros)*time.Microsecond, func() {
				b.mu.Lock()
				batch := b.take()
				b.mu.Unlock()
				b.flush(batch)
			})
		}
		b.mu.Unlock()
	}
	return <-r.out
}

func (b *RequestBatcher) take() []requestItem {
	batch := b.pending
	b.pending = nil
	if b.timer != nil {
		b.timer.Stop()
		b.timer = nil
	}
	return batch
}

func (b *RequestBatcher) flush(batch []requestItem) {
	if len(batch) == 0 {
		return
	}
	bodies := make([][]byte, len(batch))
	for i, r := range batch {
		bodies[i] = r.body
	}
	res, err := b.V.VerifyRequestBatch(bodies, b.Resolve)
	if err != nil {
		res, _ = RequestStdlib{}.VerifyRequestBatch(bodies, b.Resolve)
	}
	for i, r := range batch {
		r.out <- res[i]
	}
}
