//go:build cgo && cuda

package crypto

/*
#include "afcrypto.h"
*/
import "C"

import "unsafe"

// WebhookCUDA builds and signs a batch in one afc_webhook_sign_batch call.  Deliveries the device leaves to the host
// (AFC_WEBHOOK_HOST) go through WebhookStdlib one by one; any non-zero return code sends the whole batch there.
type WebhookCUDA struct {
	c        *CUDA
	fallback WebhookStdlib
}

func NewWebhookCUDA(c *CUDA) *WebhookCUDA { return &WebhookCUDA{c: c} }

func (s *WebhookCUDA) SignWebhookBatch(ds []WebhookDelivery) ([]SignedWebhook, error) {
	n := len(ds)
	if n == 0 {
		return nil, nil
	}
	const nc = C.AFC_WEBHOOK_COLUMNS
	var cols, results, secrets []byte
	colOff := make([]uint64, 0, n*nc+1)
	resOff := make([]uint64, 0, n+1)
	secOff := make([]uint32, 0, n+1)
	dur := make([]int64, n)
	flags := make([]uint8, n)
	for i := range ds {
		d := &ds[i]
		em := ""
		if d.ErrorMessage != nil {
			em = *d.ErrorMessage
			flags[i] |= C.AFC_WEBHOOK_HAS_ERROR_MESSAGE
		}
		for _, c := range [nc]string{d.ExecutionID, d.RunID, d.Status, d.NodeID, d.ReasonerID, d.TargetType, d.Timestamp, em} {
			colOff = append(colOff, uint64(len(cols)))
			cols = append(cols, c...)
		}
		if d.DurationMS != nil {
			dur[i] = *d.DurationMS
			flags[i] |= C.AFC_WEBHOOK_HAS_DURATION
		}
		resOff = append(resOff, uint64(len(results)))
		results = append(results, d.ResultPayload...)
		secOff = append(secOff, uint32(len(secrets)))
		if d.Secret != nil {
			secrets = append(secrets, *d.Secret...)
			flags[i] |= C.AFC_WEBHOOK_HAS_SECRET
		}
	}
	colOff = append(colOff, uint64(len(cols)))
	resOff = append(resOff, uint64(len(results)))
	secOff = append(secOff, uint32(len(secrets)))
	defer func() { // secrets do not outlive the call in this process either
		for i := range secrets {
			secrets[i] = 0
		}
	}()
	bound := uint64(C.afc_webhook_bound((*C.uint64_t)(unsafe.Pointer(&colOff[0])), (*C.uint64_t)(unsafe.Pointer(&resOff[0])), C.uint32_t(n)))
	bodies := make([]byte, bound+1)
	bodyOff := make([]uint64, n+1)
	headers := make([]byte, n*C.AFC_WEBHOOK_HEADER_CHARS)
	status := make([]uint8, n)
	d := s.c.pick()
	rc := C.afc_webhook_sign_batch(d.ctx, bytesPtr(cols), (*C.uint64_t)(unsafe.Pointer(&colOff[0])), (*C.int64_t)(unsafe.Pointer(&dur[0])),
		(*C.uint8_t)(unsafe.Pointer(&flags[0])), bytesPtr(results), (*C.uint64_t)(unsafe.Pointer(&resOff[0])), bytesPtr(secrets),
		(*C.uint32_t)(unsafe.Pointer(&secOff[0])), C.uint32_t(n), (*C.uint8_t)(unsafe.Pointer(&bodies[0])), C.uint64_t(bound+1),
		(*C.uint64_t)(unsafe.Pointer(&bodyOff[0])), (*C.uint8_t)(unsafe.Pointer(&headers[0])), (*C.uint8_t)(unsafe.Pointer(&status[0])))
	if rc != 0 {
		return s.fallback.SignWebhookBatch(ds)
	}
	out := make([]SignedWebhook, n)
	for i := range ds {
		if status[i] == C.AFC_WEBHOOK_HOST {
			one, err := signWebhookOne(&ds[i])
			if err != nil {
				return nil, err
			}
			out[i] = one
			continue
		}
		out[i].Body = bodies[bodyOff[i]:bodyOff[i+1]:bodyOff[i+1]]
		if ds[i].Secret != nil {
			out[i].Signature = string(headers[i*C.AFC_WEBHOOK_HEADER_CHARS : (i+1)*C.AFC_WEBHOOK_HEADER_CHARS])
		}
	}
	return out, nil
}

// bytesPtr is the address of a byte slice's first element, or NULL for an empty one.
func bytesPtr(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&b[0]))
}
