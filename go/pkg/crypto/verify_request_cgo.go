//go:build cgo && cuda

package crypto

/*
#include <stdlib.h>
#include "afcrypto.h"
*/
import "C"

import (
	"net/http"
	"unsafe"
)

// RequestCUDA answers request bodies on the GPU (afc_vc_verify_request_batch) against the named key set of a StoredCUDA.  Bodies the
// device leaves to the host (AFC_VREQ_HOST), and every body of a call that fails, are answered by RequestStdlib.
type RequestCUDA struct{ *StoredCUDA }

func (s RequestCUDA) VerifyRequestBatch(bodies [][]byte, resolve Resolver) ([]VerifyResponse, error) {
	n := len(bodies)
	if n == 0 {
		return nil, nil
	}
	total := 0
	for _, b := range bodies {
		total += len(b)
	}
	buf := C.malloc(C.size_t(total + 1))
	off := C.malloc(C.size_t(8 * (n + 1)))
	defer C.free(buf)
	defer C.free(off)
	b := unsafe.Slice((*byte)(buf), total+1)
	o := unsafe.Slice((*uint64)(off), n+1)
	pos := 0
	for i, d := range bodies {
		o[i] = uint64(pos)
		pos += copy(b[pos:], d)
	}
	o[n] = uint64(pos)
	capacity := C.afc_vc_verify_request_bound((*C.uint64_t)(off), C.uint32_t(n))
	out := C.malloc(C.size_t(capacity) + 1)
	boff := C.malloc(C.size_t(8 * (n + 1)))
	state := C.malloc(C.size_t(n))
	defer C.free(out)
	defer C.free(boff)
	defer C.free(state)
	rc := C.afc_vc_verify_request_batch(s.ctx, s.ks, (*C.uint8_t)(buf), (*C.uint64_t)(off), C.uint32_t(n), (*C.uint8_t)(out), capacity,
		(*C.uint64_t)(boff), (*C.uint8_t)(state))
	if rc != 0 {
		observeFallback("verify_request")
		return RequestStdlib{}.VerifyRequestBatch(bodies, resolve)
	}
	bo := unsafe.Slice((*uint64)(boff), n+1)
	st := unsafe.Slice((*byte)(state), n)
	ob := unsafe.Slice((*byte)(out), int(bo[n])+1)
	res := make([]VerifyResponse, n)
	for i := range bodies {
		switch st[i] {
		case C.AFC_VREQ_OK:
			res[i] = VerifyResponse{Status: http.StatusOK, Body: append([]byte(nil), ob[bo[i]:bo[i+1]]...)}
		case C.AFC_VREQ_BAD_REQUEST:
			res[i] = VerifyResponse{Status: http.StatusBadRequest, Body: badRequestBody}
		default:
			res[i] = verifyRequestOne(bodies[i], resolve)
		}
	}
	return res, nil
}
