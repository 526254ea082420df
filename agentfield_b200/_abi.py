"""ctypes binding of libafcrypto.so (include/afcrypto.h).

This is the Python twin of the cgo binding a reference maintainer adds (INTEGRATION.md): the same
entry points, packed buffers + offset arrays, negative return codes.  The library has NO CPU
implementation; loading it without a GPU works (so the symbol table can be checked) but `Context()`
raises AfcError(AFC_ECUDA).
"""
import ctypes as C
import os

import numpy as np

AFC_OK, AFC_EINVAL, AFC_ECUDA, AFC_ENOMEM, AFC_ENCCL, AFC_ESTATE = 0, -1, -2, -3, -4, -5
DOC_EXECUTION_VC, DOC_WORKFLOW_VC = 0, 1
VC_INVALID, VC_VALID, VC_HOST, VC_UNRESOLVED, VC_BAD_ENCODING = 0, 1, 2, 3, 4
VREQ_OK, VREQ_BAD_REQUEST, VREQ_HOST = 0, 1, 2
AUDIT_COLUMNS = ("issuer_did", "execution_id", "workflow_id", "session_id", "caller_did", "target_did", "status", "input_hash", "output_hash",
                 "signature")
# AFC_AUDIT_*: bit k < 10 = column k of AUDIT_COLUMNS differs from the document
AUDIT_INVALID_TIMESTAMP, AUDIT_MISSING_CONTEXT, AUDIT_MISSING_TYPE, AUDIT_MISSING_ID = 1 << 10, 1 << 11, 1 << 12, 1 << 13
AUDIT_MISSING_ISSUER, AUDIT_MISSING_ISSUANCE_DATE, AUDIT_NOT_W3C, AUDIT_NOT_AGENTFIELD = 1 << 14, 1 << 15, 1 << 16, 1 << 17
AUDIT_STATUS_UNDECIDED, AUDIT_TIMESTAMP_UNDECIDED = 1 << 18, 1 << 19
ISSUE_COLUMNS = ("vc_id", "caller_did", "issuance_date", "execution_id", "workflow_id", "session_id", "caller_type", "agent_node_did",
                 "target_did", "function_name", "timestamp", "status", "error_message", "proof_created")
ISSUE_HASH_DATA = 1
WORKFLOW_COLUMNS = ("workflow_id", "session_id", "issuer_did", "vc_id", "issuance_date", "snapshot_time", "proof_created")
WORKFLOW_RECORD_COLUMNS = ("vc_id", "status")
WORKFLOW_BUILT, WORKFLOW_HOST = 0, 1
CHAIN_WORKFLOW_COLUMNS = ("workflow_vc_id", "resolved_at")
CHAIN_RECORD_COLUMNS = ("execution_id", "workflow_id", "session_id", "agent_node_id", "workflow_name", "issuer_did", "target_did", "caller_did",
                        "vc_document", "signature", "storage_uri", "input_hash", "output_hash")
CHAIN_AGENT_NODE_ID_NIL, CHAIN_WORKFLOW_NAME_NIL, CHAIN_VC_DOCUMENT_NIL = 1, 2, 4
CHAIN_BUILT, CHAIN_HOST = 0, 1
DID_KIND_SERVER, DID_KIND_AGENT, DID_KIND_REASONER, DID_KIND_SKILL = 0, 1, 2, 3
DID_IDENTITY_COLUMNS = ("derivation_path", "function_name", "public_key_jwk")
DIDRES_RESOLVE, DIDRES_DOCUMENT = 0, 1
DIDRES_FOUND, DIDRES_NOT_FOUND, DIDRES_BAD_REQUEST, DIDRES_HOST = 0, 1, 2, 3
WEBHOOK_COLUMNS = ("execution_id", "run_id", "status", "node_id", "reasoner_id", "target_type", "timestamp", "error_message")
WEBHOOK_HAS_DURATION, WEBHOOK_HAS_ERROR_MESSAGE, WEBHOOK_HAS_SECRET = 1, 2, 4
WEBHOOK_BUILT, WEBHOOK_HOST = 0, 1
WEBHOOK_HEADER_CHARS = 71
DID_CHARS, DID_PATH_SLOT, DID_KEPT = 55, 48, 1
DIDRR_UNCHANGED, DIDRR_REMOVED, DIDRR_PARTIAL, DIDRR_INVALID = 0, 1, 2, 3
DIDRR_GONE, DIDRR_NEW = 1, 2
MERKLE_STATE_BYTES = 8 + 64 * 32
SHA256_STATE_BYTES = 108

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("AFC_LIB", os.path.join(_HERE, "libafcrypto.so"))   # AFC_LIB: experiment builds only

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
vp = C.c_void_p

# name -> (restype, argtypes): every symbol include/afcrypto.h declares
SYMBOLS = {
    "afc_init": (C.c_int, [C.c_int, C.POINTER(vp)]),
    "afc_destroy": (None, [vp]),
    "afc_strerror": (C.c_char_p, [C.c_int]),
    "afc_last_cuda_error": (C.c_char_p, [vp]),
    "afc_version": (C.c_char_p, []),
    "afc_device_info": (C.c_int, [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), u64p]),
    "afc_launch_count": (C.c_uint64, [vp]),
    "afc_alloc_pinned": (vp, [C.c_size_t]),
    "afc_free_pinned": (None, [vp]),
    "afc_alloc_pinned_for": (vp, [vp, C.c_size_t]),
    "afc_numa_info": (C.c_int, [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "afc_sha256_batch": (C.c_int, [vp, vp, vp, C.c_uint32, vp]),
    "afc_sha256_batch_dev": (C.c_int, [vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_sha256_stream_init": (C.c_int, [vp, C.c_uint32]),
    "afc_sha256_update_batch": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_sha256_update_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp]),
    "afc_hmac_sha256_batch": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp]),
    "afc_hmac_sha256_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_ed25519_verify_batch": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp]),
    "afc_ed25519_verify_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_ed25519_sign_batch": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp]),
    "afc_ed25519_sign_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_ed25519_pubkey_batch": (C.c_int, [vp, vp, C.c_uint32, vp]),
    "afc_ed25519_pubkey_batch_dev": (C.c_int, [vp, vp, C.c_uint32, vp, vp]),
    "afc_ed25519_expand_batch": (C.c_int, [vp, vp, C.c_uint32, vp]),
    "afc_ed25519_expand_batch_dev": (C.c_int, [vp, vp, C.c_uint32, vp, vp]),
    "afc_ed25519_sign_expanded_batch": (C.c_int, [vp, vp, vp, C.c_uint32, vp, vp, C.c_uint32, vp]),
    "afc_ed25519_sign_expanded_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_ed25519_sign_expanded_keys_batch_dev": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_sign_configure": (C.c_int, [vp, C.c_int]),
    "afc_sign_mode": (C.c_int, [vp]),
    "afc_keycache_configure": (C.c_int, [vp, C.c_uint32]),
    "afc_keycache_info": (C.c_int, [vp, u32p, u32p, u32p]),
    "afc_keycache_clear": (C.c_int, [vp, vp]),
    "afc_keycache_stats": (C.c_int, [vp, vp]),
    "afc_keyset_new": (C.c_int, [vp, vp, C.c_uint32, C.POINTER(vp)]),
    "afc_keyset_free": (None, [vp]),
    "afc_keyset_info": (C.c_int, [vp, u32p, u64p]),
    "afc_ed25519_verify_keyed_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint32, vp]),
    "afc_ed25519_verify_keyed_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_keyset_new_named": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.POINTER(vp)]),
    "afc_vc_verify_stored_batch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_uint32, vp, vp]),
    "afc_vc_verify_stored_batch_dev": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_uint32, vp, vp, vp]),
    "afc_vc_verify_json_batch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_uint32, vp, vp]),
    "afc_vc_verify_json_batch_dev": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_uint32, vp, vp, vp]),
    "afc_vc_verify_request_bound": (C.c_uint64, [vp, C.c_uint32]),
    "afc_vc_verify_request_batch": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp]),
    "afc_vc_verify_request_batch_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp]),
    "afc_vc_audit_stored_batch": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_vc_audit_stored_batch_dev": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, C.c_uint32, vp, vp, vp]),
    "afc_vc_issue_bound": (C.c_uint64, [vp, C.c_uint32]),
    "afc_vc_issue_execution_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, C.c_uint32, vp, vp, C.c_uint64, vp, vp,
                                               vp]),
    "afc_vc_issue_execution_batch_dev": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, C.c_uint32, vp, vp, C.c_uint64, vp,
                                                   vp, vp, vp]),
    "afc_vc_workflow_bound": (C.c_uint64, [vp, vp, vp, C.c_uint32]),
    "afc_vc_issue_workflow_batch": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp]),
    "afc_vc_issue_workflow_batch_dev": (C.c_int, [vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp, vp]),
    "afc_did_directory_new": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.POINTER(vp)]),
    "afc_did_directory_free": (None, [vp]),
    "afc_vc_workflow_chain_bound": (C.c_uint64, [vp, vp, vp, vp, vp, C.c_uint32]),
    "afc_vc_workflow_chain_batch": (C.c_int, [vp, vp, C.c_uint32] + [vp] * 16 + [C.c_uint32, vp, C.c_uint64, vp, vp]),
    "afc_vc_workflow_chain_batch_dev": (C.c_int, [vp, vp, C.c_uint32] + [vp] * 16 + [C.c_uint32, vp, C.c_uint64, vp, vp, vp]),
    "afc_did_directory_set_identities": (C.c_int, [vp, vp, vp, vp]),
    "afc_did_resolve_bound": (C.c_uint64, [vp, vp, C.c_uint32]),
    "afc_did_resolve_batch": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp]),
    "afc_did_resolve_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp]),
    "afc_webhook_bound": (C.c_uint64, [vp, vp, C.c_uint32]),
    "afc_webhook_sign_batch": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp]),
    "afc_webhook_sign_batch_dev": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp, C.c_uint64, vp, vp, vp, vp]),
    "afc_did_register_bound": (C.c_uint64, [vp, vp, vp, C.c_uint32, C.c_uint64]),
    "afc_did_register_batch": (C.c_int, [vp, vp, vp, C.c_uint64, vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp]),
    "afc_did_register_batch_dev": (C.c_int, [vp, vp, vp, C.c_uint64, vp, vp, vp, vp, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_uint64, vp,
                                             vp]),
    "afc_did_reregister_bound": (C.c_uint64, [vp, vp, vp, vp, vp, C.c_uint32, C.c_uint64]),
    "afc_did_reregister_batch": (C.c_int, [vp, vp, vp, C.c_uint64] + [vp] * 9 + [C.c_uint32] + [vp] * 9 + [C.c_uint64, vp]),
    "afc_did_reregister_batch_dev": (C.c_int, [vp, vp, vp, C.c_uint64] + [vp] * 9 + [C.c_uint32] + [vp] * 9 + [C.c_uint64, vp, vp]),
    "afc_merkle_new": (C.c_int, [vp, C.POINTER(vp)]),
    "afc_merkle_free": (None, [vp]),
    "afc_merkle_append": (C.c_int, [vp, vp, vp, C.c_uint32, vp, u64p]),
    "afc_merkle_append_dev": (C.c_int, [vp, vp, vp, C.c_uint32, vp]),
    "afc_merkle_append_hashes": (C.c_int, [vp, vp, C.c_uint32, vp, u64p]),
    "afc_merkle_append_hashes_dev": (C.c_int, [vp, vp, C.c_uint32, vp]),
    "afc_merkle_root": (C.c_int, [vp, vp, u64p]),
    "afc_merkle_root_dev": (C.c_int, [vp, vp, vp]),
    "afc_merkle_save": (C.c_int, [vp, vp]),
    "afc_merkle_load": (C.c_int, [vp, vp]),
    "afc_merkle_leaf_hashes_dev": (C.c_int, [vp, vp, vp, C.c_uint32, vp, vp]),
    "afc_merkle_tree_build": (C.c_int, [vp, vp, C.c_uint64, C.POINTER(vp)]),
    "afc_merkle_tree_build_dev": (C.c_int, [vp, vp, C.c_uint64, C.POINTER(vp)]),
    "afc_merkle_tree_free": (None, [vp]),
    "afc_merkle_tree_root": (C.c_int, [vp, vp, u64p, u32p]),
    "afc_merkle_tree_inclusion_proofs": (C.c_int, [vp, vp, C.c_uint32, vp, vp]),
    "afc_merkle_verify_inclusion_batch": (C.c_int, [vp, vp, vp, C.c_uint64, vp, vp, vp, C.c_uint32, vp]),
    "afc_merkle_tree_consistency_proof": (C.c_int, [vp, C.c_uint64, vp, u32p]),
    "afc_merkle_verify_consistency_batch": (C.c_int, [vp, vp, vp, C.c_uint64, vp, vp, vp, C.c_uint32, vp]),
    "afc_comm_unique_id": (C.c_int, [vp]),
    "afc_comm_init": (C.c_int, [vp, C.c_int, C.c_int, vp]),
    "afc_comm_allgather_roots": (C.c_int, [vp, vp, vp]),
    "afc_comm_destroy": (C.c_int, [vp]),
    "afc_b64url_encode_fixed_dev": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, vp, vp]),
    "afc_hex_encode_fixed_dev": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, vp, vp]),
    "afc_json_fill_sizes_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, vp, C.c_uint32, vp, u64p, vp]),
    "afc_json_fill_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, vp, vp, C.c_uint32, vp, vp, vp]),
    "afc_ingest_new": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
    "afc_ingest_free": (None, [vp]),
    "afc_ingest_submit": (C.c_int, [vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, u64p]),
    "afc_ingest_wait": (C.c_int, [vp, C.c_uint64, vp, vp]),
    "afc_ingest_flush": (C.c_int, [vp]),
    "afc_ingest_stats_get": (C.c_int, [vp, vp]),
    "afc_ingest_soak": (C.c_int, [vp, C.c_double, C.c_double, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, vp, C.POINTER(C.c_double), u64p]),
    "afc_selftest": (C.c_int, [vp, C.c_uint32]),
    "afc_staging_find": (C.c_int, [vp, vp, C.c_uint32, u64p]),
    "afc_profile_begin": (C.c_int, [vp, C.c_int]),
    "afc_profile_end": (C.c_int, [vp, vp, C.c_int]),
    "afc_microbench": (C.c_int, [vp, C.c_int, C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
}


class IngestStats(C.Structure):
    _fields_ = [("submitted", C.c_uint64), ("completed", C.c_uint64), ("batches", C.c_uint64), ("avg_batch", C.c_double),
                ("p50_us", C.c_uint32), ("p99_us", C.c_uint32), ("max_us", C.c_uint32), ("log_size", C.c_uint64),
                ("log_root", C.c_uint8 * 32), ("last_error", C.c_int)]


class KeycacheStats(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("max_keys", "cached_keys", "last_hot", "last_cold", "last_distinct", "last_built", "last_evicted",
                                          "total_built", "total_evicted", "calls", "base_window", "base_build_us")] + [
        ("base_table_bytes", C.c_uint64)]


class ProfileEntry(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("count", C.c_uint32), ("total_ms", C.c_double), ("min_ms", C.c_double), ("max_ms", C.c_double)]


class AfcError(RuntimeError):
    def __init__(self, rc, detail=""):
        self.rc = rc
        msg = "afcrypto error %d" % rc
        try:
            msg = "afcrypto: %s (%d)" % (load().afc_strerror(rc).decode(), rc)
        except Exception:
            pass
        if detail:
            msg += ": " + detail
        super().__init__(msg)


_lib = None


def load():
    """dlopen libafcrypto.so; raises if the CUDA extension has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "agentfield_b200: %s is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)       # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def ptr(x):
    """Address of a numpy array / torch tensor / bytes-like / int (device pointer) / None."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    if isinstance(x, (bytes, bytearray)):
        return C.cast(C.c_char_p(bytes(x)), vp).value
    raise TypeError("unsupported buffer type %r" % type(x))


def check(rc, ctx=None):
    if rc < 0:
        detail = ""
        if ctx is not None and rc == AFC_ECUDA:
            detail = load().afc_last_cuda_error(ctx).decode()
        raise AfcError(rc, detail)
    return rc
