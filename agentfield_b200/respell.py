"""Credential documents re-spelled the way clients write them: Python's json.dumps (default, indent=2, ensure_ascii=False,
compact separators), JavaScript's JSON.stringify (also pretty-printed) and CRLF / tab-indented files.  Every number token is kept
exactly as it stood (a plain json.loads / json.dumps round trip would turn -0 into 0).  Used to build inputs for
afc_vc_verify_json_batch in tests and in tools/bench_stored_vc.py."""
import json

from . import _abi


class Num(str):
    """A number token exactly as it stood."""


def parse_keep(doc):
    return json.loads(doc, object_pairs_hook=lambda ps: ("obj", ps), parse_int=Num, parse_float=Num)


def _esc_js(s):
    """JSON.stringify's string escaping (also json.dumps(ensure_ascii=False)): " \\ and control characters only."""
    return json.dumps(s, ensure_ascii=False)


def write(v, *, ascii=True, item=",", key=":", indent=None, nl="\n", esc=None):
    esc = esc or (lambda s: json.dumps(s, ensure_ascii=ascii))

    def w(x, lvl):
        if isinstance(x, Num):
            return str(x)
        if isinstance(x, str):
            return esc(x)
        if x is None or isinstance(x, bool):
            return json.dumps(x)
        if isinstance(x, tuple):
            items = [esc(k) + key + w(y, lvl + 1) for k, y in x[1]]
            o, c = "{", "}"
        else:
            items = [w(y, lvl + 1) for y in x]
            o, c = "[", "]"
        if not items:
            return o + c
        if indent is None:
            return o + item.join(items) + c
        pad, pad0 = nl + indent * (lvl + 1), nl + indent * lvl
        return o + pad + ("," + pad).join(items) + pad0 + c
    return w(v, 0)


SPELLINGS = {
    "indent2": lambda v: write(v, key=": ", indent="  "),                                  # json.dumps(doc, indent=2)
    "dumps": lambda v: write(v, item=", ", key=": "),                                      # json.dumps(doc): what requests sends
    "no_ascii": lambda v: write(v, ascii=False, item=", ", key=": "),                      # json.dumps(doc, ensure_ascii=False)
    "compact": lambda v: write(v),                                                         # separators=(",", ":")
    "js_pretty": lambda v: write(v, key=": ", indent="  ", esc=_esc_js),                   # JSON.stringify(doc, null, 2)
    "crlf_tab": lambda v: write(v, ascii=False, key=" :\t", indent="\t", nl="\r\n"),       # CRLF lines, tab indentation
}


def spell(doc, how):
    return SPELLINGS[how](parse_keep(doc)).encode("utf-8")


def respelled_stored_vcs_dev(ctx, dev, n, K, seed, how, distinct=1 << 16):
    """n execution VCs from K issuers in one client spelling: `distinct` documents built on the device (synthetic_stored_vcs_dev),
    re-spelled on the host with every number token kept, tiled to n, then 1 % (i % 100 == 37) with a corrupted signature.  how:
    None for the canonical bytes, else a key of SPELLINGS.  Returns (d_docs, d_doc_off int64, the named KeySet,
    the planted statuses)."""
    import numpy as np
    import torch
    from . import canonical as CA
    from .identity import ExpandedKeys, KeySet
    rng = np.random.default_rng(seed)
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (7000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    m = min(n, distinct)
    d_ki = (torch.arange(m, device=dev) % K).to(torch.int32)
    d_docs, d_doff, _, _, _ = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, m, seed=seed)
    buf, off = d_docs.cpu().numpy(), d_doff.cpu().numpy()
    docs = [buf[off[i]:off[i + 1]].tobytes() for i in range(m)]
    if how is not None:
        docs = [spell(d, how) for d in docs]
    pv = np.array([d.index(b'"proofValue"') + 20 for d in docs], dtype=np.int64)      # a character inside the proofValue
    lens = np.array([len(d) for d in docs], dtype=np.int64)
    one = np.frombuffer(b"".join(docs), dtype=np.uint8)
    reps = (n + m - 1) // m
    cat = np.tile(one, reps)
    l_all = np.tile(lens, reps)[:n]
    d_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(l_all, out=d_off[1:])
    cat = cat[:d_off[-1]]
    bad = np.arange(n) % 100 == 37
    at = d_off[:-1][bad] + np.tile(pv, reps)[:n][bad]
    cat = cat.copy()
    cat[at] = np.where(cat[at] == 0x41, 0x42, 0x41)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    want = torch.from_numpy(np.where(bad, _abi.VC_INVALID, _abi.VC_VALID).astype(np.uint8)).to(dev)
    return torch.from_numpy(cat).to(dev), torch.from_numpy(d_off).to(dev), ks, want
