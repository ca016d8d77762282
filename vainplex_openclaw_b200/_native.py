"""ctypes binding of the C ABI in include/openclaw_gov.h (the same symbols the Node N-API shim binds).

There is no CPU fallback: if the shared library is missing or no CUDA device is usable, every
compute entry point raises GovError -- the caller's failMode decides (reference: src/hooks.ts:232-241).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _build

CG_OK = 0
ERR_NAMES = {-1: "INVALID_ARG", -2: "NOT_INITIALIZED", -3: "CUDA", -4: "SYNTAX", -5: "UNSUPPORTED",
             -6: "TOO_LARGE", -7: "CAPACITY", -8: "NOMEM"}
CG_ERR_SYNTAX, CG_ERR_UNSUPPORTED, CG_ERR_TOO_LARGE, CG_ERR_CAPACITY = -4, -5, -6, -7
FLAG_ICASE = 1
CAT = {"credential": 0, "financial": 1, "pii": 2, "custom": 3}
OPT_STRIDE_AUTO, OPT_STRIDE2, OPT_STRIDE4 = 0, 2, 4


class GovError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("openclaw_gov: %s (%d): %s" % (ERR_NAMES.get(code, "?"), code, msg))
        self.code = code


class cg_rule(C.Structure):
    _fields_ = [("source", C.c_char_p), ("source_len", C.c_uint32), ("flags", C.c_uint32), ("category", C.c_uint32)]


class cg_ruleset_info(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_rules", "n_ok", "n_always_candidate", "n_sets", "stride", "gram_keys",
                                          "gram_entries", "factor_len", "image_bytes", "program_words", "n_factors",
                                          "bitmap_bytes", "n_triggers", "tables_resident")]


class cg_stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("messages_scanned", "bytes_scanned", "candidate_events", "verified_pairs",
                                          "hits", "spans", "sha256_items", "merkle_leaves", "kernel_launches")] + \
               [("last_scan_ms", C.c_double), ("last_merkle_ms", C.c_double)]


HIT_DTYPE = np.dtype([("msg", np.uint32), ("rule", np.uint32)])
SPAN_DTYPE = np.dtype([("msg", np.uint32), ("rule", np.uint32), ("start_byte", np.uint32), ("end_byte", np.uint32),
                       ("start16", np.uint32), ("end16", np.uint32)])

EXPORTS = ["cg_init", "cg_shutdown", "cg_last_error", "cg_version", "cg_device_count", "cg_get_stats", "cg_launch_count",
           "cg_set_profiling", "cg_last_kernel_ms", "cg_last_tail_ms", "cg_scan_work_counters", "cg_scan_join", "cg_redact_batch", "cg_ruleset_set_policy", "cg_policy_verdict_batch",
           "cg_merkle_log_create", "cg_merkle_log_destroy", "cg_merkle_log_append", "cg_merkle_log_size", "cg_merkle_log_root",
           "cg_merkle_log_frontier", "cg_merkle_log_restore", "cg_merkle_log_proof", "cg_merkle_verify_proof",
           "cg_merkle_log_append_jsonl", "cg_merkle_log_consistency", "cg_merkle_verify_consistency", "cg_merkle_log_reserve",
           "cg_shard_range", "cg_comm_unique_id", "cg_comm_init", "cg_comm_destroy", "cg_merkle_root_sharded_device",
           "cg_ruleset_create", "cg_ruleset_destroy", "cg_ruleset_get_info", "cg_rule_check", "cg_scan_batch",
           "cg_scan_one", "cg_find_matches_batch", "cg_scan_batch_device", "cg_find_matches_batch_device", "cg_redact_batch_device", "cg_sha256_batch", "cg_merkle_root",
           "cg_merkle_root_fixed", "cg_merkle_block_roots_device", "cg_merkle_fold", "cg_merkle_fold_device"]

_lib = None


def lib_path() -> str:
    return _build.LIB


def load():
    """dlopen the in-tree library (building it first when sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    if _build.needs_build():
        if os.path.exists("/usr/local/cuda/bin/nvcc") or os.environ.get("NVCC"):
            _build.build()
        elif not os.path.exists(_build.LIB):
            raise GovError(-2, "libopenclaw_gov.so is not built and nvcc is unavailable")
    L = C.CDLL(_build.LIB)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.cg_init.argtypes = [i32]; L.cg_init.restype = i32
    L.cg_shutdown.restype = None
    L.cg_last_error.restype = C.c_char_p
    L.cg_version.restype = i32
    L.cg_device_count.restype = i32
    L.cg_get_stats.argtypes = [C.POINTER(cg_stats)]; L.cg_get_stats.restype = i32
    L.cg_launch_count.restype = u64
    L.cg_set_profiling.argtypes = [i32]; L.cg_set_profiling.restype = i32
    L.cg_last_kernel_ms.argtypes = [vp]; L.cg_last_kernel_ms.restype = i32
    L.cg_last_tail_ms.argtypes = [vp]; L.cg_last_tail_ms.restype = i32
    L.cg_scan_work_counters.argtypes = [vp, vp]; L.cg_scan_work_counters.restype = i32
    L.cg_scan_join.argtypes = [vp, vp]; L.cg_scan_join.restype = i32
    L.cg_redact_batch.argtypes = [vp, vp, vp, u32, vp, u64, vp, vp, vp, u32, vp, vp]; L.cg_redact_batch.restype = i32
    L.cg_ruleset_set_policy.argtypes = [vp, vp, vp, u32]; L.cg_ruleset_set_policy.restype = i32
    L.cg_policy_verdict_batch.argtypes = [vp, vp, vp, u32, vp]; L.cg_policy_verdict_batch.restype = i32
    L.cg_merkle_log_create.argtypes = [vp, i32]; L.cg_merkle_log_create.restype = i32
    L.cg_merkle_log_destroy.argtypes = [vp]; L.cg_merkle_log_destroy.restype = None
    L.cg_merkle_log_append.argtypes = [vp, vp, vp, u64]; L.cg_merkle_log_append.restype = i32
    L.cg_merkle_log_size.argtypes = [vp, vp]; L.cg_merkle_log_size.restype = i32
    L.cg_merkle_log_root.argtypes = [vp, vp]; L.cg_merkle_log_root.restype = i32
    L.cg_merkle_log_frontier.argtypes = [vp, vp, vp]; L.cg_merkle_log_frontier.restype = i32
    L.cg_merkle_log_restore.argtypes = [vp, u64, vp, u32]; L.cg_merkle_log_restore.restype = i32
    L.cg_merkle_log_proof.argtypes = [vp, u64, vp, u32, vp]; L.cg_merkle_log_proof.restype = i32
    L.cg_merkle_verify_proof.argtypes = [vp, u64, u64, u64, vp, u32, vp, vp]; L.cg_merkle_verify_proof.restype = i32
    L.cg_merkle_log_append_jsonl.argtypes = [vp, vp, u64, vp]; L.cg_merkle_log_append_jsonl.restype = i32
    L.cg_merkle_log_reserve.argtypes = [vp, u64, u64]; L.cg_merkle_log_reserve.restype = i32
    L.cg_shard_range.argtypes = [u64, i32, i32, u64, vp, vp]; L.cg_shard_range.restype = None
    L.cg_comm_unique_id.argtypes = [vp]; L.cg_comm_unique_id.restype = i32
    L.cg_comm_init.argtypes = [i32, i32, vp]; L.cg_comm_init.restype = i32
    L.cg_comm_destroy.argtypes = []; L.cg_comm_destroy.restype = None
    L.cg_merkle_root_sharded_device.argtypes = [vp, u64, u64, u64, u32, vp, vp]; L.cg_merkle_root_sharded_device.restype = i32
    L.cg_merkle_log_consistency.argtypes = [vp, u64, vp, u32, vp]; L.cg_merkle_log_consistency.restype = i32
    L.cg_merkle_verify_consistency.argtypes = [u64, u64, vp, vp, vp, u32, vp]; L.cg_merkle_verify_consistency.restype = i32
    L.cg_ruleset_create.argtypes = [C.POINTER(cg_rule), u32, u32, C.POINTER(vp), vp]; L.cg_ruleset_create.restype = i32
    L.cg_ruleset_destroy.argtypes = [vp]; L.cg_ruleset_destroy.restype = None
    L.cg_ruleset_get_info.argtypes = [vp, C.POINTER(cg_ruleset_info)]; L.cg_ruleset_get_info.restype = i32
    L.cg_rule_check.argtypes = [C.c_char_p, u32, u32, C.c_char_p, u32]; L.cg_rule_check.restype = i32
    L.cg_scan_batch.argtypes = [vp, vp, vp, u32, vp, vp, u32, C.POINTER(u32)]; L.cg_scan_batch.restype = i32
    L.cg_scan_one.argtypes = [vp, vp, u32, C.POINTER(u64), vp, u32, C.POINTER(u32)]; L.cg_scan_one.restype = i32
    L.cg_find_matches_batch.argtypes = [vp, vp, vp, u32, vp, u32, C.POINTER(u32)]; L.cg_find_matches_batch.restype = i32
    L.cg_scan_batch_device.argtypes = [vp, vp, vp, u32, vp, vp]; L.cg_scan_batch_device.restype = i32
    L.cg_find_matches_batch_device.argtypes = [vp, vp, vp, u32, vp, u32, vp, vp]; L.cg_find_matches_batch_device.restype = i32
    L.cg_redact_batch_device.argtypes = [vp, vp, vp, u32, vp, u64, vp, vp, u32, vp, vp, vp]; L.cg_redact_batch_device.restype = i32
    L.cg_sha256_batch.argtypes = [vp, vp, u32, vp]; L.cg_sha256_batch.restype = i32
    L.cg_merkle_root.argtypes = [vp, vp, u64, vp]; L.cg_merkle_root.restype = i32
    L.cg_merkle_root_fixed.argtypes = [vp, u64, u64, vp]; L.cg_merkle_root_fixed.restype = i32
    L.cg_merkle_block_roots_device.argtypes = [vp, u64, u64, u32, vp, vp]; L.cg_merkle_block_roots_device.restype = i32
    L.cg_merkle_fold.argtypes = [vp, u64, vp]; L.cg_merkle_fold.restype = i32
    L.cg_merkle_fold_device.argtypes = [vp, u64, vp, vp]; L.cg_merkle_fold_device.restype = i32
    _lib = L
    return L


def check(rc: int):
    if rc != CG_OK:
        raise GovError(rc, (load().cg_last_error() or b"").decode("utf-8", "replace"))


_inited = False


def init(device: int = -1):
    """cg_init; raises GovError(CUDA) when no sm_90 (H100-class) device is present."""
    global _inited
    check(load().cg_init(device))
    _inited = True


def rule_check(source: str, flags: int = 0) -> int:
    """What would `new RegExp(source)` do: CG_OK, CG_ERR_SYNTAX, or CG_ERR_UNSUPPORTED/TOO_LARGE (no device needed)."""
    b = js_utf8(source)
    return load().cg_rule_check(b, len(b), flags, None, 0)


def js_utf8(s: str) -> bytes:
    """Buffer.from(str,'utf8'): lone surrogates become U+FFFD."""
    try:
        return s.encode("utf-8")
    except UnicodeEncodeError:
        return s.encode("utf-16-le", "surrogatepass").decode("utf-16-le", "replace").encode("utf-8")


def pack(messages) -> tuple[np.ndarray, np.ndarray]:
    """list of bytes -> (uint8 buffer padded by 64 bytes, uint32 offsets[n+1])."""
    off = np.zeros(len(messages) + 1, dtype=np.uint32)
    if len(messages):
        off[1:] = np.cumsum([len(m) for m in messages], dtype=np.uint64).astype(np.uint32)
    data = np.frombuffer(b"".join(messages) + b"\0" * 64, dtype=np.uint8).copy()
    return data, off


class Ruleset:
    """cg_ruleset handle.  rules: iterable of (source:str|bytes, flags:int, category:int)."""

    def __init__(self, rules, options: int = OPT_STRIDE_AUTO, strict: bool = False):
        L = load()
        if not _inited:
            init()
        rules = list(rules)
        self._keep = [r[0] if isinstance(r[0], bytes) else js_utf8(r[0]) for r in rules]
        arr = (cg_rule * max(1, len(rules)))()
        for i, r in enumerate(rules):
            arr[i].source = self._keep[i]; arr[i].source_len = len(self._keep[i])
            arr[i].flags = r[1]; arr[i].category = r[2]
        self.status = np.zeros(max(1, len(rules)), dtype=np.int32)
        h = C.c_void_p()
        check(L.cg_ruleset_create(arr, len(rules), options, C.byref(h), None if strict else self.status.ctypes.data))
        self.handle = h
        self.n_rules = len(rules)
        self.status = self.status[:len(rules)]

    def close(self):
        if getattr(self, "handle", None):
            load().cg_ruleset_destroy(self.handle)
            self.handle = None

    __del__ = close

    def info(self) -> cg_ruleset_info:
        o = cg_ruleset_info()
        check(load().cg_ruleset_get_info(self.handle, C.byref(o)))
        return o

    def scan_batch(self, data: np.ndarray, off: np.ndarray, want_hits: bool = True):
        """-> (words[n] uint64, hits structured array sorted by (msg, rule))."""
        n = len(off) - 1
        words = np.zeros(max(n, 1), dtype=np.uint64)
        nh = C.c_uint32(0)
        cap = 1024
        while True:
            hits = np.zeros(cap, dtype=HIT_DTYPE)
            rc = load().cg_scan_batch(self.handle, data.ctypes.data, off.ctypes.data, n, words.ctypes.data,
                                      hits.ctypes.data if want_hits else None, cap, C.byref(nh))
            if rc == CG_ERR_CAPACITY and nh.value > cap:
                cap = nh.value
                continue
            check(rc)
            return words[:n], hits[:nh.value]

    def scan_one(self, msg: bytes):
        """The synchronous hooks' path (before_message_write / tool_result_persist): one message, blocking.
        -> (word, [hit rule indices])"""
        buf = np.frombuffer(msg + b"\0" * 64, dtype=np.uint8)
        word, nr = C.c_uint64(0), C.c_uint32(0)
        rules = np.zeros(max(64, self.n_rules), dtype=np.uint32)
        check(load().cg_scan_one(self.handle, buf.ctypes.data, len(msg), C.byref(word), rules.ctypes.data, len(rules), C.byref(nr)))
        return word.value, [int(x) for x in rules[:nr.value]]

    def find_matches_batch(self, data: np.ndarray, off: np.ndarray):
        """-> spans structured array, resolved per registry.ts:288-316, sorted by (msg, start)."""
        n = len(off) - 1
        ns = C.c_uint32(0)
        cap = 1024
        while True:
            spans = np.zeros(cap, dtype=SPAN_DTYPE)
            rc = load().cg_find_matches_batch(self.handle, data.ctypes.data, off.ctypes.data, n, spans.ctypes.data, cap, C.byref(ns))
            if rc == CG_ERR_CAPACITY and ns.value > cap:
                cap = ns.value
                continue
            check(rc)
            return spans[:ns.value]

    def set_policy(self, rule_policy, rule_action):
        """rule i belongs to policy rule_policy[i] (evaluation order, non-decreasing) with effect rule_action[i] (0 allow, 1 audit, 2 deny)."""
        pol = np.ascontiguousarray(rule_policy, dtype=np.uint32); act = np.ascontiguousarray(rule_action, dtype=np.uint8)
        check(load().cg_ruleset_set_policy(self.handle, pol.ctypes.data, act.ctypes.data, len(pol)))

    def verdict_batch(self, data: np.ndarray, off: np.ndarray) -> np.ndarray:
        """-> uint32 verdict per message: action | matched policies << 2 | deciding rule << 12 (openclaw_gov.h)."""
        n = len(off) - 1
        out = np.zeros(max(n, 1), dtype=np.uint32)
        check(load().cg_policy_verdict_batch(self.handle, data.ctypes.data, off.ctypes.data, n, out.ctypes.data))
        return out[:n]

    def redact_batch(self, data: np.ndarray, off: np.ndarray):
        """RedactionEngine.scanString for a batch, spliced on the device.
        -> (out_bytes uint8[..], out_offsets uint32[n+1], resolved spans, digests uint8[ns, 32])"""
        n = len(off) - 1
        total = int(off[n]) if n else 0
        out_off = np.zeros(n + 1, dtype=np.uint32)
        need, ns = C.c_uint64(0), C.c_uint32(0)
        cap_bytes, cap_spans = total + 4096, 1024
        while True:
            out = np.zeros(cap_bytes + 64, dtype=np.uint8)
            spans = np.zeros(cap_spans, dtype=SPAN_DTYPE)
            dig = np.zeros((cap_spans, 32), dtype=np.uint8)
            rc = load().cg_redact_batch(self.handle, data.ctypes.data, off.ctypes.data, n, out.ctypes.data, cap_bytes, C.byref(need),
                                        out_off.ctypes.data, spans.ctypes.data, cap_spans, C.byref(ns), dig.ctypes.data)
            if rc == CG_ERR_CAPACITY and (need.value > cap_bytes or ns.value > cap_spans):
                cap_bytes, cap_spans = max(cap_bytes, need.value), max(cap_spans, ns.value)
                continue
            check(rc)
            return out[:need.value], out_off, spans[:ns.value], dig[:ns.value]

    def work_counters(self):
        """(slots, VM pairs, spans, error flags, confirmed factor occurrences, cursor, flagged grams, ...) of the last step whose
        counters reached the host (device path: after scan_join)."""
        out = np.zeros(16, dtype=np.uint32)
        check(load().cg_scan_work_counters(self.handle, out.ctypes.data))
        return tuple(int(x) for x in out)

    def scan_join(self, stream: int = 0):
        """Wait for `stream`; raises if a batch issued through scan_batch_device since the last join overflowed a queue
        (its result words are all ones) -- the scratch has been grown, scan it again."""
        check(load().cg_scan_join(self.handle, stream))

    def scan_batch_device(self, d_bytes: int, d_off: int, n: int, d_words: int, stream: int = 0):
        check(load().cg_scan_batch_device(self.handle, d_bytes, d_off, n, d_words, stream))

    def find_matches_batch_device(self, d_bytes: int, d_off: int, n: int, d_spans: int, spans_cap: int, d_nspans: int, stream: int = 0):
        """cg_find_matches_batch_device on raw device pointers (asynchronous; status from scan_join): resolved spans
        (SPAN_DTYPE, at most spans_cap) into d_spans, their number (uint32) into d_nspans."""
        check(load().cg_find_matches_batch_device(self.handle, d_bytes, d_off, n, d_spans or None, spans_cap, d_nspans, stream))

    def redact_batch_device(self, d_bytes: int, d_off: int, n: int, d_out: int, out_cap: int, d_out_off: int, d_spans: int,
                            spans_cap: int, d_digests: int, d_sizes: int, stream: int = 0):
        """cg_redact_batch_device on raw device pointers (asynchronous; status from scan_join): redacted bytes into d_out,
        offsets (uint32[n+1]) into d_out_off, spans and their SHA-256 (32 bytes each) into d_spans / d_digests, and
        uint64[2] = (bytes needed, resolved spans) into d_sizes."""
        check(load().cg_redact_batch_device(self.handle, d_bytes, d_off, n, d_out or None, out_cap, d_out_off, d_spans or None,
                                            spans_cap, d_digests or None, d_sizes, stream))


def sha256_batch(data: np.ndarray, off64: np.ndarray) -> np.ndarray:
    if not _inited:
        init()
    n = len(off64) - 1
    out = np.zeros((max(n, 1), 32), dtype=np.uint8)
    check(load().cg_sha256_batch(data.ctypes.data, off64.ctypes.data, n, out.ctypes.data))
    return out[:n]


def merkle_root(data: np.ndarray, off64: np.ndarray) -> bytes:
    if not _inited:
        init()
    out = np.zeros(32, dtype=np.uint8)
    check(load().cg_merkle_root(data.ctypes.data, off64.ctypes.data, len(off64) - 1, out.ctypes.data))
    return out.tobytes()


def merkle_root_fixed(data: np.ndarray, leaf_len: int, n: int) -> bytes:
    if not _inited:
        init()
    out = np.zeros(32, dtype=np.uint8)
    check(load().cg_merkle_root_fixed(data.ctypes.data, leaf_len, n, out.ctypes.data))
    return out.tobytes()


def merkle_fold(nodes: np.ndarray) -> bytes:
    if not _inited:
        init()
    nodes = np.ascontiguousarray(nodes, dtype=np.uint8)
    out = np.zeros(32, dtype=np.uint8)
    check(load().cg_merkle_fold(nodes.ctypes.data, nodes.shape[0], out.ctypes.data))
    return out.tobytes()


def stats() -> cg_stats:
    s = cg_stats()
    check(load().cg_get_stats(C.byref(s)))
    return s


def set_profiling(on: bool):
    check(load().cg_set_profiling(1 if on else 0))


def last_kernel_ms():
    """(scan_ms, confirm_ms, verify_ms, finalize_ms) of the last completed scan step (profiling must be on)."""
    out = np.zeros(4, dtype=np.float32)
    check(load().cg_last_kernel_ms(out.ctypes.data))
    return tuple(float(x) for x in out)


def last_tail_ms():
    """(confirm_kernel_ms, resolve_kernel_ms) of the last completed scan step (profiling must be on)."""
    out = np.zeros(2, dtype=np.float32)
    check(load().cg_last_tail_ms(out.ctypes.data))
    return tuple(float(x) for x in out)


def launch_count() -> int:
    return int(load().cg_launch_count())


class MerkleLog:
    """cg_merkle_log: append-only Merkle tree over event-log leaves (frontier state, optional audit paths)."""

    def __init__(self, keep_leaf_digests: bool = True, _handle=None):
        if _handle is not None:
            self.handle = _handle
            return
        h = C.c_void_p()
        check(load().cg_merkle_log_create(C.byref(h), 1 if keep_leaf_digests else 0))
        self.handle = h

    @classmethod
    def restore(cls, n: int, frontier: np.ndarray):
        f = np.ascontiguousarray(frontier, dtype=np.uint8)
        h = C.c_void_p()
        check(load().cg_merkle_log_restore(C.byref(h), n, f.ctypes.data, f.shape[0] if f.size else 0))
        return cls(_handle=h)

    def append(self, leaves):
        """leaves: list of bytes."""
        if not leaves:
            return
        off = np.zeros(len(leaves) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(x) for x in leaves])
        data = np.frombuffer(b"".join(leaves) + b"\0" * 64, dtype=np.uint8).copy()
        check(load().cg_merkle_log_append(self.handle, data.ctypes.data, off.ctypes.data, len(leaves)))

    def reserve(self, n_leaves: int, n_bytes: int = 0):
        check(load().cg_merkle_log_reserve(self.handle, n_leaves, n_bytes))

    def append_packed(self, data: np.ndarray, off64: np.ndarray):
        """leaves already packed: data uint8, off64 uint64 (m + 1 entries)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        off64 = np.ascontiguousarray(off64, dtype=np.uint64)
        check(load().cg_merkle_log_append(self.handle, data.ctypes.data, off64.ctypes.data, len(off64) - 1))

    def append_jsonl(self, data) -> int:
        """the day file's bytes (JSON lines, src/audit-trail.ts:151-179); returns the number of lines appended."""
        buf = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)
        k = C.c_uint64(0)
        check(load().cg_merkle_log_append_jsonl(self.handle, buf.ctypes.data if buf.size else None, buf.size, C.byref(k)))
        return k.value

    def consistency(self, first_size: int):
        out = np.zeros((64, 32), dtype=np.uint8)
        k = C.c_uint32(0)
        check(load().cg_merkle_log_consistency(self.handle, first_size, out.ctypes.data, 64, C.byref(k)))
        return [out[i].tobytes() for i in range(k.value)]

    def size(self) -> int:
        n = C.c_uint64(0)
        check(load().cg_merkle_log_size(self.handle, C.byref(n)))
        return n.value

    def root(self) -> bytes:
        out = np.zeros(32, dtype=np.uint8)
        check(load().cg_merkle_log_root(self.handle, out.ctypes.data))
        return out.tobytes()

    def frontier(self) -> np.ndarray:
        out = np.zeros((64, 32), dtype=np.uint8)
        k = C.c_uint32(0)
        check(load().cg_merkle_log_frontier(self.handle, out.ctypes.data, C.byref(k)))
        return out[:k.value].copy()

    def proof(self, index: int):
        out = np.zeros((64, 32), dtype=np.uint8)
        k = C.c_uint32(0)
        check(load().cg_merkle_log_proof(self.handle, index, out.ctypes.data, 64, C.byref(k)))
        return [out[i].tobytes() for i in range(k.value)]

    def close(self):
        if self.handle:
            load().cg_merkle_log_destroy(self.handle)
            self.handle = None


def shard_range(n: int, rank: int, world: int, align: int = 1):
    """cg_shard_range: this rank's contiguous [lo, hi); needs no device."""
    lo, hi = C.c_uint64(0), C.c_uint64(0)
    load().cg_shard_range(n, rank, world, align, C.byref(lo), C.byref(hi))
    return lo.value, hi.value


def comm_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    check(load().cg_comm_unique_id(buf))
    return buf.raw


def comm_init(rank: int, world: int, uid: bytes):
    buf = C.create_string_buffer(uid, 128)
    check(load().cg_comm_init(rank, world, buf))


def comm_destroy():
    load().cg_comm_destroy()


def merkle_root_sharded_device(d_ptr: int, leaf_len: int, n_local: int, n_total: int, block_log2: int, stream: int = 0) -> bytes:
    out = np.zeros(32, dtype=np.uint8)
    check(load().cg_merkle_root_sharded_device(d_ptr, leaf_len, n_local, n_total, block_log2, out.ctypes.data, stream))
    return out.tobytes()


def merkle_verify_consistency(first_size: int, second_size: int, root_first: bytes, root_second: bytes, path) -> bool:
    p = np.frombuffer(b"".join(path) + b"\0" * 32, dtype=np.uint8).copy()
    r1 = np.frombuffer(root_first, dtype=np.uint8).copy()
    r2 = np.frombuffer(root_second, dtype=np.uint8).copy()
    ok = C.c_int(0)
    check(load().cg_merkle_verify_consistency(first_size, second_size, r1.ctypes.data, r2.ctypes.data, p.ctypes.data, len(path), C.byref(ok)))
    return bool(ok.value)


def merkle_verify_proof(leaf: bytes, index: int, tree_size: int, path, root: bytes) -> bool:
    p = np.frombuffer(b"".join(path) + b"\0" * 32, dtype=np.uint8).copy()
    lb = np.frombuffer(leaf + b"\0", dtype=np.uint8).copy()
    r = np.frombuffer(root, dtype=np.uint8).copy()
    ok = C.c_int(0)
    check(load().cg_merkle_verify_proof(lb.ctypes.data, len(leaf), index, tree_size, p.ctypes.data, len(path), r.ctypes.data, C.byref(ok)))
    return bool(ok.value)
