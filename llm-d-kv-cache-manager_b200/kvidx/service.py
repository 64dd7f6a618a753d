"""The callers either side of the hot path, around the C ABI: text in, KVEvents in, gRPC out.

    IndexerService   api/indexer.proto:24-43 -- `indexer.v1.IndexerService/GetPodScores`, the reference's one network surface
                     (examples/kv_cache_index_service/server/server.go:70-96): unwrap the request, GetPodScores(prompt, model,
                     pods), flatten the map into repeated PodScore.  One handler thread per RPC, like the reference's goroutine per
                     RPC; concurrent RPCs meet in libkvidx's submission queue and share launches.
    TokenizationPool pkg/tokenization/pool.go:149-237 -- prompt text -> token ids through the HF `tokenizers` core (the same Rust
                     library the reference links), behind the prefix store (kvhost_prefix_store_*, lru_store.go:93-190) with the
                     reference's reuse rule (overlap ratio >= 0.8 returns the cached prefix's tokens).
    ZmqSubscriber    pkg/kvcache/kvevents/zmq_subscriber.go:81-162 -- SUB socket that BINDS (:90), 250 ms poll (:112), 3-part
                     messages [topic "kv@<pod>@<model>", 8-byte big-endian sequence, msgpack payload] (:124-144) -> Pool.AddTask;
                     a drain loop turns what has queued up into one kvidx_apply_events batch (kvhost_pool_process).

Go is not in this image, so this layer is Python over the C++ host mirror (include/kvidx_host.h); the message classes are
built from the proto's descriptor at import time (no protoc here either) and are wire-compatible with the reference's stubs.
"""
from __future__ import annotations

import threading
import time
from concurrent import futures
from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np

SERVICE = "indexer.v1.IndexerService"
METHOD = "/%s/GetPodScores" % SERVICE


# ---- api/indexer.proto as a descriptor (same package, message and field names, numbers and types) ----------------
def _build_messages():
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fd = descriptor_pb2.FileDescriptorProto()
    fd.name = "kvidx/indexer.proto"
    fd.package = "indexer.v1"
    fd.syntax = "proto3"
    T = descriptor_pb2.FieldDescriptorProto

    def msg(name, fields):
        m = fd.message_type.add()
        m.name = name
        for fname, num, ftype, label, tname in fields:
            f = m.field.add()
            f.name, f.number, f.type, f.label = fname, num, ftype, label
            if tname:
                f.type_name = tname
    msg("GetPodScoresRequest", [("prompt", 1, T.TYPE_STRING, T.LABEL_OPTIONAL, None), ("model_name", 2, T.TYPE_STRING, T.LABEL_OPTIONAL, None),
                                ("pod_identifiers", 3, T.TYPE_STRING, T.LABEL_REPEATED, None)])
    msg("PodScore", [("pod", 1, T.TYPE_STRING, T.LABEL_OPTIONAL, None), ("score", 2, T.TYPE_DOUBLE, T.LABEL_OPTIONAL, None)])
    msg("GetPodScoresResponse", [("scores", 1, T.TYPE_MESSAGE, T.LABEL_REPEATED, ".indexer.v1.PodScore")])
    svc = fd.service.add()
    svc.name = "IndexerService"
    mth = svc.method.add()
    mth.name, mth.input_type, mth.output_type = "GetPodScores", ".indexer.v1.GetPodScoresRequest", ".indexer.v1.GetPodScoresResponse"
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    get = message_factory.GetMessageClass
    return (get(pool.FindMessageTypeByName("indexer.v1.GetPodScoresRequest")), get(pool.FindMessageTypeByName("indexer.v1.GetPodScoresResponse")),
            get(pool.FindMessageTypeByName("indexer.v1.PodScore")))


GetPodScoresRequest, GetPodScoresResponse, PodScore = _build_messages()


# ---- tokenization front end ------------------------------------------------------------------------------------------
class TokenizationPool:
    """tokenization.Pool.processTask (pool.go:198-237) without the chat-template branch (BASELINE passes raw prompts):
    FindLongestContainedTokens; if the overlap ratio is below minPrefixOverlapRatio (0.8, pool.go:31-34) Encode with
    add_special_tokens=False (tokenizer.go:411) and AddTokenization; else the cached prefix's tokens."""

    def __init__(self, tokenizer=None, tokenizer_file: Optional[str] = None, min_prefix_overlap_ratio: float = 0.8, store=None):
        from .host import PrefixStore
        if tokenizer is None:
            from tokenizers import Tokenizer
            tokenizer = Tokenizer.from_file(tokenizer_file)
        self.tokenizer = tokenizer
        self.ratio = min_prefix_overlap_ratio
        self.store = store if store is not None else PrefixStore()
        self._mu = threading.Lock()          # the store is one LRU (the reference's is behind a mutex too, lru_store.go:58)
        self.encodes = 0

    def _encode(self, prompt: str):
        enc = self.tokenizer.encode(prompt, add_special_tokens=False)
        ids, offs = enc.ids, enc.offsets
        if not prompt.isascii():             # HF reports CHARACTER offsets for a str; the store slices BYTES like Go strings do
            cum = np.zeros(len(prompt) + 1, np.int64)
            cum[1:] = np.cumsum([len(ch.encode("utf-8")) for ch in prompt])
            offs = [(int(cum[a]), int(cum[b])) for a, b in offs]
        return ids, offs

    def tokenize(self, prompt: str) -> List[int]:
        raw = prompt.encode("utf-8")
        with self._mu:
            tokens, ratio = self.store.find_longest_contained_tokens(raw)
        if ratio < self.ratio:
            ids, offs = self._encode(prompt)
            self.encodes += 1
            with self._mu:
                self.store.add_tokenization(raw, ids, offs)
            return list(ids)
        return tokens


# ---- Indexer over the host mirror --------------------------------------------------------------------------------------
class Indexer:
    """kvcache.Indexer (indexer.go:132-166): Tokenize -> (TokensToKVBlockKeys -> Lookup -> Score on the device).

    get_pod_scores serves one prompt through the TokenizationPool's host prefix store (a device round trip costs more than
    the host store's lookup for a single prompt).  get_pod_scores_batch serves a batch through a prefix store on the device
    (kvidx_text_store_*, created on first use with text_cache_blocks / text_block_bytes): one Score() from text, the
    tokenizer for the prompts whose cached prefix is too short, one add and one Score() for those."""

    def __init__(self, host_indexer, tokenization: TokenizationPool, text_cache_blocks: int = 500000, text_block_bytes: int = 256):
        self.host = host_indexer
        self.tok = tokenization
        self.text_cache_blocks, self.text_block_bytes = text_cache_blocks, text_block_bytes
        self._dev = None
        self._dev_mu = threading.Lock()

    def get_pod_scores(self, prompt: str, model_name: str, pod_identifiers: Sequence[str] = ()) -> Optional[Dict[str, float]]:
        tokens = self.tok.tokenize(prompt)
        return self.host.get_pod_scores(np.asarray(tokens, np.uint32), model_name, list(pod_identifiers))

    def _device_store(self):
        with self._dev_mu:
            if self._dev is None:
                from ._native import Index
                ix = Index.borrow(self.host.L.kvhost_index(self.host.h), self.host.block_size, self.host.max_pods)
                ix.text_store_init(self.text_cache_blocks, self.text_block_bytes)
                self._dev = ix
            return self._dev

    def text_store_snapshot(self) -> bytes:
        """The device prefix store's image (kvidx_text_store_snapshot): save it with the index's to warm-start both."""
        return self._device_store().text_store_snapshot()

    def text_store_restore(self, image) -> int:
        """Load a text_store_snapshot image into the device prefix store (created with text_cache_blocks /
        text_block_bytes if this indexer has not used it yet; it must hold no block).  -> blocks resident."""
        return self._device_store().text_store_restore(image)

    def get_pod_scores_batch(self, prompts: Sequence[str], model_name: str,
                             pod_identifiers: Sequence[str] = ()) -> List[Optional[Dict[str, float]]]:
        """GetPodScores for every prompt of a batch, on the device prefix store.  -> per prompt a dict pod -> score, or None
        for the reference's (nil, nil) (no full block).  The batch's finds all run before its adds, so a prompt is not served
        from the tokenization of another prompt of the same batch."""
        from ._native import pack_text
        ix = self._device_store()
        if not prompts:
            return []
        pods = list(pod_identifiers)
        text, text_off = pack_text(prompts)
        out, tokz = self.host.get_pod_scores_text(text, text_off, model_name, pods, self.tok.ratio)
        redo = np.flatnonzero(tokz)
        if len(redo):
            enc = [self.tok._encode(prompts[i]) for i in redo]
            with self.tok._mu:
                self.tok.encodes += len(redo)
            r_text, r_off = pack_text([prompts[i] for i in redo])
            tok_off = np.zeros(len(redo) + 1, np.int64)
            tok_off[1:] = np.cumsum([len(ids) for ids, _ in enc])
            tok = np.concatenate([np.asarray(ids, np.uint32) for ids, _ in enc]) if tok_off[-1] else np.zeros(0, np.uint32)
            span = np.concatenate([np.asarray(offs, np.uint64).reshape(-1, 2) for _, offs in enc]) if tok_off[-1] else np.zeros((0, 2), np.uint64)
            ix.text_store_add(r_text, r_off, tok, span, tok_off)
            for i, row in zip(redo, self.host.get_pod_scores_batch(tok, tok_off, model_name, pods)):
                out[i] = row
        return out


# ---- gRPC --------------------------------------------------------------------------------------------------------------
class IndexerService:
    def __init__(self, indexer: Indexer):
        self.indexer = indexer

    def GetPodScores(self, request, context):                      # server.go:70-96
        import grpc
        try:
            scores = self.indexer.get_pod_scores(request.prompt, request.model_name, list(request.pod_identifiers))
        except Exception as e:      # noqa: BLE001
            context.abort(grpc.StatusCode.UNKNOWN, "failed to get pod scores: %s" % e)
        resp = GetPodScoresResponse()
        for pod, sc in (scores or {}).items():
            p = resp.scores.add()
            p.pod, p.score = pod, sc
        return resp


def serve(indexer: Indexer, address: str = "127.0.0.1:0", max_workers: int = 64):
    """Start a gRPC server for `indexer`; returns (server, bound_port)."""
    import grpc
    svc = IndexerService(indexer)
    handler = grpc.method_handlers_generic_handler(SERVICE, {
        "GetPodScores": grpc.unary_unary_rpc_method_handler(svc.GetPodScores, request_deserializer=GetPodScoresRequest.FromString,
                                                            response_serializer=lambda m: m.SerializeToString())})
    server = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers))
    server.add_generic_rpc_handlers((handler,))
    port = server.add_insecure_port(address)
    server.start()
    return server, port


class IndexerClient:
    """What examples/kv_cache_index_service/client does: one unary call per prompt."""

    def __init__(self, address: str):
        import grpc
        self.channel = grpc.insecure_channel(address)
        self._call = self.channel.unary_unary(METHOD, request_serializer=lambda m: m.SerializeToString(),
                                              response_deserializer=GetPodScoresResponse.FromString)

    def get_pod_scores(self, prompt: str, model_name: str, pod_identifiers: Iterable[str] = (), timeout: float = 30.0) -> Dict[str, float]:
        req = GetPodScoresRequest(prompt=prompt, model_name=model_name, pod_identifiers=list(pod_identifiers))
        resp = self._call(req, timeout=timeout)
        return {p.pod: p.score for p in resp.scores}

    def close(self):
        self.channel.close()


# ---- KVEvents ingest ---------------------------------------------------------------------------------------------------
class ZmqSubscriber:
    """zmqSubscriber.runSubscriber (zmq_subscriber.go:81-162) + the pool's workers: messages go to the host mirror's per-pod
    queues (FNV-32a(pod) % concurrency, pool.go:132-144) as they arrive; the drain thread applies whatever has queued up as
    ONE device batch, so the batch size follows the arrival rate.  Sequence numbers are parsed and, like the reference,
    not acted upon (gaps are never replayed)."""

    def __init__(self, host_indexer, endpoint: str, topic_filter: str = "kv@", drain_interval_s: float = 0.002, bind: bool = True):
        import zmq
        self.host, self.endpoint, self.topic_filter = host_indexer, endpoint, topic_filter
        self.drain_interval_s = drain_interval_s
        self.ctx = zmq.Context.instance()
        self.sock = self.ctx.socket(zmq.SUB)
        if bind:
            self.sock.bind(endpoint)                                 # zmq_subscriber.go:90: the subscriber binds, publishers connect
        else:
            self.sock.connect(endpoint)
        self.sock.setsockopt_string(zmq.SUBSCRIBE, topic_filter)
        self.bound_endpoint = self.sock.getsockopt_string(zmq.LAST_ENDPOINT)
        self._stop = threading.Event()
        self._pending = threading.Event()
        self.messages = self.malformed = self.events_applied = self.events_dropped = self.batches = 0
        self.last_seq: Dict[str, int] = {}
        self._threads = [threading.Thread(target=self._recv_loop, daemon=True), threading.Thread(target=self._drain_loop, daemon=True)]

    def start(self):
        for t in self._threads:
            t.start()
        return self

    def _recv_loop(self):
        import zmq
        poller = zmq.Poller()
        poller.register(self.sock, zmq.POLLIN)
        while not self._stop.is_set():
            if not dict(poller.poll(250)):                           # :112
                continue
            while True:
                try:
                    parts = self.sock.recv_multipart(flags=zmq.NOBLOCK)
                except zmq.Again:
                    break
                if len(parts) != 3:                                  # :124 expected 3 parts
                    self.malformed += 1
                    continue
                topic, seq, payload = parts
                tp = topic.decode("utf-8", "replace").split("@")      # :136-144 kv@<pod>@<model>
                if len(tp) != 3 or len(seq) != 8:
                    self.malformed += 1
                    continue
                self.last_seq[tp[1]] = int.from_bytes(seq, "big")
                if self.host.add_task(tp[1], tp[2], payload) == 0:
                    self.messages += 1
                    self._pending.set()
                else:
                    self.malformed += 1

    def _drain_loop(self):
        while not self._stop.is_set():
            if not self._pending.wait(0.05):
                continue
            self._pending.clear()
            time.sleep(self.drain_interval_s)                        # let a burst accumulate into one device batch
            n, dropped = self.host.process()
            if n > 0:
                self.events_applied += n; self.events_dropped += dropped; self.batches += 1

    def flush(self, timeout: float = 5.0):
        """Wait until everything received so far has been applied (tests / shutdown)."""
        t0 = time.time()
        while time.time() - t0 < timeout:
            if not self._pending.is_set():
                n, dropped = self.host.process()
                if n > 0:
                    self.events_applied += n; self.events_dropped += dropped; self.batches += 1
                return True
            time.sleep(0.005)
        return False

    def stop(self):
        self._stop.set()
        for t in self._threads:
            t.join(timeout=2)
        self.sock.close(0)
