"""`python -m arks_b200`: the process the reference builds from cmd/gateway/main.go -- ext_proc gRPC + health on
--server.grpc-port (50052), /v1/models on --server.http-port (8080), /metrics on --metrics.port (9110), the config provider
started before the listeners, SIGINT / SIGTERM -> graceful shutdown (main.go:171-231; flag names kept, main.go:96-116).

What differs, because this image has neither a cluster nor Redis: the rate-limit and quota stores ARE the library (counters in
HBM: no --ratelimiter.* / --quota.* / --redis.* flags), and the provider takes its objects from the outside instead of
client-go: `--provider.objects FILE` is a (re)list (YAML or JSON documents of kind ArksToken / ArksQuota / ArksEndpoint, e.g.
examples/quickstart/quickstart.yaml; re-read when the file changes) and `--provider.events FILE|-` a stream of Kubernetes
watch events, one JSON object per line (what `kubectl get arkstokens,arksquotas,arksendpoints -A --watch
--output-watch-events -o json` prints). ArksQuota status updates are written, one JSON object per line, to
--provider.status-out (default stdout) for whoever holds the API credentials.

No CUDA device -> the process exits with the library's error: there is no CPU path."""
from __future__ import annotations

import argparse
import json
import os
import signal
import sys
import threading

from . import extproc, metrics
from .provider import KINDS, ArksProvider, ProviderLoop


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m arks_b200", description=__doc__.split("\n\n")[0])
    p.add_argument("--server.grpc-port", dest="grpc_port", type=int, default=50052, help="gRPC server port")
    p.add_argument("--server.http-port", dest="http_port", type=int, default=8080, help="http server port")
    p.add_argument("--server.bind", dest="bind", default="0.0.0.0", help="address the three listeners bind (the reference: all)")
    p.add_argument("--metrics.port", dest="metrics_port", type=int, default=9110, help="Prometheus metrics port")
    p.add_argument("--provider.objects", dest="objects", default=None, help="YAML / JSON documents of the three kinds (a list)")
    p.add_argument("--provider.events", dest="events", default=None, help="watch events, JSON lines; '-' = stdin")
    p.add_argument("--provider.status-out", dest="status_out", default="-", help="ArksQuota status updates, JSON lines; '-' = stdout")
    p.add_argument("--provider.restore-on-start", dest="restore", type=int, default=1,
                   help="first status pass raises the counters to the CRs (0: the reference's behaviour, which zeroes them)")
    p.add_argument("--device", type=int, default=0, help="CUDA device of this process (one process per GPU)")
    p.add_argument("--max-batch", dest="max_batch", type=int, default=8192, help="rows per micro-batch")
    p.add_argument("--max-batch-bytes", dest="max_bytes", type=int, default=64 << 20)
    p.add_argument("--batcher", choices=("compiled", "python"), default="compiled", help="the C++ micro-batcher or its Python twin")
    p.add_argument("--grpc-workers", dest="workers", type=int, default=256, help="concurrent ext_proc streams served")
    p.add_argument("--bpe.tokenizer", dest="bpe_tokenizer", default=None,
                   help="tokenizer.json every model's text is BPE-counted with unless bound to another (off by default)")
    p.add_argument("--bpe.model-tokenizer", dest="bpe_model_tokenizer", action="append", default=[], metavar="MODEL=PATH",
                   help="count MODEL (an ArksEndpoint name) with the tokenizer.json at PATH; repeatable, the same PATH shares one "
                        "vocabulary; needs --bpe.tokenizer")
    p.add_argument("--bpe.precharge", dest="bpe_precharge", action="store_true",
                   help="charge admitted requests' BPE counts to tpm / tpd at request time (needs --bpe.tokenizer)")
    p.add_argument("--bpe.stream-metering", dest="bpe_stream_metering", action="store_true",
                   help="decide and bill streams without stream_options.include_usage by their BPE counts (needs --bpe.tokenizer)")
    p.add_argument("--gateway.ratelimit-headers", dest="ratelimit_headers", action="store_true",
                   help="send x-ratelimit-{limit,remaining,reset}-{requests,tokens} on every decided request and retry-after on "
                        "rate-limit 429s (off by default: the reference sends none)")
    p.add_argument("--ratelimiter.sliding-window", dest="sliding_window", action="store_true",
                   help="admit against the current window plus the previous window's remaining share, so that no burst across "
                        "a window boundary exceeds a limit (off by default: the reference's fixed window)")
    return p.parse_args(argv)


def configure_ratelimit_headers(engine, batcher, args):
    """--gateway.ratelimit-headers as library calls, made before the first generation is published: the rate-limit report of
    the context (arks_set_ratelimit_report), through the compiled batcher when there is one (its stream state machine shapes
    the headers). Without the flag: no call at all."""
    if not args.ratelimit_headers:
        return
    if batcher is not None:
        batcher.b.set_ratelimit_report(True)
    engine.set_ratelimit_report(True)


def configure_sliding_window(engine, batcher, args):
    """--ratelimiter.sliding-window as library calls (arks_set_sliding_window), through the compiled batcher when there is one
    (its stream state machine shapes the reset / retry headers). Without the flag: no call at all."""
    if not args.sliding_window:
        return
    if batcher is not None:
        batcher.b.set_sliding_window(True)
    engine.set_sliding_window(True)


def configure_bpe(engine, args, load=None):
    """The --bpe.* flags as library calls, made before the first generation is published so that its tables already carry
    the bindings: the default vocabulary into slot 0, every other tokenizer file into a slot of its own (models naming the
    same file share it), one binding per model, then the pre-charge and stream metering switches. Without the flags: no
    call at all. ValueError on flags that cannot work together."""
    from . import bpe
    load = load or bpe.load_tokenizer
    a = args
    pairs = []
    for spec in a.bpe_model_tokenizer:
        model, eq, path = spec.partition("=")
        if not eq or not model or not path:
            raise ValueError(f"--bpe.model-tokenizer {spec!r}: expected MODEL=PATH")
        pairs.append((model, path))
    if not a.bpe_tokenizer:
        if pairs or a.bpe_precharge or a.bpe_stream_metering:
            raise ValueError("--bpe.model-tokenizer, --bpe.precharge and --bpe.stream-metering need --bpe.tokenizer")
        return
    # one slot per FILE: two spellings of the same path (relative / absolute, a symlink) share it
    key = os.path.realpath
    slot_of, first_path = {key(a.bpe_tokenizer): 0}, [a.bpe_tokenizer]
    for _, path in pairs:
        if key(path) not in slot_of:
            slot_of[key(path)] = len(first_path)
            first_path.append(path)
    if len(first_path) > bpe.MAX_VOCABS:
        raise ValueError(f"{len(first_path)} tokenizer files: at most {bpe.MAX_VOCABS} vocabularies")
    for slot, path in enumerate(first_path):
        t = load(path)
        if slot == 0 and not t.flags & bpe.BPE_IGNORE_MERGES:
            engine.load_bpe(t)
        else:
            engine.load_bpe_vocab(slot, t)
    for model, path in pairs:
        if slot_of[key(path)]:
            engine.bind_model_vocab(model, slot_of[key(path)])
    if a.bpe_precharge:
        engine.set_precharge(True)
    if a.bpe_stream_metering:
        engine.set_stream_metering(True)


def read_objects(path):
    """every ArksToken / ArksQuota / ArksEndpoint in a YAML (multi-document) or JSON file; `kind: List` items are unfolded"""
    text = open(path).read()
    if path.endswith(".json"):
        docs = json.loads(text)
        docs = docs if isinstance(docs, list) else [docs]
    else:
        import yaml
        docs = [d for d in yaml.safe_load_all(text) if d]
    out = []
    for d in docs:
        for o in (d.get("items") or []) if str(d.get("kind", "")).endswith("List") else [d]:
            if o.get("kind") in KINDS:
                out.append(o)
    return out


class Assembly:
    """everything main() starts, around an engine (arks_b200.gateway.Gateway); ports 0 = pick free ones (tests)"""

    def __init__(self, engine, args, batcher=None, status_out=None):
        self.engine, self.args = engine, args
        self.srv = extproc.ExtProcServer(engine, None, _bearer(), batcher=batcher)
        self.provider = ArksProvider(engine, publish=self.srv.publisher(engine))
        self._status_out = status_out
        self.loop = ProviderLoop(self.provider, write_status=self._write_status, restore_on_start=bool(args.restore))
        self.threads, self.grpc = [], None
        self._objects_mtime = None

    # ---- provider inputs
    def relist(self):
        """--provider.objects: the file is the list; returns how many objects changed anything"""
        objs = read_objects(self.args.objects)
        n = sum(self.provider.replace(kind, [o for o in objs if o["kind"] == kind]) for kind in KINDS)
        self._objects_mtime = os.path.getmtime(self.args.objects)
        return n

    def _watch_objects(self):
        while not self.loop.stop.wait(1.0):
            try:
                if os.path.getmtime(self.args.objects) != self._objects_mtime and self.relist():
                    self.provider.flush()
            except Exception as e:  # noqa: BLE001  a half-written or malformed file: keep the configuration, try again
                print(f"provider.objects: {e!r}", file=sys.stderr)

    def _read_events(self, f):
        for line in f:
            line = line.strip()
            if not line:
                continue
            try:
                self.loop.offer(json.loads(line))
            except ValueError as e:
                print(f"provider.events: {e!r}", file=sys.stderr)

    def _write_status(self, updates):
        f = self._status_out or sys.stdout
        for u in updates:
            f.write(json.dumps({"apiVersion": "arks.ai/v1", "kind": "ArksQuota", "metadata": {"namespace": u["namespace"], "name": u["name"]},
                                "status": u["status"]}, separators=(",", ":")) + "\n")
        f.flush()

    # ---- /metrics: device rows (per tenant, counted by the kernels) + the host's wall-clock series
    def render_metrics(self):
        snap = getattr(self.engine, "snapshot_metrics", None)
        text = ""
        if snap is not None and self.engine.tables is not None:
            between = getattr(self.srv.batcher, "between_batches", None)
            grab = lambda: (self.engine.tables, snap())  # noqa: E731  (rows and names of the same generation)
            with self.provider.no_publish():  # the snapshot must not meet a table swap
                tables, rows = between(grab) if between else grab()
            if len(rows) == tables.n_qos:
                text = metrics.exposition(tables, rows)
        return text + self.srv.metrics.exposition()

    # ---- main.go:196-214
    def start(self):
        a = self.args
        if a.objects:
            self.relist()
            self.provider.flush()  # "wait cache sync" (arks_impl.go:167-170): the first generation precedes the listeners
            if a.restore and self.engine.tables is not None:
                # the restore pass belongs BEFORE the first request, not one ticker period after it: a gateway that restarts
                # must not hand every tenant a fresh quota for ten seconds (the reference's first pass comes with the ticker,
                # arks_impl.go:217-225, and zeroes instead of restoring)
                updates = self.provider.sync_quota_status(restore=True)
                self.loop.restore_next = False
                if updates:
                    self._write_status(updates)
            self.threads.append(threading.Thread(target=self._watch_objects, daemon=True))
        self.threads.append(threading.Thread(target=self.loop.run, daemon=True))
        if a.events:
            f = sys.stdin if a.events == "-" else open(a.events)
            self.threads.append(threading.Thread(target=self._read_events, args=(f,), daemon=True))
        for t in self.threads:
            t.start()
        self.grpc, self.grpc_port = extproc.serve(self.srv, port=a.grpc_port, max_workers=a.workers, host=a.bind)
        self.http, self.http_port = extproc.serve_http(lambda: self.srv.tables, port=a.http_port, host=a.bind)
        self.metrics_srv, self.metrics_port = extproc.serve_metrics(self.render_metrics, port=a.metrics_port, host=a.bind)
        return self

    def shutdown(self):
        """Server.GracefullyShutdown, then the provider's context is cancelled (main.go:222-229)"""
        errors = extproc.gracefully_shutdown(self.grpc, self.http, self.metrics_srv)
        self.loop.stop.set()
        self.srv.batcher.close()
        return errors


def _bearer():
    from .gateway import extract_bearer
    return extract_bearer


def main(argv=None) -> int:
    args = parse_args(argv)
    from . import cpphost
    from .gateway import Gateway
    g = Gateway(args.device, args.max_batch, args.max_bytes)  # raises without a CUDA device
    g.enable_metrics(True)
    configure_bpe(g, args)  # before Assembly.start() publishes the first generation
    batcher = None
    if args.batcher == "compiled":
        batcher = extproc.CompiledBatcher(cpphost.Batcher(cpphost.load(cpphost.build()), g._h, max_batch=args.max_batch,
                                                          max_bytes=args.max_bytes))
    configure_ratelimit_headers(g, batcher, args)  # before Assembly.start() publishes the first generation
    configure_sliding_window(g, batcher, args)
    status_out = None if args.status_out == "-" else open(args.status_out, "a")
    asm = Assembly(g, args, batcher=batcher, status_out=status_out).start()
    print(f"arks_b200 gateway: gRPC :{asm.grpc_port}, http :{asm.http_port}, metrics :{asm.metrics_port}, device {args.device}, "
          f"generation {g.generation}", file=sys.stderr)
    stop = threading.Event()
    for s in (signal.SIGINT, signal.SIGTERM):
        signal.signal(s, lambda *_: stop.set())
    stop.wait()
    print("Received shutdown signal, initiating graceful shutdown...", file=sys.stderr)
    errors = asm.shutdown()
    for e in errors:
        print(e, file=sys.stderr)
    return 1 if errors else 0


if __name__ == "__main__":
    sys.exit(main())
