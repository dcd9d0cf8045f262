"""BackupServer -- mirror of lib/backupServer.js: the backupQueue REST surface.

POST /backup/   {host, port, dataset}  -> {jobid, jobPath: '/backup/<uuid>'}
                any of the three missing -> 409 MissingParameter
                (restify.MissingParameterError, lib/backupServer.js:135-138)
GET  /backup/:uuid -> the live job object (the sender mutates the same object)
                unknown uuid -> 404 ResourceNotFound (:111)
                job.err set  -> 500 InternalError    (:119)
"""
import json
import threading
import uuid as uuidlib
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from urllib.parse import parse_qs, urlparse

from .backup_queue import BackupQueue


def _job_json(job):
    out = {}
    for k, v in job.items():
        if k.startswith("_"):
            continue
        out[k] = str(v) if isinstance(v, BaseException) else v
    return out


class BackupServer(object):
    def __init__(self, options):
        assert isinstance(options, dict), "options (object) is required"
        assert isinstance(options.get("port"), int), "options.port (number) is required"
        self._port = options["port"]
        self._host = options.get("host", "0.0.0.0")
        self._queue = BackupQueue({"log": options.get("log")})
        self._server = None
        self._thread = None
        self._init()

    @staticmethod
    def start(cfg):
        return BackupServer(cfg)

    def getQueue(self):
        return self._queue

    @property
    def port(self):
        return self._server.server_address[1]

    def close(self):
        if self._server is not None:
            self._server.shutdown()
            self._server.server_close()
            self._server = None

    def _init(self):
        queue = self._queue

        class Handler(BaseHTTPRequestHandler):
            protocol_version = "HTTP/1.1"

            def log_message(self, *a):
                pass

            def _send(self, code, obj):
                body = json.dumps(obj).encode()
                self.send_response(code)
                self.send_header("Content-Type", "application/json")
                self.send_header("Content-Length", str(len(body)))
                self.end_headers()
                self.wfile.write(body)

            def do_GET(self):  # checkBackup, lib/backupServer.js:108-130
                parts = urlparse(self.path).path.strip("/").split("/")
                if len(parts) != 2 or parts[0] != "backup":
                    return self._send(404, {"code": "ResourceNotFound", "message": self.path})

                def cb(job):
                    if not job:
                        return self._send(404, {"code": "ResourceNotFound", "message": ""})
                    if job.get("err"):
                        return self._send(500, {"code": "InternalError", "message": str(job["err"])})
                    return self._send(200, _job_json(job))
                return queue.get(parts[1], cb)

            def do_POST(self):  # postBackup, lib/backupServer.js:133-155
                if urlparse(self.path).path.rstrip("/") != "/backup":
                    return self._send(404, {"code": "ResourceNotFound", "message": self.path})
                n = int(self.headers.get("Content-Length") or 0)
                raw = self.rfile.read(n) if n else b""
                params = {k: v[0] for k, v in parse_qs(urlparse(self.path).query).items()}
                try:
                    if raw:
                        if "json" in (self.headers.get("Content-Type") or "json"):
                            params.update(json.loads(raw.decode()))
                        else:
                            params.update({k: v[0] for k, v in parse_qs(raw.decode()).items()})
                except ValueError:
                    return self._send(400, {"code": "InvalidContent", "message": "Invalid JSON"})
                if not params.get("host") or not params.get("dataset") or not params.get("port"):
                    return self._send(409, {"code": "MissingParameter",
                                            "message": "host, dataset, and port parameters required"})
                job = {"uuid": str(uuidlib.uuid4()), "host": params["host"], "port": params["port"],
                       "dataset": params["dataset"], "done": False}
                if params.get("accept"):
                    job["accept"] = params["accept"]      # wire capability of the receiver (f2)
                if params.get("acceptGzip") in (True, "true"):
                    job["acceptGzip"] = True              # ... and gzip frames on that wire
                self._send(200, {"jobid": job["uuid"], "jobPath": "/backup/" + job["uuid"]})
                queue.push(job)

        self._server = ThreadingHTTPServer((self._host, self._port), Handler)
        self._server.daemon_threads = True
        self._thread = threading.Thread(target=self._server.serve_forever, daemon=True)
        self._thread.start()
