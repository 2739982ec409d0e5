"""Answers of the reference's own compiled code (oracle/_ref), recorded once and replayed from tests/golden/.

The reference tree is not part of this repository, so a test that compares with it cannot call it wherever the
suite runs.  Such a test asks an `Answers` table instead: with `live` given (where oracle/_ref is built) every call
runs the reference and is recorded, and `save()` writes tests/golden/<name>.json; without it the call is answered
from that file.  Calls are keyed by the SHA-256 of their arguments, so the file holds results only."""
import base64
import hashlib
import json
import os

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _enc(v):
    if isinstance(v, (bytes, bytearray)):
        return {"b64": base64.b64encode(bytes(v)).decode()}
    if isinstance(v, (list, tuple)):
        return [_enc(x) for x in v]
    if isinstance(v, dict):
        return {k: _enc(x) for k, x in v.items()}
    return v


def _dec(v):
    if isinstance(v, dict):
        return base64.b64decode(v["b64"]) if list(v) == ["b64"] else {k: _dec(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_dec(x) for x in v]
    return v


class Answers:
    def __init__(self, name, live=None):
        self.path = os.path.join(GOLDEN, name + ".json")
        self.live = live
        self.table = {} if live is not None else None

    def __call__(self, *args):
        key = hashlib.sha256(json.dumps(_enc(list(args))).encode()).hexdigest()
        if self.live is not None:
            self.table[key] = _enc(self.live(*args))
        elif self.table is None:
            with open(self.path) as f:
                self.table = json.load(f)
        assert key in self.table, f"{os.path.basename(self.path)} holds no answer for this call: re-record it"
        return _dec(self.table[key])

    def save(self):
        with open(self.path, "w") as f:
            json.dump(self.table, f, sort_keys=True, separators=(",", ":"))
