"""What the reference's own code computed, stored as golden data under tests/golden/reference/<name>.json.gz
(gzip-compressed JSON: the records are highly repetitive; `zcat` shows them).

Tests compare against the stored values unconditionally.  To regenerate them, run the tests with
RF_RECORD_REFERENCE=1 and the reference tree at RF_REFERENCE_ROOT (default /root/reference): every `value`
call then runs its `compute` callable (the reference code) and stores the result."""
import gzip
import json
import os

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
RECORD = os.environ.get("RF_RECORD_REFERENCE") == "1"
REFERENCE_ROOT = os.environ.get("RF_REFERENCE_ROOT", "/root/reference")


def _default(o):
    if hasattr(o, "tolist"):  # numpy / torch scalars and arrays
        return o.tolist()
    if isinstance(o, (set, frozenset)):
        return sorted(o)
    raise TypeError(f"not JSON-storable: {type(o).__name__}")


def norm(x):
    """x as it reads back from the store (tuples -> lists, dict keys -> str, numpy scalars -> Python)"""
    return json.loads(json.dumps(x, default=_default))


def ref_path(relpath):
    """path of a reference source file; only read while recording"""
    return os.path.join(REFERENCE_ROOT, relpath)


class Store:
    def __init__(self, name):
        self.path = os.path.join(GOLD, name + ".json.gz")
        self.data = {}
        if os.path.exists(self.path):
            with gzip.open(self.path, "rt", encoding="utf-8") as f:
                self.data = json.load(f)

    def value(self, key, compute):
        """the stored reference result `key`; with RF_RECORD_REFERENCE=1, compute() and store it first"""
        if RECORD:
            self.data[key] = norm(compute())
            os.makedirs(GOLD, exist_ok=True)
            text = json.dumps(self.data, indent=0, sort_keys=True)
            with open(self.path, "wb") as f:
                f.write(gzip.compress(text.encode("utf-8"), mtime=0))
        assert key in self.data, f"{key} missing from {self.path}: regenerate with RF_RECORD_REFERENCE=1"
        return self.data[key]
