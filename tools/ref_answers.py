"""The reference's answers in a differential fuzz run, kept so that the run can be repeated without the reference's tree.

`--record` (the reference's tree present): every answer is computed by the reference's own code, in call order, and the list is written
to tests/golden/fuzz_<tool>.json.gz together with the run's arguments.  Otherwise the same seeded run reads the answers back in the same
order.  Answers pass through JSON in both modes (tuples become lists), so both modes compare the same values; `canon` gives the product's
side the same form."""
import gzip
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def canon(v):
    return json.loads(json.dumps(v, default=str))


class Answers:
    def __init__(self, tool: str, args, record: bool):
        self.path = os.path.join(ROOT, "tests", "golden", f"fuzz_{tool}.json.gz")
        self.args = [str(a) for a in args]
        self.live = record
        self.i = 0
        if record:
            self.values = []
            return
        with gzip.open(self.path, "rt", encoding="utf-8") as f:
            stored = json.load(f)
        if stored["args"] != self.args:
            raise SystemExit(f"{self.path} holds the answers for arguments {stored['args']}, not {self.args}")
        self.values = stored["answers"]

    def __call__(self, fn):
        """fn() computes the answer with the reference (record mode only)."""
        if self.live:
            v = canon(fn())
            self.values.append(v)
            return v
        if self.i >= len(self.values):
            raise SystemExit(f"{self.path}: the run asks for more answers than were recorded (the generator changed: record again)")
        self.i += 1
        return self.values[self.i - 1]

    def finish(self) -> None:
        if self.live:
            with gzip.GzipFile(self.path, "wb", mtime=0) as f:
                f.write(json.dumps({"args": self.args, "answers": self.values}, ensure_ascii=True, separators=(",", ":")).encode())
            print(f"wrote {self.path}: {os.path.getsize(self.path)} bytes")
        elif self.i != len(self.values):
            raise SystemExit(f"{self.path}: {len(self.values) - self.i} recorded answers were not asked for (the generator changed: record again)")
