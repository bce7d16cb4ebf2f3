"""HierarchicalLogger with the reference's accumulate_means semantics (util/logger.py:71-342),
without the stable-baselines3 dependency: inside `accumulate_means(name)` every record goes to
`raw/<name>/<key>` and its running mean to `mean/<name>/<key>` on the root.  Output formats:
"stdout" (human table) and "csv"; default is silent (the hot path never waits on logging)."""
import collections
import contextlib
import csv
import os
import sys
import tempfile
from typing import Any, Dict, List, Optional, Sequence


class _Writer:
    def write(self, kv: Dict[str, Any], step: int) -> None:
        raise NotImplementedError

    def close(self) -> None:
        pass


class _Stdout(_Writer):
    def write(self, kv, step):
        if not kv:
            return
        w = max(len(k) for k in kv) + 2
        print("-" * (w + 16))
        for k in sorted(kv):
            v = kv[k]
            print(f"| {k:<{w}}| {v:<12.5g}|" if isinstance(v, float) else f"| {k:<{w}}| {str(v):<12}|")
        print("-" * (w + 16), file=sys.stdout, flush=True)


class _Csv(_Writer):
    def __init__(self, path):
        self.path, self.keys, self.rows = path, [], []

    def write(self, kv, step):
        self.rows.append(dict(kv))
        for k in kv:
            if k not in self.keys:
                self.keys.append(k)
        with open(self.path, "w", newline="") as f:
            w = csv.DictWriter(f, fieldnames=self.keys)
            w.writeheader()
            w.writerows(self.rows)


class HierarchicalLogger:
    def __init__(self, folder: Optional[str] = None, format_strs: Sequence[str] = ()):
        self.dir = folder or tempfile.mkdtemp(prefix="imb_log_")
        os.makedirs(self.dir, exist_ok=True)
        self._writers = []
        for f in format_strs:
            if f == "stdout":
                self._writers.append(_Stdout())
            elif f == "csv":
                self._writers.append(_Csv(os.path.join(self.dir, "progress.csv")))
            elif f in ("log", "json", "tensorboard", "wandb"):
                continue  # accepted for config compatibility, not implemented offline
            else:
                raise ValueError(f"unknown log format {f!r}")
        self.name_to_value: Dict[str, Any] = collections.defaultdict(float)
        self.name_to_count: Dict[str, int] = collections.defaultdict(int)
        self._prefix: Optional[str] = None
        self._key_prefixes: List[str] = []
        self.history = []

    def get_dir(self):
        return self.dir

    @contextlib.contextmanager
    def add_accumulate_prefix(self, prefix: str):
        if self._prefix is None:
            raise RuntimeError("No accumulate means context.")
        old = self._prefix
        self._prefix = f"{old}/{prefix}"
        try:
            yield
        finally:
            self._prefix = old

    @contextlib.contextmanager
    def add_key_prefix(self, prefix: str):
        """Inside `accumulate_means`: record(key) records `<prefix>/key` (nested prefixes are joined in order)."""
        if self._prefix is None:
            raise RuntimeError("Cannot add key prefix when accumulate_means context is not active.")
        self._key_prefixes.append(prefix)
        try:
            yield
        finally:
            self._key_prefixes.pop()

    @contextlib.contextmanager
    def accumulate_means(self, name: str):
        if self._prefix is not None:
            raise RuntimeError("Nested `accumulate_means` context")
        self._prefix = name
        try:
            yield
        finally:
            self._prefix = None

    def record(self, key: str, val: Any, exclude=None) -> None:
        if self._prefix is not None:
            key = "/".join(self._key_prefixes + [key])
            self.name_to_value[f"raw/{self._prefix}/{key}"] = val
            self.record_mean(f"mean/{self._prefix}/{key}", val, _direct=True)
        else:
            self.name_to_value[key] = val

    def record_mean(self, key: str, val: Any, exclude=None, _direct=False) -> None:
        if val is None:
            return
        if self._prefix is not None and not _direct:
            key = f"mean/{self._prefix}/{key}"
        c = self.name_to_count[key]
        self.name_to_value[key] = self.name_to_value[key] * c / (c + 1) + val / (c + 1)
        self.name_to_count[key] = c + 1

    def dump(self, step: int = 0) -> None:
        if self._prefix is not None:
            # inside accumulate_means only the raw records are flushed (util/logger.py:317-324)
            raw = {k: v for k, v in self.name_to_value.items() if k.startswith("raw/")}
            for w in self._writers:
                w.write(raw, step)
            self.history.append((step, raw))
            for k in raw:
                del self.name_to_value[k]
            return
        kv = dict(self.name_to_value)
        for w in self._writers:
            w.write(kv, step)
        self.history.append((step, kv))
        self.name_to_value.clear()
        self.name_to_count.clear()

    def log(self, *args, **kwargs):
        pass

    def warn(self, *args):
        print("WARNING:", *args, file=sys.stderr)

    def close(self):
        for w in self._writers:
            w.close()


def configure(folder: Optional[str] = None, format_strs: Optional[Sequence[str]] = None) -> HierarchicalLogger:
    return HierarchicalLogger(folder, format_strs if format_strs is not None else ())
