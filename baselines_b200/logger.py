"""Key/value logger with the call surface and the on-disk formats of the reference's baselines/logger.py.

API used by the learners: logkv (:196), logkv_mean (:204), logkvs (:210), dumpkvs (:217), getkvs (:223), log / info
(:227-246), get_dir (:262), configure (:372-398).  Output formats (make_output_format :174-190), selected by
`format_strs` or $OPENAI_LOG_FORMAT (default "stdout,log,csv"; ranks > 0: $OPENAI_LOG_FORMAT_MPI, default "log", files
suffixed "-rank%03i"):

  stdout / log : the boxed key-value table (HumanOutputFormat :27-83; numbers as %-8.3g, cells cut at 30 characters,
                 keys sorted case-insensitively) on stdout or in <dir>/log.txt
  json         : one JSON object per dump in <dir>/progress.json (:85-98)
  csv          : <dir>/progress.csv whose header grows when new keys appear, earlier rows padded (:100-136)
  tensorboard  : needs TensorFlow event writers (:138-172) -- not available here, raises NotImplementedError

A directory comes from `dir`, else $OPENAI_LOGDIR; without either only stdout is written (the reference would invent a
temp directory, :377-381 -- the learners here must not litter /tmp when called from tests).
"""
import json
import os
import sys
from collections import OrderedDict, defaultdict

_kvs = OrderedDict()
_counts = defaultdict(int)
_dir = None
_writers = []
_quiet = False


def _rank():
    for var in ("RANK", "PMI_RANK", "OMPI_COMM_WORLD_RANK"):      # torchrun, then the reference's MPI variables (:363-369)
        if var in os.environ:
            return int(os.environ[var])
    return 0


class _Human:
    def __init__(self, target):
        self.own = isinstance(target, str)
        self._stdout = target is sys.stdout          # follow later redirections of sys.stdout (test capture, tee)
        self._f = open(target, "wt") if self.own else target

    @property
    def f(self):
        return sys.stdout if self._stdout else self._f

    @staticmethod
    def _cut(s):
        return s[:27] + "..." if len(s) > 30 else s

    def writekvs(self, kvs):
        cells = {}
        for k, v in sorted(kvs.items()):
            cells[self._cut(k)] = self._cut("%-8.3g" % v if hasattr(v, "__float__") else str(v))
        if not cells:
            return
        kw, vw = max(map(len, cells)), max(map(len, cells.values()))
        bar = "-" * (kw + vw + 7)
        rows = [bar] + ["| %s | %s |" % (k.ljust(kw), v.ljust(vw)) for k, v in sorted(cells.items(), key=lambda kv: kv[0].lower())] + [bar]
        self.f.write("\n".join(rows) + "\n")
        self.f.flush()

    def writeseq(self, parts):
        self.f.write(" ".join(parts) + "\n")
        self.f.flush()

    def close(self):
        if self.own:
            self._f.close()


class _Json:
    def __init__(self, path):
        self.f = open(path, "wt")

    def writekvs(self, kvs):
        self.f.write(json.dumps({k: (float(v) if hasattr(v, "dtype") else v) for k, v in sorted(kvs.items())}) + "\n")
        self.f.flush()

    def close(self):
        self.f.close()


class _Csv:
    def __init__(self, path):
        self.path, self.keys, self.rows = path, [], []
        open(path, "wt").close()

    def writekvs(self, kvs):
        new = sorted(k for k in kvs if k not in self.keys)
        self.rows.append(dict(kvs))
        if new:                                                   # header grows; earlier rows get empty cells
            self.keys.extend(new)
            with open(self.path, "wt") as f:
                f.write(",".join(self.keys) + "\n")
                for r in self.rows:
                    f.write(",".join("" if r.get(k) is None else str(r[k]) for k in self.keys) + "\n")
        else:
            with open(self.path, "at") as f:
                f.write(",".join("" if kvs.get(k) is None else str(kvs[k]) for k in self.keys) + "\n")

    def close(self):
        pass


def _make_writer(fmt, d, suffix):
    if fmt == "stdout":
        return _Human(sys.stdout)
    if d is None:
        raise ValueError("log format %r needs a directory (dir= or $OPENAI_LOGDIR)" % fmt)
    if fmt == "log":
        return _Human(os.path.join(d, "log%s.txt" % suffix))
    if fmt == "json":
        return _Json(os.path.join(d, "progress%s.json" % suffix))
    if fmt == "csv":
        return _Csv(os.path.join(d, "progress%s.csv" % suffix))
    if fmt == "tensorboard":
        raise NotImplementedError("the tensorboard writer (logger.py:138-172) builds TensorFlow event files; "
                                  "TensorFlow is not available in this build")
    raise ValueError("Unknown format specified: %s" % (fmt,))


def configure(dir=None, format_strs=None, comm=None, log_suffix="", quiet=False):
    global _dir, _writers, _quiet
    for w in _writers:
        w.close()
    _kvs.clear()
    _counts.clear()
    _quiet = quiet
    _dir = dir or os.environ.get("OPENAI_LOGDIR")
    if _dir:
        _dir = os.path.expanduser(_dir)
        os.makedirs(_dir, exist_ok=True)
    rank = _rank()
    if rank > 0:
        log_suffix = log_suffix + "-rank%03i" % rank
    if format_strs is None:
        if rank == 0:
            format_strs = os.environ.get("OPENAI_LOG_FORMAT", "stdout,log,csv").split(",")
        else:
            format_strs = os.environ.get("OPENAI_LOG_FORMAT_MPI", "log").split(",")
        if not _dir:
            format_strs = [f for f in format_strs if f == "stdout"]
    _writers = [_make_writer(f, _dir, log_suffix) for f in format_strs if f and not (quiet and f == "stdout")]
    if _dir and _writers:
        log("Logging to %s" % _dir)


def get_dir():
    return _dir


def logkv(key, val):
    _kvs[key] = val


def logkv_mean(key, val):
    old, cnt = _kvs.get(key, 0.0), _counts[key]
    _kvs[key] = old * cnt / (cnt + 1) + val / (cnt + 1)
    _counts[key] = cnt + 1


def logkvs(d):
    for k, v in d.items():
        logkv(k, v)


def getkvs():
    return _kvs


def info(*args):
    if _quiet:
        return
    if not _writers and _dir is None:                              # never configured: behave like a plain stdout logger
        print(*args, file=sys.stdout, flush=True)
        return
    for w in _writers:
        if isinstance(w, _Human):
            w.writeseq([str(a) for a in args])


log = info


def warn(*args):
    info(*args)


def dumpkvs():
    d = OrderedDict(_kvs)
    if d:
        if not _writers and _dir is None and not _quiet:
            _Human(sys.stdout).writekvs(d)
        for w in _writers:
            w.writekvs(d)
    _kvs.clear()
    _counts.clear()
    return d


# the names her.py and its config use (logger.py:461-463 of the reference)
record_tabular = logkv
dump_tabular = dumpkvs
