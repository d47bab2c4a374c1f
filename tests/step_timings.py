"""The packing rules of a Story generation's step timings (bf_topology_timings), the twin of go/frontier/packer.go's stepTiming:
what the reference's parseSleepConfig / parseGateConfig / parseWaitConfig (internal/controller/runs/dag.go:1549-1653) make of a
step's `with`, as (code, delay in clock units) or None.  Durations follow Go's time.ParseDuration and are rounded up to whole
clock units, so that no armed timer fires before the reference's deadline."""
import json

from bobrapet_b200 import _abi as A

_UNITS = {"ns": 1, "us": 1_000, "µs": 1_000, "μs": 1_000, "ms": 1_000_000, "s": 1_000_000_000,
          "m": 60_000_000_000, "h": 3_600_000_000_000}
_MAX = (1 << 63) - 1


class DurationError(ValueError):
    pass


def parse_duration(s):
    """Go's time.ParseDuration -> nanoseconds (int), or DurationError"""
    orig, d, neg = s, 0, False
    if s and s[0] in "+-":
        neg, s = s[0] == "-", s[1:]
    if s == "0":
        return 0
    if s == "":
        raise DurationError("invalid duration %r" % orig)
    while s:
        i = 0
        while i < len(s) and s[i].isdigit() and s[i].isascii():
            i += 1
        pre = i > 0
        v = 0
        for ch in s[:i]:
            v = v * 10 + int(ch)
            if v > 1 << 63:
                raise DurationError("invalid duration %r" % orig)
        s = s[i:]
        f, scale, post = 0, 1.0, False
        if s.startswith("."):
            s = s[1:]
            i, overflow = 0, False
            while i < len(s) and s[i].isdigit() and s[i].isascii():
                if not overflow:
                    if f > (_MAX - int(s[i])) // 10:
                        overflow = True
                    else:
                        f, scale = f * 10 + int(s[i]), scale * 10
                i += 1
            post = i > 0
            s = s[i:]
        if not pre and not post:
            raise DurationError("invalid duration %r" % orig)
        i = 0
        while i < len(s) and s[i] != "." and not (s[i].isdigit() and s[i].isascii()):
            i += 1
        u, s = s[:i], s[i:]
        if u not in _UNITS:
            raise DurationError("unknown unit %r in duration %r" % (u, orig))
        unit = _UNITS[u]
        if v > (1 << 63) // unit:
            raise DurationError("invalid duration %r" % orig)
        v *= unit
        if f > 0:
            v += int(float(f) * (float(unit) / scale))
            if v > 1 << 63:
                raise DurationError("invalid duration %r" % orig)
        d += v
        if d > 1 << 63:
            raise DurationError("invalid duration %r" % orig)
    if neg:
        return -d
    if d > _MAX:
        raise DurationError("invalid duration %r" % orig)
    return d


def _positive(raw):
    d = parse_duration(raw)   # parsePositiveDuration, steprun_controller.go:1364
    if d <= 0:
        raise DurationError("duration must be positive")
    return d


def _fields(with_raw, names):
    """encoding/json into a struct of string fields: keys match case-insensitively (the last one wins), null leaves a field
    blank, any other non-string value or a non-object document is an error"""
    doc = json.loads(with_raw)
    out = dict.fromkeys(names, "")
    if doc is None:
        return out
    if not isinstance(doc, dict):
        raise ValueError("with is not an object")
    for k, v in doc.items():
        for n in names:
            if k.lower() == n.lower():
                if v is None:
                    continue
                if not isinstance(v, str):
                    raise ValueError("with.%s is not a string" % n)
                out[n] = v
    return out


def _units(ns, unit_ns):
    return min(-(-ns // unit_ns), 0xFFFFFFFF)


def _on_timeout(raw):
    if raw.strip() and raw.strip().lower() not in ("fail", "skip"):
        raise ValueError("unsupported onTimeout %r" % raw)


def step_timing(step_type, with_raw, unit_ns=1_000_000_000):
    """the timing of one step: step_type A.STEP_*, with_raw the step's `with` as JSON text or None (absent) -> (code, delay) or
    None (no timer: the step's decision arrives as a delta, or the step is not a sleep, gate or wait)"""
    if step_type == A.STEP_SLEEP:
        if not with_raw:
            return A.DEC_SUCCEED, 0
        try:
            dur = _fields(with_raw, ("duration",))["duration"]
            if dur.strip() == "":
                return A.DEC_SUCCEED, 0
            return A.DEC_SUCCEED, _units(_positive(dur), unit_ns)
        except ValueError:
            return A.DEC_FAIL, 0
    if step_type == A.STEP_GATE:
        if with_raw is None:
            return None
        try:
            f = _fields(with_raw, ("timeout", "pollInterval", "onTimeout"))
            timeout = _positive(f["timeout"]) if f["timeout"] != "" else None
            if f["pollInterval"] != "":
                _positive(f["pollInterval"])
            _on_timeout(f["onTimeout"])
        except ValueError:
            return A.DEC_FAIL, 0
        return None if timeout is None else (A.DEC_TIMED_OUT, _units(timeout, unit_ns))
    if step_type == A.STEP_WAIT:
        if with_raw is None:
            return A.DEC_FAIL, 0
        try:
            f = _fields(with_raw, ("until", "timeout", "pollInterval", "onTimeout"))
            if f["until"].strip() == "":
                return A.DEC_FAIL, 0
            timeout = _positive(f["timeout"]) if f["timeout"] != "" else None
            poll = _positive(f["pollInterval"]) if f["pollInterval"] != "" else None
            _on_timeout(f["onTimeout"])
        except ValueError:
            return A.DEC_FAIL, 0
        if timeout is not None:
            return A.DEC_TIMED_OUT, _units(timeout, unit_ns)
        return None if poll is None else (A.DEC_PENDING, _units(poll, unit_ns))
    return None
