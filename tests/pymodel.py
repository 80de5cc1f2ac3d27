"""Independent pure-Python model of the reference's grouped streaming window (small inputs only).

Written separately from oracle/dnz_oracle.c (dict-of-dicts, row at a time) so the two can check each other.
Follows grouped_window_agg_stream.rs:326-349 (per-batch order), streaming_window.rs:1053-1094 (windows),
utils/time.rs:31-57 (watermark) and the DataFusion-42 accumulator rules listed in SURVEY.md §8a.
"""
import struct

F64_MAX = 1.7976931348623157e308


def total_key(d: float) -> int:
    b = struct.unpack("<q", struct.pack("<d", d))[0]
    return b ^ (((b >> 63) & 0xFFFFFFFFFFFFFFFF) >> 1)


def windows_for(mn, mx, L, S):
    Ls = L // 1000

    def snap(t):
        return (t // 1000 // Ls) * Ls * 1000
    out = []
    if S:
        cur = snap(mn - L)
        while cur <= mx:
            end = cur + L
            if not (mn > end or mx < cur):
                out.append((cur, end))
            cur += S
    else:
        cur = snap(mn)
        while cur <= mx:
            out.append((cur, cur + L))
            cur += L
    return out


class PyModel:
    def __init__(self, L, S=0, filt=None):
        self.L, self.S, self.filt = L, S, filt
        self.frames = {}      # start -> {"end":, "groups": {key: state}, order: [keys]}
        self.wm = None
        self.seq = 0
        self.out = []

    def push(self, rows):
        """rows: list of (ts|None, val|None, key(bytes)|None)"""
        seq = self.seq
        self.seq += 1
        if not rows:
            return
        tss = [r[0] for r in rows if r[0] is not None]
        mn, mx = min(tss), max(tss)
        for (s, e) in windows_for(mn, mx, self.L, self.S):
            fr = self.frames.setdefault(s, {"end": e, "groups": {}})
            for ts, val, key in rows:
                if ts is None or not (s <= ts < e):
                    continue
                st = fr["groups"].setdefault(key, {"cnt": 0, "mn": F64_MAX, "mx": -F64_MAX, "sum": 0.0, "seen": False})
                if val is not None:
                    st["cnt"] += 1
                    st["seen"] = True
                    if st["mn"] > val:
                        st["mn"] = val
                    if st["mx"] < val:
                        st["mx"] = val
                    st["sum"] += val
        if self.wm is None or self.wm <= mn:
            self.wm = mn
        for s in sorted(self.frames):
            fr = self.frames[s]
            if self.wm >= fr["end"]:
                for key, st in fr["groups"].items():
                    if st["seen"]:     # sum(reading) is the avg state's sum: +0.0, then += v in row order
                        row = (s, fr["end"], key, st["cnt"], st["mn"], st["mx"], st["sum"] / st["cnt"], seq, st["sum"])
                    else:
                        row = (s, fr["end"], key, st["cnt"], None, None, None, seq, None)
                    if self._pass(row):
                        self.out.append(row)
                del self.frames[s]

    def _pass(self, row):
        if not self.filt:
            return True
        col, op, lit = self.filt
        v = {"count": row[3], "min": row[4], "max": row[5], "average": row[6], "avg": row[6], "sum": row[8]}[col]
        if v is None:
            return False
        a, b = total_key(float(v)), total_key(float(lit))
        return {">": a > b, ">=": a >= b, "<": a < b, "<=": a <= b, "==": a == b, "!=": a != b}[op]


class PyUngroupedModel:
    """Independent model of `.window([], aggs, ..)`: one partition of StreamingWindowExec(Partial) -> StreamingWindowExec(Final).

    Written from the reference, not from oracle/dnz_oracle.c:
      Partial  WindowAggStream::poll_next_inner      streaming_window.rs:791-828  (windows of the batch, push, watermark, trigger)
               PartialWindowAggFrame::push            rows with start <= ts < end, row accumulators updated
               trigger_windows                        :703-733  ONE concatenated batch, a row per frame with watermark >= end, ascending
      Final    FullWindowAggStream::poll_next_inner   :954-1032 frame chosen by the MAX window start in the incoming batch, EVERY row of
                                                      the batch merged into it, seen_windows late drop, watermark = max window START
               finalize_windows                       :926-951  frames with watermark > end, ascending start
    Row accumulators (DataFusion 42): count of non-null values; min / max of the non-null values under IEEE totalOrder, NULL when there
    are none; avg state (count, sum), merged by addition, evaluated as sum / count, NULL when no value was seen.
    out rows: (window_start, window_end, None, count, min, max, avg, seq of the input batch that made the Final stage emit it, sum)."""

    def __init__(self, L, S=0):
        self.L, self.S = L, S
        self.partial = {}            # start -> frame (a dict), the BTreeMap of the Partial stream
        self.p_wm = None
        self.final = {}              # cached_frames of the Final stream
        self.seen = set()            # seen_windows
        self.f_wm = None             # a window START
        self.seq = 0
        self.out = []

    @staticmethod
    def _new(start, end):
        return {"start": start, "end": end, "cnt": 0, "sum": None, "mn": None, "mx": None}

    @staticmethod
    def _absorb(fr, cnt, s, mn, mx):
        fr["cnt"] += cnt
        if s is not None:        # AvgAccumulator: `let v = self.sum.get_or_insert(0.); *v += x` -- the sum starts from +0.0
            fr["sum"] = (0.0 if fr["sum"] is None else fr["sum"]) + s
        if mn is not None and (fr["mn"] is None or total_key(mn) < total_key(fr["mn"])):
            fr["mn"] = mn
        if mx is not None and (fr["mx"] is None or total_key(mx) > total_key(fr["mx"])):
            fr["mx"] = mx

    def push(self, rows):
        seq = self.seq
        self.seq += 1
        if not rows:
            return
        tss = [r[0] for r in rows if r[0] is not None]
        mn, mx = min(tss), max(tss)
        # ---- Partial
        for (s, e) in windows_for(mn, mx, self.L, self.S):
            fr = self.partial.setdefault(s, self._new(s, e))
            for ts, val, _key in rows:
                if ts is None or not (s <= ts < e) or val is None:
                    continue
                self._absorb(fr, 1, val, val, val)
        if self.p_wm is None or self.p_wm <= mn:
            self.p_wm = mn
        closed = [self.partial[s] for s in sorted(self.partial) if self.p_wm >= self.partial[s]["end"]]
        for fr in closed:
            del self.partial[fr["start"]]
        if not closed:
            return                   # an empty batch goes downstream: the Final stream ignores it
        # ---- Final: one incoming batch with len(closed) rows
        start = max(fr["start"] for fr in closed)
        end = max(fr["end"] for fr in closed)
        if start in self.seen and start not in self.final:
            return                   # late data for a finalized window: the whole batch is dropped
        ff = self.final.setdefault(start, self._new(start, end))
        self.seen.add(start)
        for fr in closed:
            self._absorb(ff, fr["cnt"], fr["sum"], fr["mn"], fr["mx"])
        self.f_wm = start if self.f_wm is None else max(self.f_wm, start)
        for s in sorted(self.final):
            fr = self.final[s]
            if self.f_wm > fr["end"]:
                avg = None if fr["sum"] is None else fr["sum"] / fr["cnt"]
                self.out.append((fr["start"], fr["end"], None, fr["cnt"], fr["mn"], fr["mx"], avg, seq, fr["sum"]))
                del self.final[s]
