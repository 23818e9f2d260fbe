"""What the signal event log must hold, derived from per-frame transmission lists (shared by the event-log tests).

A key in frame f's list and not in frame f-1's was inserted in f (a START); the reverse is an erasure in f (a STOP). The lists
do not show the order in which one frame's keys were inserted, so a frame's STARTs are compared as a set; everything else is
compared in order: frames ascending, a frame's STARTs before its STOPs, the STOPs in ascending key."""
START, STOP, LOST = 1, 2, 3


class Expected:
    """Feed it consecutive frames' lists [(shift_hz, flush, key, power)]; it returns the frames whose map changed."""

    def __init__(self):
        self.prev = {}  # key -> shift_hz of the previous frame's list
        self.frame = 0

    def reset(self):  # the map was cleared without events; the frame count goes on
        self.prev = {}

    def feed(self, lists):
        out = []
        for fr in lists:
            cur = {k: s for s, _, k, _ in fr}
            starts = {k: s for k, s in cur.items() if k not in self.prev}
            stops = sorted((k, s) for k, s in self.prev.items() if k not in cur)
            if starts or stops:
                out.append((self.frame, starts, stops))
            self.prev = cur
            self.frame += 1
        return out


def assert_log_equals(events, expected, where=""):
    """events: [(kind, key, shift_hz, frame, time_ms, first_ms, last_ms)] as Band.get_events returns them."""
    frames = [e[3] for e in events]
    assert frames == sorted(frames), (where, "frames out of order")
    by_frame = {}
    for e in events:
        by_frame.setdefault(e[3], []).append(e)
    assert sorted(by_frame) == [f for f, _, _ in expected], (where, sorted(by_frame), [f for f, _, _ in expected])
    for f, starts, stops in expected:
        got = by_frame[f]
        kinds = [e[0] for e in got]
        assert kinds == [START] * len(starts) + [STOP] * len(stops), (where, f, kinds)
        assert {e[1]: e[2] for e in got[: len(starts)]} == starts, (where, f, "starts")
        assert [(e[1], e[2]) for e in got[len(starts):]] == stops, (where, f, "stops")


def assert_times(events, timeout_ms, max_time_ms, frame_time, live=None):
    """A START carries its frame's clock three times; a STOP the Signal's two times, and one of the two limits has passed.
    `live` (key -> start time) carries the open signals from one call to the next."""
    live = {} if live is None else live
    for kind, key, _, frame, t, first, last in events:
        assert t == frame_time(frame), (frame, t)
        if kind == START:
            assert first == last == t, (frame, key)
            live[key] = t
        else:
            assert kind == STOP and first == live.pop(key), (frame, key)
            assert last + timeout_ms <= t or first + max_time_ms <= t, (frame, key, first, last, t)
            assert first <= last <= t
    return live
