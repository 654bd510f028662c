"""Helpers for tests/test_spec_text.py: the reference's VSR.tla executed by oracle/tla_eval.py, side by side with the
C++ oracle.  States travel between the two as text: the oracle prints a state (TLC value syntax), tla_eval parses it.

The spec's text is not part of this repository.  What the text evaluator answered is stored in tests/golden/
spec_text_answers.json, in the order the tests ask; the tests compare the oracle and the product with those answers.
With VSR_SPEC_TLA naming the reference's VSR.tla, the evaluator runs on the text instead and the answers are recorded
again (tests/golden/make_spec_text_answers.py)."""
import atexit
import collections
import ctypes as C
import hashlib
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import tla_eval as T  # noqa: E402
import orc  # noqa: E402

SPEC = os.environ.get("VSR_SPEC_TLA")
ANSWERS = os.path.join(ROOT, "tests", "golden", "spec_text_answers.json")
ACTIONS = ["Initial predicate", "TimerSendSVC", "ReceiveHigherSVC", "ReceiveMatchingSVC", "SendDVC", "ReceiveHigherDVC",
           "ReceiveMatchingDVC", "SendSV", "ReceiveSV", "ReceiveClientRequest", "ReceivePrepareMsg", "ReceivePrepareOkMsg",
           "ExecuteOp", "SendGetState", "ReceiveGetState", "ReceiveNewState", "RestartEmpty", "ReceivesRecoveryMsg",
           "ReceivesRecoveryResponseMsg", "CompleteRecovery"]


def evaluator(R, V, L, restart=0):
    """the text evaluator, or None when only the recorded answers are available"""
    return T.load_vsr(SPEC, R, 1, ["v%d" % (i + 1) for i in range(V)], L, restart) if SPEC else None


_recorded = None


class Answers:
    """The text's answers to one test, in the order it asks.  value(fn): with the spec's text, fn() is computed, stored and
    returned; without it, the stored answer is returned.  Answers are JSON values (lists, not tuples)."""

    def __init__(self, name):
        global _recorded
        self.name = name
        if SPEC:
            self.seq = []
            if name is None:  # a comparison no test replays (tests/golden/make_spec_text_fixture.py's sweep)
                return
            if _recorded is None:
                _recorded = {}
                atexit.register(_write_answers)
            _recorded[name] = self.seq
        else:
            with open(ANSWERS) as f:
                self.seq = json.load(f)[name]
        self.i = 0

    def value(self, fn):
        if SPEC:
            v = json.loads(json.dumps(fn()))
            self.seq.append(v)
            return v
        assert self.i < len(self.seq), "%s asks more of the text than was recorded" % self.name
        self.i += 1
        return self.seq[self.i - 1]


def _write_answers():
    old = {}
    if os.path.exists(ANSWERS):
        with open(ANSWERS) as f:
            old = json.load(f)
    old.update(_recorded)
    with open(ANSWERS, "w") as f:
        f.write("{\n" + ",\n".join(json.dumps(k) + ":" + json.dumps(old[k], separators=(",", ":")) for k in sorted(old)) + "\n}\n")


def digest(items):
    """a multiset of values (tla_eval values, in tuples) as a short hash: the order of tla_eval.vkey, not of printing"""
    def key(x):
        return tuple(key(y) for y in x) if isinstance(x, tuple) else T.vkey(x)
    return hashlib.sha1(repr(sorted(key(x) for x in items)).encode()).hexdigest()[:12]


def to_py(q, flat):
    return T.parse_state_record(orc.print_flat(q, flat))


class Pair:
    """one configuration: the text evaluator and the oracle (symmetry off: literal successors on both sides)"""

    def __init__(self, pkg, R, V, L, restart=0, name=None):
        self.Flat = pkg.checker.VsrFlatState
        self.ev = evaluator(R, V, L, restart)
        self.text = Answers(name)
        self.q = orc.params(R, V, L, symmetry=False, restart=restart)
        self.q_awem = orc.params(R, V, L, symmetry=False, invariant=2, restart=restart)
        self.stats = collections.Counter()
        self.choose_retries = 0

    def init_flat(self):
        f = self.Flat()
        orc.lib().orc_init_flat(self.q, C.byref(f))
        return f

    def oracle_successors(self, flat, cap=512):
        out = (self.Flat * cap)()
        acts = (C.c_int * cap)()
        n = orc.lib().orc_successors_flat(self.q, C.byref(flat), out, acts, cap)
        assert 0 <= n <= cap, n
        return [(ACTIONS[acts[i]], out[i]) for i in range(n)]

    def compare(self, flat):
        """successors of one state from the text and from the oracle, as multisets of (action, whole next state);
        also the two safety invariants on the state itself.  Returns the oracle's successor flats."""
        st = to_py(self.q, flat)
        osucc = self.oracle_successors(flat)
        want = collections.Counter((a, T.Fn(to_py(self.q, f))) for a, f in osucc)
        text = self.text.value(lambda: self._text_answer(st, want))
        assert text[0] == digest(want.elements()), "successors differ from the text's\nstate: %s" % {k: T.fmt(v) for k, v in st.items()}
        for a, _ in osucc:
            self.stats[a] += 1
        assert text[1] == bool(orc.lib().orc_invariant_flat(self.q, C.byref(flat)))
        assert text[2] == bool(orc.lib().orc_invariant_flat(self.q_awem, C.byref(flat)))
        return osucc

    def _text_answer(self, st, want):
        """[digest of the text's successors, AcknowledgedWriteNotLost, AcknowledgedWritesExistOnMajority] of one state"""
        pick, got = 0, None
        while True:
            self.ev.choose_pick, self.ev.choose_log = pick, []
            got = collections.Counter((a, T.Fn(sp)) for a, sp in self.ev.successors(st))
            ambiguous = bool(self.ev.choose_log)
            if got == want or not ambiguous or pick >= 3:
                break
            pick += 1  # the result depended on which maximal DVC a CHOOSE took: try the others (TLC's order is not known here)
        self.ev.choose_pick = 0
        if pick and got == want:
            self.choose_retries += 1
        if got != want:
            only_text = [(a, T.fmt(s)) for (a, s) in (got - want)]
            only_orc = [(a, T.fmt(s)) for (a, s) in (want - got)]
            raise AssertionError("successors differ\nstate: %s\nonly from the text: %s\nonly from the oracle: %s" %
                                 ({k: T.fmt(v) for k, v in st.items()}, only_text[:3], only_orc[:3]))
        return [digest(got.elements()), bool(self.ev.holds("AcknowledgedWriteNotLost", st)),
                bool(self.ev.holds("AcknowledgedWritesExistOnMajority", st))]

    def walk(self, flat, steps, rng, prefer=()):
        """compare along a random walk; `prefer` = actions taken whenever enabled (to reach rare neighbourhoods)"""
        n = 0
        for _ in range(steps):
            succ = self.compare(flat)
            n += 1
            if not succ:
                break
            pref = [f for a, f in succ if a in prefer]
            flat = rng.choice(pref) if pref and rng.random() < 0.7 else rng.choice(succ)[1]
        return n


def follow(P, flat, actions):
    """depth-first: a path from `flat` whose steps carry the given action names (every state on the way is compared);
    returns the flats of the path or None"""
    succ = P.compare(flat)
    if not actions:
        return [flat]
    for a, f in succ:
        if a == actions[0]:
            r = follow(P, f, actions[1:])
            if r:
                return [flat] + r
    return None


def find_behaviour(ev, actions, invariant):
    """depth-first search for a behaviour of the module whose i-th step is an `actions[i]` step and whose last state
    violates `invariant`; returns the list of states or None"""
    init = ev.initial_states()[0]
    dead = set()

    def rec(st, i, path):
        if i == len(actions):
            return path if not ev.holds(invariant, st) else None
        key = (i, T.Fn(st))
        if key in dead:
            return None
        for a, sp in ev.successors(st):
            if a == actions[i]:
                r = rec(sp, i + 1, path + [sp])
                if r:
                    return r
        dead.add(key)
        return None
    return rec(init, 0, [init])
