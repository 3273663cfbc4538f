"""generate()'s device token loop, driven on the CPU through a stand-in session that records its calls: the decode_steps(n)
sequence per recorder set and with a streamer, the host synchronisations, the early stop, one streamer column per generated
step, and every recorder detached when the loop raises."""
from types import SimpleNamespace

import pytest
import torch

from parler_tts_b200.modeling import (ParlerTTSForConditionalGeneration, Sampling, StepAlignment, StepOutputs, StepProbes,
                                      take_shards)

B, K, V, S, H = 2, 3, 8, 4, 4


class FakeSession:
    """Columns advance by one per sampled step while the session is active; the step `stop_step` (its column n0 + stop_step)
    turns the active flag state[1] to 0, and decode step number `fail_call` raises."""

    def __init__(self, stop_step=None, fail_call=None):
        self.B, self.K, self.n0 = B, K, 1
        self.stop_step, self.fail_call = stop_step, fail_call
        self.calls = []
        self._state = torch.zeros(8, dtype=torch.int32)

    def begin(self, max_length, **kw):
        self.calls.append(("begin",))
        self._raw = torch.zeros(B * K, max_length, dtype=torch.int64)
        self._state[0], self._state[1] = 1, 1

    def prefill(self, *a):
        self.calls.append(("prefill",))

    def _advance(self, n):
        for _ in range(n):
            if self._state[1] == 0:
                return
            col = int(self._state[0])
            self._raw[:, col] = col
            self._state[0] += 1
            if self.stop_step is not None and col - self.n0 == self.stop_step:
                self._state[1] = 0

    def sample(self, forced=None):
        self.calls.append(("sample",))
        self._advance(1)

    def decode_steps(self, n):
        self.calls.append(("decode_steps", n))
        if self.fail_call is not None and sum(c[0] == "decode_steps" for c in self.calls) == self.fail_call:
            raise RuntimeError("decode step failed")
        self._advance(n)

    @property
    def state(self):
        self.calls.append(("state",))
        return self._state

    @property
    def raw_ids(self):
        return self._raw

    def set_outputs(self, logits, scores, first_step=0, n_steps=0, step_stride=0):
        self.calls.append(("set_outputs", None if logits is None and scores is None else first_step))

    def set_probes(self, self_attn=None, cross_attn=None, hidden=None, first_step=0, n_steps=0, self_ld=0):
        self.calls.append(("set_probes", None if self_attn is None and hidden is None else first_step))

    def set_alignment(self, heads=None, key0=0, key_len=0, out=None, first_row=0, n_rows=0):
        self.calls.append(("set_alignment", None if out is None else first_row))


class Streamer:
    def __init__(self):
        self.cols, self.ended = [], False

    def put(self, v):
        self.cols.append(v)

    def end(self):
        self.ended = True


def _model(sess):
    m = object.__new__(ParlerTTSForConditionalGeneration)
    m.config = SimpleNamespace(decoder=SimpleNamespace(num_codebooks=K, bos_token_id=V + 1, pad_token_id=V, eos_token_id=V))
    m.decoder = SimpleNamespace(engine=SimpleNamespace(session=lambda *a, **k: sess))
    m.device = torch.device("cpu")
    return m


def _recorders(names, L):
    make = dict(outputs=lambda: StepOutputs(B * K, V, "cpu", scores=True, logits=False),
                align=lambda: StepAlignment([[0, 0]], B, L - 1, 0, 2, "cpu"),
                probes=lambda: StepProbes(1, B, 1, S, H, 0, 1, torch.float32, "cpu", attentions=True, hidden=False))
    return [make[n]() for n in names]


def _sampling(L):   # greedy, nothing the host-driven loop needs
    return Sampling(L, False, 1.0, 0, 1.0, 0, 0, False, V, 0, None, None, [], [])


def _run(L, names=(), streamer=None, **fake):
    sess = FakeSession(**fake)
    ids = _model(sess)._run_token_loop(torch.zeros(B, S, H), None, None, None, None, _sampling(L), take_shards(B, 1, None)[0],
                                        _recorders(names, L), streamer)
    return sess, ids


def _steps(sess):
    return [c[1] for c in sess.calls if c[0] == "decode_steps"]


@pytest.mark.parametrize("names, expect", [
    ((), [64, 64, 64, 6]),                             # up to 64 tokens per call (one cluster kernel launch)
    (("align",), [64, 64, 64, 6]),                     # the alignment window spans the whole call
    (("outputs",), [63, 64, 64, 7]),                   # each call inside one 64-step chunk, from step 1
    (("probes",), [63, 64, 64, 7]),
    (("outputs", "align", "probes"), [63, 64, 64, 7]),
])
def test_decode_steps_calls_per_recorder_set(names, expect):
    sess, ids = _run(200, names)
    assert _steps(sess) == expect
    assert ids.shape == (B * K, 200)
    # the device `active` flag is read once after every call but the last, and cur_len once at the end
    loop = [c for c in sess.calls if c[0] in ("decode_steps", "state")]
    assert loop == [x for n in expect for x in (("decode_steps", n), ("state",))]


def test_recorder_windows_follow_the_chunks():
    sess, _ = _run(200, ("outputs", "align", "probes"))
    win = [c for c in sess.calls if c[0].startswith("set_")]
    assert win[:2] == [("set_alignment", 0), ("set_probes", 0)]              # attached for the prefill, in the given order
    assert [c[1] for c in win if c[0] == "set_outputs"] == [0, 0, 64, 128, 192, None]
    assert [c[1] for c in win if c[0] == "set_probes"] == [0, 1, 64, 128, 192, None]
    assert win[-3:] == [("set_probes", None), ("set_alignment", None), ("set_outputs", None)]   # detached in reverse


def test_early_stop_ends_the_loop_after_the_call_that_ended_it():
    sess, ids = _run(200, stop_step=100)
    assert _steps(sess) == [64, 64]
    assert ids.shape[1] == 1 + 101                                           # the BOS column and steps 0 .. 100


@pytest.mark.parametrize("stop_step", [None, 5])
def test_streamer_gets_one_column_per_generated_step(stop_step):
    st = Streamer()
    sess, ids = _run(40, ("outputs",), streamer=st, stop_step=stop_step)
    n_gen = ids.shape[1] - 1
    assert n_gen == (39 if stop_step is None else stop_step + 1)
    assert _steps(sess) == [1] * (n_gen - 1)
    assert st.ended and len(st.cols) == 1 + n_gen                           # the BOS column, then one per step
    assert all(torch.equal(c, ids[:, j]) for j, c in enumerate(st.cols[1:], start=1))
    # the active flag is read before every step, so no column follows the step that ended the session
    loop = [c[0] for c in sess.calls if c[0] in ("decode_steps", "state")]
    assert loop[:2] == ["state", "decode_steps"] and loop.count("decode_steps") == n_gen - 1


def test_every_recorder_is_detached_when_the_loop_raises():
    sess = FakeSession(fail_call=2)
    with pytest.raises(RuntimeError, match="decode step failed"):
        _model(sess)._run_token_loop(torch.zeros(B, S, H), None, None, None, None, _sampling(200), (0, B, 0, B),
                                     _recorders(("outputs", "align", "probes"), 200))
    assert sess.calls[-4:] == [("decode_steps", 64), ("set_probes", None), ("set_alignment", None), ("set_outputs", None)]
