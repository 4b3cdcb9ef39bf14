"""Sessions and models own their HBM: starting and freeing LLaMA (graph and per-op decode), GPT-NeoX and GPT-2 sessions over and over, decoding
two tokens in each, gives back every buffer they took (the tests and bench.py open many sessions in one process)."""
import ctypes as C

import pytest

from oracle import bindings as B
from oracle import synth

pytestmark = pytest.mark.gpu

NO_GRAPH = 1          # B200_SESSION_NO_GRAPH
SLACK = 2 << 20       # bytes: allocator granularity, far below one session's buffers
NEOX = dict(n_vocab=384, n_ctx=128, n_embd=256, n_head=4, n_layer=2, n_rot=16, use_parallel_residual=1, wtype=B.Q4_0)
GPT2 = dict(n_vocab=320, n_ctx=128, n_embd=256, n_head=4, n_layer=2, wtype=B.Q4_0)


def free_bytes():
    from llm_b200 import _lib
    fr = C.c_size_t()
    assert _lib.lib().b200_device_info(None, C.byref(fr), None) == 0
    return fr.value


def decode_two(s):
    s.evaluate([1])
    s.evaluate([2])
    s.close()


def cycle():
    import llm_b200
    from llm_b200.neox import Gpt2, GptNeoX
    hp = dict(synth.CONFIGS["tiny8"], wtype=B.Q4_0)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]))
    m.synthesize(1)
    for flags in (0, NO_GRAPH):
        decode_two(m.start_session(llm_b200.InferenceSessionConfig(n_batch=8, flags=flags)))
    m.close()
    for cls, hp in ((GptNeoX, NEOX), (Gpt2, GPT2)):
        m = cls(hp)
        m.synthesize(2)
        decode_two(m.start_session(8))
        m.close()


def test_sessions_release_their_memory():
    cycle()                               # warm-up: module loads, rope tables, the op arena
    first = free_bytes()
    for _ in range(5):
        cycle()
    last = free_bytes()
    assert first - last <= SLACK, f"{(first - last) / 2**20:.1f} MiB of HBM not returned over 5 cycles"
