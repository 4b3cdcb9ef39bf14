"""Decode kernels enqueued one by one (B200_SESSION_NO_GRAPH), token after token with nothing on the stream between them: the attention
kernel reads n_past and the older KV cache ahead of griddepcontrol.wait, which is only right if every kernel of the previous token has completed
before the next token's first kernel starts.  Logits and KV cache must stay bit-identical to the oracle."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import synth

pytestmark = pytest.mark.gpu

NO_GRAPH = 1      # B200_SESSION_NO_GRAPH


@pytest.mark.parametrize("cfg", ["tiny8", "gqa8"])
def test_back_to_back_device_decode_without_graph(orc, cfg):
    import llm_b200
    hp, tens = synth.make_llama(synth.CONFIGS[cfg], B.Q4_0, orc.quantize)
    toks = synth.make_tokens(hp, 40)
    mo = orc.llama(hp, tens)
    m = llm_b200.Llama(hp, llm_b200.ModelParameters(context_size=hp["n_ctx"]), tens)
    s = m.start_session(llm_b200.InferenceSessionConfig(n_batch=64, flags=NO_GRAPH))
    s.evaluate(toks[:21])
    mo.eval(toks[:21])
    # the device-resident call takes the token ids already in HBM (the first id of the last evaluate) and returns without synchronising
    for _ in range(12):
        assert s.L.b200_session_evaluate_device(s._s, None, 1) == 0
        mo.eval(toks[:1])
    g = s.evaluate(toks[21:22], all_logits=True)
    c = mo.eval(toks[21:22])
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32), np.asarray(c, np.float32).view(np.uint32)), "logits not bit-identical"
    for which in (0, 1):
        a = s.kv(which)
        assert np.array_equal(a, mo.kv(which)[:a.size]), which
    s.close()
    m.close()
