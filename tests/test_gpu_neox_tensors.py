"""The tensor contract of the GPT-NeoX-family runtime (b200_neox_load_tensor / b200_neox_start_session), for every architecture it hosts.

For each of GPT-NeoX, GPT-2 with and without model/lm_head, MPT, BLOOM and GPT-J, with the names and shapes the oracle's synthetic models use:
every tensor loads from a zero buffer of its type and size; one byte too many, or the wrong type, is a shape error; a session does not start while
any tensor is missing (loading one twice does not count twice) and starts once all are loaded; a layer index past the last layer, the other
architectures' names and GPT-2's model/lm_head in a model without it are unknown tensors."""
import ctypes as C

import numpy as np
import pytest

from oracle import alibi as A
from oracle import bindings as B
from oracle import gptj as J
from oracle import synth as S

pytestmark = pytest.mark.gpu

OK, UNKNOWN_TENSOR, TENSOR_SHAPE = 0, -3, -4
F32_MATRICES = {"model/wpe"}            # GPT-2's learned positions: the one 2-D tensor stored as f32

# name -> (arch, config, tensor shapes, has_lm_head)
ARCHS = {
    "neox": (0, S.NEOX_CONFIGS["neox-tiny"], S.neox_tensor_shapes, 0),
    "gpt2": (1, S.GPT2_CONFIGS["gpt2-tiny"], S.gpt2_tensor_shapes, 0),
    "gpt2_lm_head": (1, S.GPT2_CONFIGS["gpt2-tiny"], lambda hp: S.gpt2_tensor_shapes(hp, lm_head=True), 1),
    "mpt": (2, A.MPT_CONFIGS["mpt-tiny"], A.mpt_tensor_shapes, 0),
    "bloom": (3, A.BLOOM_CONFIGS["bloom-tiny"], A.bloom_tensor_shapes, 0),
    "gptj": (4, J.GPTJ_CONFIGS["gptj-tiny"], J.gptj_tensor_shapes, 0),
}
WTYPE = B.Q4_0


def tensor_type(name, shape):
    return B.F32 if len(shape) == 1 or name in F32_MATRICES else WTYPE


def zeros(name, shape, extra=0):
    typ = tensor_type(name, shape)
    n = B.row_bytes(typ, shape[-1]) * (shape[0] if len(shape) == 2 else 1)
    return typ, np.zeros(n + extra, np.uint8)


@pytest.mark.parametrize("which", list(ARCHS))
def test_tensor_contract(which):
    from llm_b200 import _lib
    from llm_b200.neox import NeoxHparams, _bind
    L = _bind(_lib.lib())
    assert L.b200_init(0) == 0
    arch, cfg, shapes_of, has_lm_head = ARCHS[which]
    hp = NeoxHparams(n_vocab=cfg["n_vocab"], n_embd=cfg["n_embd"], n_head=cfg["n_head"], n_layer=cfg["n_layer"], n_rot=cfg.get("n_rot", 0),
                     use_parallel_residual=cfg.get("use_parallel_residual", 1), wtype=WTYPE, context_size=cfg["n_ctx"], arch=arch, has_lm_head=has_lm_head)
    m = L.b200_neox_new_alibi(C.byref(hp), float(cfg.get("alibi_bias_max", 8.0))) if arch in (2, 3) else L.b200_neox_new(C.byref(hp))
    assert m

    def load(name, typ, buf):
        return L.b200_neox_load_tensor(m, name.encode(), typ, buf.ctypes.data_as(C.c_void_p), buf.nbytes)

    try:
        shapes = shapes_of(cfg)
        names = list(shapes)
        for i, name in enumerate(names):
            typ, buf = zeros(name, shapes[name])
            assert load(name, typ, zeros(name, shapes[name], extra=1)[1]) == TENSOR_SHAPE, name
            wrong = WTYPE if typ == B.F32 else B.F32
            assert load(name, wrong, buf) == TENSOR_SHAPE, name
            assert not L.b200_neox_start_session(m, 8), name
            assert load(name, typ, buf) == OK, name
            if i == len(names) - 2:                 # every tensor but the last loaded: loading one again does not complete the model
                assert load(names[0], *zeros(names[0], shapes[names[0]])) == OK
                assert not L.b200_neox_start_session(m, 8)
        s = L.b200_neox_start_session(m, 8)
        assert s
        L.b200_neox_session_free(s)

        one = np.zeros(4, np.uint8)
        past_last = set(shapes_of(dict(cfg, n_layer=cfg["n_layer"] + 1))) - set(shapes)
        assert past_last
        others = set()
        for _, o_cfg, o_shapes, _ in ARCHS.values():
            others |= set(o_shapes(o_cfg))
        others -= set(shapes)
        if which == "gpt2":
            assert "model/lm_head" in others
        for name in sorted(past_last | others):
            assert load(name, B.F32, one) == UNKNOWN_TENSOR, name
            assert load(name, WTYPE, one) == UNKNOWN_TENSOR, name
    finally:
        L.b200_neox_free(m)
