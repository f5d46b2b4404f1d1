"""Page ownership across a failed batch admission.

The refusals of test_batch_admit_gpu.test_errors_admit_nothing all happen before any device work.  Here the admission fails after its
device work has begun: the vision tower of an image request whose prompt has one <|image_pad|> too few has run, and in batch_add_many the
text requests beside it have had their pages mapped and their pack prefilled.  Every page and slot the call took must go back: the running
request steps on to its oracle ids, eight requests can then fill the whole KV pool, and the handle serves single requests again."""
import numpy as np
import pytest

from conftest import make_model, make_oracle
from test_batch_admit_gpu import _Session, _ids, _oracle_generate

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vl():
    cfg, w, m = make_model("qwen3vl", "tiny", max_ctx=2048, max_patches=1024)
    yield cfg, w, m, make_oracle("qwen3vl", cfg, w)
    m.close()


def _text(V, n, seed, max_tokens):
    return dict(input_ids=_ids(n, V, seed), data=[None] * 5, max_tokens=max_tokens)


def _image_request_one_pad_short(cfg):
    from aha_b200 import synth
    from oracle.qwen3vl import process_image
    pv, grid = process_image(synth.synth_image(256, 320, 1))
    ids = synth.vl_prompt_ids(cfg, grid, 12)
    pad = int(np.flatnonzero(ids == cfg["image_token_id"])[0])
    return dict(input_ids=np.delete(ids, pad), data=[pv, grid, None, None, None], max_tokens=10)


@pytest.mark.parametrize("many", [True, False], ids=["batch_add_many", "batch_add"])
def test_failed_admission_returns_pages_and_slots(vl, many):
    from aha_b200 import B200Error
    cfg, w, m, o = vl
    V = cfg["text_config"]["vocab_size"]
    running = _text(V, 40, 31, 24)
    bad = _image_request_one_pad_short(cfg)
    s = _Session(m)
    try:
        s.add("A", running)
        s.step(2)
        with pytest.raises(B200Error, match="n_image_token num"):
            if many:   # the two text requests are packed and prefilled before the image request is reached
                m.batch_add_many([_text(V, 50, 32, 8), _text(V, 20, 33, 8), bad])
            else:      # prefilled alone on the slot's own table
                m.batch_add(**bad)
        s.drain()
        assert s.out["A"] == _oracle_generate(o, running)
        # nothing leaked: eight requests of 8 pages each exactly fill the 64-page pool (max_ctx 2048) and every slot
        res = m.batch_add_many([_text(V, 200, 40 + i, 56) for i in range(8)])
        assert [r[0] for r in res] == list(range(8))
        assert len(m.batch_step()) == 8
    finally:
        s.close()
    single = _text(V, 30, 50, 6)
    toks, _ = m.generate(single["input_ids"], single["data"], max_tokens=single["max_tokens"])
    assert toks == _oracle_generate(o, single)
