"""oracle/sample.py pinned by what can be pinned here: the ChaCha core against the RFC 7539 block vector, the PCG32 seed
expansion and Uniform<f32> against hand-computed values of their published definitions, and the sampling modes against
brute-force restatements (full sort) on small vocabularies."""
import numpy as np

from oracle import sample as S


def test_chacha_core_rfc7539_block():
    key = [int.from_bytes(bytes(range(4 * i, 4 * i + 4)), "little") for i in range(8)]
    # RFC 7539 2.3.2: counter 1, nonce 00:00:00:09 00:00:00:4a 00:00:00:00 -> in djb's layout counter = 1 | 0x09000000 << 32, stream id words (0x4a000000, 0)
    blk = S.chacha_block(key, 1 | (0x09000000 << 32), 20, (0x4A000000, 0))
    assert blk[:4] == [0xE4E7F110, 0x15593BD1, 0x1FDD0F50, 0xC47120A3] and blk[15] == 0x4E3C50A2


def test_seed_expansion_and_uniform():
    w = S.seed_from_u64(0)
    # first PCG32 output for state 0: state' = INC; xorshifted = ((s >> 18) ^ s) >> 27; rot = s >> 59
    s = 11634580027462260723
    xs = (((s >> 18) ^ s) >> 27) & 0xFFFFFFFF
    rot = s >> 59
    assert w[0] == ((xs >> rot) | (xs << ((32 - rot) & 31))) & 0xFFFFFFFF
    r = S.StdRng(42)
    assert r.word(0) == S.chacha_block(r.key, 0, 12)[0] and r.word(17) == S.chacha_block(r.key, 1, 12)[1]
    u = r.uniform01(3)
    assert 0.0 <= u < 1.0 and u == np.float32(np.uint32((r.word(3) >> 9) | 0x3F800000).view(np.float32) - np.float32(1))


def test_sampling_mode_selection_follows_get_logit_processor():
    assert S.sampling_mode(None, 0.9, 10) == "argmax" and S.sampling_mode(1e-8, None, None) == "argmax"
    assert S.sampling_mode(0.7, None, None) == "all" and S.sampling_mode(0.7, 0.9, None) == "topp"
    assert S.sampling_mode(0.7, None, 5) == "topk" and S.sampling_mode(0.7, 0.9, 5) == "topk_topp"


def _brute_topp(p, top_p):
    order = np.lexsort((np.arange(len(p)), -p.astype(np.float64)))
    out = p.copy()
    cum = np.float32(0)
    for i in order:
        if cum >= np.float32(top_p):
            out[i] = 0
        else:
            cum = np.float32(cum + p[i])
    return out


def test_topp_weights_equal_the_sorted_walk_on_small_vocabularies():
    rng = np.random.default_rng(0)
    for trial in range(30):
        V = int(rng.integers(5, 400))
        lg = (rng.standard_normal(V) * 2).astype(np.float32)
        if trial % 3 == 0:
            lg[rng.integers(0, V, V // 3)] = lg[0]          # ties
        p = S.softmax_blocked(lg, 0.9)
        tp = float(rng.uniform(0.05, 0.98))
        assert np.array_equal(S.topp_weights(p, tp) > 0, _brute_topp(p, tp) > 0)


def test_blocked_pick_is_a_weighted_index():
    w = np.array([0, 0.5, 0, 0.25, 0.25], np.float32)
    assert S.blocked_pick(w, np.float32(0.0)) == 1 and S.blocked_pick(w, np.float32(0.49)) == 1
    assert S.blocked_pick(w, np.float32(0.5)) == 3 and S.blocked_pick(w, np.float32(0.76)) == 4
    big = np.ones(1000, np.float32)
    assert S.blocked_pick(big, np.float32(0.2555)) == 255 and S.blocked_pick(big, np.float32(0.256)) == 256   # crosses a chunk boundary
    counts = np.bincount([S.blocked_pick(w, S.StdRng(1).uniform01(i)) for i in range(2000)], minlength=5)
    assert counts[0] == 0 and counts[2] == 0 and abs(counts[1] / 2000 - 0.5) < 0.05


def test_topk_then_topp_with_k_over_the_vocabulary_is_a_nucleus_even_at_p_1():
    """candle's sample_topk_topp with k >= V runs sample_topp, which has no p >= 1 shortcut: where the fp32 sum of the softmax rounds
    to >= 1 the smallest entries are dropped and the pick moves.  These are the values the device sampler test pins at V = 151936."""
    lg = (np.random.default_rng(7).standard_normal(151936) * 1.5).astype(np.float32)
    p = S.softmax_blocked(lg, 0.9)
    assert S.blocked_sum(p) >= 1
    w = S.topp_weights(p, 1.0)
    assert np.count_nonzero(p) == 151936 and np.count_nonzero(w == 0) == 68
    assert np.count_nonzero(S.topp_weights(p, 1.5)) == 151936                 # p > 1 keeps everything
    r = S.StdRng(77)
    for draw, nucleus, plain in ((90, 106616, 106615), (384, 57439, 57440)):
        assert S.sample(lg, 0.9, 1.0, 151936, r, draw) == nucleus and S.blocked_pick(p, r.uniform01(draw)) == plain
        assert S.sample(lg, 0.9, 1.0, None, r, draw) == plain                   # TopP alone keeps candle's p >= 1 shortcut
        assert S.sample(lg, 0.9, None, 151936, r, draw) == plain                # and so does TopK with k >= V
    assert all(S.blocked_pick(w, r.uniform01(d)) == S.blocked_pick(p, r.uniform01(d)) for d in range(90))   # draw 90 is the first to move


def test_topk_then_topp_and_penalty():
    rng = np.random.default_rng(1)
    lg = rng.standard_normal(300).astype(np.float32)
    r = S.StdRng(9)
    top5 = set(np.argsort(-lg)[:5].tolist())
    assert all(S.sample(lg, 0.8, None, 5, r, i) in top5 for i in range(40))
    assert all(S.sample(lg, 0.8, 0.01, 5, r, i) == int(np.argmax(lg)) for i in range(10))      # a tiny nucleus keeps the best token only
    pen = S.use_repeat_penalty(2.0, 2, np.array([1.0, -1.0, 3.0], np.float32), [2, 0, 1, 1])
    assert pen.tolist() == [1.0, -2.0, 3.0]                                                       # last 2 tokens = [1, 1]: one application
    assert S.use_repeat_penalty(1.0, 64, lg, [1, 2]) is not None and np.array_equal(S.use_repeat_penalty(2.0, 0, lg, [1]), lg)
