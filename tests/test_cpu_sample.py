"""
The fp64 sampler restatement (oracle/sample_oracle.py) that test_gpu_sample.py holds both sampler kernels to: Philox4x32-10
against its published known-answer vectors, the processor chain against the HF processors where no ties exist, the tie rules
the kernel documents, the fp32 prefix sums of the draw, and the argument checks of the ``dtk_dbg_sample`` hook.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import sample_oracle as so

KAT = [  # (counter, key, output) from the Random123 distribution's kat_vectors (philox4x32 10 rounds)
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answer_vectors(ctr, key, want):
    assert so.philox4x32_10(ctr, key).tolist() == list(want)


def test_uniform_counter_seed_and_seq_id():
    seed = 0x1234_5678_9ABC_DEF0
    # u is the top 24 bits of the first output word, for counter (step, seq_id, 0x243F6A88, 0x85A308D3)
    x = so.philox4x32_10((77, 5, 0x243F6A88, 0x85A308D3), (seed & 0xFFFFFFFF, seed >> 32))
    assert so.uniform(seed, 77, 5) == (int(x[0]) >> 8) / 2.0**24
    # the counter is step + gen_step modulo 2^32
    assert so.uniform(seed, 2**32 - 1, 9, gen_step=1) == so.uniform(seed, 0, 9)
    assert so.uniform(seed, 2**32 - 3, 9, gen_step=5) == so.uniform(seed, 2, 9)
    # both seed words, the step and the sequence id select different streams
    steps = np.arange(64)
    base = so.uniform(seed, steps, 3)
    for other in (so.uniform(seed & 0xFFFFFFFF, steps, 3), so.uniform(seed ^ 1, steps, 3), so.uniform(seed, steps + 1, 3),
                  so.uniform(seed, steps, 4)):
        assert (other != base).sum() >= 60
    u = so.uniform(seed, np.arange(4096), 0)
    assert u.min() >= 0 and u.max() < 1 and abs(u.mean() - 0.5) < 0.02


@pytest.fixture(scope="module")
def hf():
    from conftest import model_bundle
    cfg, _, oracle = model_bundle("tiny")
    return cfg, oracle


@pytest.mark.parametrize("temp,top_p,top_k", [(0.8, 0.95, 0), (1.3, 0.5, 0), (0.3, 1.0, 0), (0.7, 0.9, 50), (2.5, 1.0, 5),
                                              (1.0, 1e-3, 0), (0.8, 0.95, 1)])
@pytest.mark.parametrize("first_token", [True, False])
def test_chain_equals_hf_processors_without_ties(hf, temp, top_p, top_k, first_token):
    cfg, oracle = hf
    V = cfg.vocab_size
    g = torch.Generator().manual_seed(11)
    logits = torch.randn(4, V, generator=g) * 3
    logits[0, cfg.eos_token_id] = 15.0
    logits[1, cfg.image_token_id] = 15.0
    prompt_len = 10
    ids = torch.zeros(1, prompt_len if first_token else prompt_len + 3, dtype=torch.long)
    got = so.processed_probs(logits.numpy(), temp, top_p, top_k, bad_token=cfg.image_token_id,
                             begin_suppress_token=cfg.eos_token_id, suppress=first_token)
    for b in range(4):
        ref = oracle.processed_probs(ids, logits[b:b + 1], prompt_len, temperature=temp, top_p=top_p, top_k=top_k)[0].double()
        ref = ref.numpy()
        # HF sums the sorted probabilities in fp32: a token whose ascending mass is within fp32 rounding of the limit may land
        # on either side
        edge = np.abs(got["mass_below"][b] - so.top_p_limit(top_p)) < 1e-6 if top_p < 1 else np.zeros(V, bool)
        assert ((ref > 0) != got["kept"][b])[~edge].sum() == 0
        if ((ref > 0) != got["kept"][b]).sum() == 0:
            np.testing.assert_allclose(got["probs"][b], ref, rtol=2e-6, atol=1e-7)
        assert got["probs"][b, cfg.image_token_id] == 0
        if first_token:
            assert got["probs"][b, cfg.eos_token_id] == 0
    if not first_token:
        assert got["probs"][0, cfg.eos_token_id] > 0


def test_chain_ties_are_kept_or_dropped_together():
    V = 10
    # an all-equal row: every top-k keeps the whole tie group, and top-p cannot split it
    flat = np.zeros((1, V))
    for top_k in (0, 1, 5, V):
        for top_p in (1.0, 0.95, 0.5, 1e-3):
            r = so.processed_probs(flat, 0.8, top_p, top_k)
            assert r["kept"].all()
            np.testing.assert_allclose(r["probs"], 1 / V, rtol=1e-15)
    # ties at the k-th score: k = 2 keeps all three tokens tied at the second score
    row = np.array([[5.0, 3.0, 3.0, 1.0, 3.0, 0.0, -1.0, 2.0, 2.5, 4.0]])
    r = so.processed_probs(row, 1.0, 1.0, 2)
    assert np.flatnonzero(r["kept"][0]).tolist() == [0, 9]
    r = so.processed_probs(row, 1.0, 1.0, 3)
    assert np.flatnonzero(r["kept"][0]).tolist() == [0, 1, 2, 4, 9]
    r = so.processed_probs(row, 1.0, 1.0, 4)
    assert np.flatnonzero(r["kept"][0]).tolist() == [0, 1, 2, 4, 9]
    # two tokens tied at the maximum survive top_k = 1 and any top_p
    row = np.array([[1.0, 4.0, 0.0, 4.0, 2.0]])
    for top_p in (1.0, 0.5, 1e-3):
        r = so.processed_probs(row, 1.0, top_p, 1)
        assert np.flatnonzero(r["kept"][0]).tolist() == [1, 3]
        np.testing.assert_allclose(r["probs"][0, [1, 3]], 0.5, rtol=1e-15)
    # ties straddling the top-p limit: probabilities (0.4, 0.2, 0.2, 0.2); ascending mass at 0.2 is 0.6 for the whole group
    row = np.log(np.array([[0.2, 0.4, 0.2, 0.2]]))
    for top_p, kept in ((0.5, [0, 1, 2, 3]), (0.45, [0, 1, 2, 3]), (0.39, [1]), (0.3, [1])):
        r = so.processed_probs(row, 1.0, top_p, 0)
        assert np.flatnonzero(r["kept"][0]).tolist() == kept, top_p
    # HF's sorted cumulative sum would split that group at top_p = 0.5 (it keeps the 0.4 and one of the 0.2s)
    np.testing.assert_allclose(so.mass_at_or_below(np.array([[0.2, 0.4, 0.2, 0.2]])), [[0.6, 1.0, 0.6, 0.6]])


def test_chain_masks_temperature_and_greedy():
    row = np.array([[1.0, 7.0, 7.0, 3.0, 9.0, 2.0]])
    r = so.processed_probs(row, 0.5, 1.0, 0, bad_token=4, begin_suppress_token=1, suppress=True)
    assert r["probs"][0, 4] == 0 and r["probs"][0, 1] == 0
    e = np.exp((np.array([1.0, 0, 7.0, 3.0, 0, 2.0]) - 7.0) / 0.5) * np.array([1, 0, 1, 1, 0, 1])
    np.testing.assert_allclose(r["probs"][0], e / e.sum(), rtol=1e-14)
    # greedy: lowest index among tied maxima of the masked logits
    assert so.greedy(row, bad_token=4).tolist() == [1]
    assert so.greedy(row, bad_token=4, begin_suppress_token=1, suppress=True).tolist() == [2]
    assert so.greedy(np.zeros((1, 7))).tolist() == [0]
    assert not so.is_sampling(True, 9e-6) and so.is_sampling(True, 1e-5) and not so.is_sampling(False, 1.0)
    # a row that is -inf outside three tokens
    row = np.full((1, 50), -np.inf)
    row[0, [3, 17, 40]] = [0.0, 1.0, 2.0]
    r = so.processed_probs(row, 1.0, 1.0, 10)
    assert np.flatnonzero(r["kept"][0]).tolist() == [3, 17, 40]


def test_draw_is_inverse_cdf_in_index_order():
    p = np.array([[0.0, 0.25, 0.0, 0.5, 0.25]])
    assert so.draw(p, 0.0).tolist() == [1]
    assert so.draw(p, 0.2499).tolist() == [1]
    assert so.draw(p, 0.25).tolist() == [3]
    assert so.draw(p, 0.75).tolist() == [4]
    assert so.draw(p, 0.999999).tolist() == [4]
    assert so.draw(p * 0.5, 0.6).tolist() == [5]   # beyond the total: the kernel falls back to the argmax


@pytest.mark.parametrize("V", [264, 32769, 128256])
def test_kernel_prefix_sums_track_fp64(V):
    rng = np.random.default_rng(V)
    x = rng.standard_normal(V) * 2
    p = np.exp(x - x.max())
    p32 = (p / p.sum()).astype(np.float32)
    p32[rng.integers(0, V, V // 7)] = 0
    b64, b32 = so.kernel_prefix_sums(p32)
    per = -(-V // 1024)
    chunks = np.add.reduceat(p32 > 0, np.arange(0, V, per))
    assert b64.size == (p32 > 0).sum() + 2 * (chunks > 0).sum()
    assert np.isclose(b64.max(), p32.astype(np.float64).sum(), rtol=0, atol=1e-12)
    # first-order bound of the fp32 summation: (2 per + 13) roundings of values <= the total
    assert np.abs(b32 - b64).max() <= (2 * per + 13) * 2.0**-24 * b64.max()


def test_dbg_sample_refuses_bad_arguments():
    """The engine-free sampler hook checks its arguments before it touches the device."""
    from detikzify_b200 import _lib
    from detikzify_b200.engine import Engine
    lib = _lib.load_library()
    params = Engine.sampling(temperature=0.8, top_p=0.95, do_sample=True, seed=1)
    buf = (C.c_float * 64)()
    ids = (C.c_int64 * 64)()
    ptr, out = C.cast(buf, C.c_void_p), C.cast(ids, C.c_void_p)

    def call(B, V, impl=0, logits=ptr, probs=ptr, p=C.byref(params)):
        return lib.dtk_dbg_sample(logits, B, V, p, None, None, None, impl, out, probs, None)
    for B, V, impl in ((0, 8, 0), (65, 8, 0), (-1, 8, 0), (1, 0, 0), (1, -5, 1), (1, 8, 2), (1, 8, -1)):
        assert call(B, V, impl) == -1, (B, V, impl)
    assert call(1, 8, probs=None) == -1          # the probability vector is required
    assert call(1, 8, logits=None) == -1
    assert call(1, 8, p=None) == -1
