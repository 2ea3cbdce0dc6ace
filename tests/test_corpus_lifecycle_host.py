"""CPU: the float64 corpus model of tests/corpus_model.py, before tests/test_corpus_lifecycle_gpu.py judges any kernel by
it.  Its scores against the numpy oracle for every storage, its id sets through scripted sequences (the documented
no-ops and refusals), its gather, and the sequence generator's reach: every operation kind and edge, for the seeds the
GPU module runs."""
import numpy as np
import pytest
import torch

import corpus_model as M
import fp8_oracle as F8
import scan_fp64 as S
from oracle import maxsim_oracle as O



def _small(storage, pid_base=5, seed=1):
    rng = np.random.default_rng(seed)
    lens = np.array([1, 3, 4, 96, 1, 17, 95, 2, 40], np.int64)
    toks = M.passage_tokens(seed, int(lens.sum()), storage)
    return M.CorpusModel(toks, lens, pid_base, storage), toks, lens, rng


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("storage", M.STORAGES)
def test_model_scores_match_the_numpy_oracle(storage, relu):
    """After appends, deletions and a compaction: live scores within the fp32 oracle's rigorous bound (e4m3: the fp8
    oracle over rounded operands), deleted ids at -inf, and a token dropped from a passage moves a score far outside."""
    m, toks, lens, _ = _small(storage)
    t2 = M.passage_tokens(2, 1 + 5 + 97, storage)
    m.append(t2, [1, 5, 97])
    m.delete([5 + 1, 5 + 10])
    m.compact()
    m.delete([5 + 3])
    Q = M.query_rows(3, 3, 33, storage)
    s, amax, rabs = m.scores(Q, relu=relu)
    D = torch.cat([toks, t2]).float().numpy()
    dl = np.concatenate([lens, [1, 5, 97]])
    if storage == "fp8":
        ref = F8.maxsim_scores_fp8(Q.float().numpy(), D, dl, relu=relu)
        a8 = S.maxsim_packed(Q.float(), torch.from_numpy(D), dl, relu=relu, storage="fp8")
        assert torch.equal(a8[1], amax) and torch.equal(a8[2], rabs)
    else:
        ref = O.maxsim_scores(Q.float().numpy(), D, dl, relu=relu)
    bound = S.simt_bound(amax, rabs, 33)
    dead = np.array([1, 10, 3])
    live = np.setdiff1d(np.arange(dl.size), dead)
    assert torch.isneginf(s[:, dead]).all()
    err = (torch.from_numpy(ref[:, live]).double() - s[:, live]).abs()
    assert (err <= bound[:, live]).all(), float((err / bound[:, live]).max())
    # sensitivity: passage 3 (96 tokens) without its best token for query 0's row 0
    if not relu and storage != "fp8":
        off = np.concatenate([[0], np.cumsum(dl)])
        m2 = M.CorpusModel(torch.cat([toks, t2]), dl, 5, storage)
        j = int((torch.from_numpy(D).double()[off[3]:off[4]] @ Q[0, 0].double()).argmax())
        keep = np.ones(D.shape[0], bool)
        keep[off[3] + j] = False
        dl2 = dl.copy()
        dl2[3] -= 1
        m3 = M.CorpusModel(torch.cat([toks, t2])[torch.from_numpy(keep)], dl2, 5, storage)
        a, b = m2.scores(Q)[0][0, 3], m3.scores(Q)[0][0, 3]
        assert (a - b).abs() > 10 * m.bound(amax, rabs, 33)[0, 3]


def test_model_id_sets_through_a_scripted_sequence():
    m = M.CorpusModel(None, [3] * 10, pid_base=100)
    assert m.append(None, [1, 2]).tolist() == [110, 111]
    assert m.delete([100, 105, 105]) == 2
    assert m.delete([100]) == 0                                # already deleted: no change
    with pytest.raises(M.ModelError):
        m.delete([101, 112])                                   # one past the end: refused, nothing changes
    with pytest.raises(M.ModelError):
        m.delete([99])
    assert m.deleted_ids().tolist() == [100, 105] and m.n_live == 10
    assert m.compact() == 2 and m.n_stored == 10 and m.n_passages == 12
    assert m.compacted_ids().tolist() == [100, 105]
    assert m.compact() == 0                                    # nothing stored is deleted: a no-op
    assert m.delete([105]) == 0 and m.n_deleted == 2           # compacted away: no change
    assert m.append(None, [4]).tolist() == [112]               # ids continue from the extent
    assert m.new_ids().tolist() == [112]
    m.delete([112, 101])
    assert m.compact() == 2 and m.n_stored == 9 and m.new_ids().size == 0
    m.delete(m.live_ids())
    with pytest.raises(M.ModelError):
        m.compact()                                            # every stored passage deleted: refused
    assert m.n_stored == 9 and m.n_live == 0 and m.n_compactions == 2
    assert m.stored_ids().tolist() == sorted(set(range(100, 113)) - {100, 105, 101, 112})


@pytest.mark.parametrize("storage", M.STORAGES)
def test_model_gather(storage):
    m, toks, lens, _ = _small(storage, pid_base=5)
    m.delete([5 + 2])
    m.compact()
    m.delete([5 + 5])
    ids = np.array([5 + 3, 5 + 2, 5 + 5, 4, 5 + 9, 5 + 0, 5 + 8])
    D, mask = m.gather(ids, 100)
    assert D.dtype == M.element_dtype(storage) and D.shape == (7, 100, 128) and mask.shape == (7, 100, 1)
    off = np.concatenate([[0], np.cumsum(lens)])
    for r, p in enumerate(ids - 5):
        if 0 <= p < lens.size and p not in (2, 5):
            n = int(lens[p])
            assert torch.equal(D[r, :n], toks[off[p]:off[p] + n]) and mask[r, :n].all()
            assert not D[r, n:].any() and not mask[r, n:].any()
        else:
            assert not D[r].any() and not mask[r].any()
    # zero rows are +0, bit for bit
    assert (D[1].view(torch.int16) == 0).all()


@pytest.mark.parametrize("case", M.SEQUENCE_CASES, ids=lambda c: "%d-%s" % (c[0], c[1]))
def test_generator_reaches_every_edge(case):
    seed, storage, pid_base, adopt = case
    spec, ops = M.generate(seed, storage, pid_base, adopt, sms=132)
    seen = set()
    for op in ops:
        seen.update(op["tags"])
    assert set(M.EDGES) <= seen, sorted(set(M.EDGES) - seen)
    assert 20 <= len(ops) <= 32, len(ops)
    assert {op["op"] for op in ops} == {"append", "delete", "compact"}
    assert {op["src"] for op in ops if op["op"] == "append"} == {"cpu", "gpu"}
    # the ops replay on a fresh model to the same expectations
    m = M.CorpusModel(None, spec["lens0"], spec["pid_base"])
    for op in ops:
        if op["op"] == "append":
            m.append(None, op["lens"])
            continue
        try:
            m.delete(op["ids"]) if op["op"] == "delete" else m.compact()
            got = "ok"
        except M.ModelError:
            got = "error"
        assert got == op["expect"], op


def test_generator_adopted_start_has_lengths_in_fours():
    spec, _ = M.generate(11, adopt=True)
    assert all(x % 4 == 0 for x in spec["lens0"]) and spec["src0"] == "gpu"


def test_large_sequence_crosses_a_physical_piece():
    spec, ops = M.large_sequence(31)
    piece_rows = (1 << 30) // 256
    lens0 = np.asarray(spec["lens0"])
    m = M.CorpusModel(None, lens0, spec["pid_base"])
    assert lens0.sum() > piece_rows
    for op in ops:
        if op["op"] == "append":
            m.append(None, op["lens"])
        elif op["op"] == "delete":
            m.delete(op["ids"])
        else:
            m.compact()
            stored = m.stored_ids() - m.pid_base
            if m.n_compactions == 1:
                assert m.lens[stored].sum() < piece_rows            # the first compaction frees the second piece
    assert m.lens[m.stored_ids() - m.pid_base].sum() > piece_rows   # and the append after it maps one again
