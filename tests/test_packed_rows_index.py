"""CPU tests of the packed-row decoder's host side: the packing index (len_s, cu, positions, padded-row map) on crafted
spliced labels, and the packed launch sequence against a recording stand-in for the C ABI."""
import ctypes

import torch

from oracle import llava_dpo_oracle as O

IGN = -100


def _labels(T, supervised):
    """[nseq, T] spliced labels; supervised[s] = the positions of sequence s that carry a label."""
    lab = torch.full((len(supervised), T), IGN, dtype=torch.int64)
    for s, ts in enumerate(supervised):
        for t in ts:
            lab[s, t] = 7
    return lab


def test_packing_index_on_crafted_labels():
    from rlaifv_b200.model import pack_rows, packed_lengths
    T = 10
    # no supervised label -> 1 row; truncated at max_len (label at T-1) -> T rows; a label at 0 -> 1 row; a gap
    lab = _labels(T, [[], [3, 4, 9], [0], [2, 5]])
    assert packed_lengths(lab).tolist() == [1, 10, 1, 6]
    pk = pack_rows(lab)
    assert (pk.nseq, pk.T, pk.M, pk.max_len) == (4, T, 18, 10)
    assert pk.cu.dtype == torch.int32 and pk.cu.tolist() == [0, 1, 11, 12, 18]
    assert pk.pos.tolist() == [0] + list(range(10)) + [0] + list(range(6))
    assert pk.rows.tolist() == [0] + list(range(10, 20)) + [20] + list(range(30, 36))
    # padded positions of the compact head -> packed rows (-1 slots stay -1)
    rp = torch.tensor([13, 18, -1, 32, 34, -1], dtype=torch.int32)
    assert pk.packed_rows(rp).tolist() == [4, 9, -1, 14, 16, -1]
    # every sequence already ends at its last supervised position: nothing to pack
    assert pack_rows(_labels(T, [[9], [1, 9], [9]])) is None
    # all sequences of length 1
    pk = pack_rows(_labels(T, [[], [0]]))
    assert pk.M == 2 and pk.max_len == 1 and pk.rows.tolist() == [0, 10] and pk.pos.tolist() == [0, 0]


def test_packed_launch_sequence_dry_run(monkeypatch):
    """A ragged batch with packing on: the decoder's attention, RoPE and LoRA dropout go through the packed entry
    points with M rows, the head through the packed rows of the supervised positions."""
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    c = O.TINY
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    calls, argv = [], {}

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name
        calls.append(name)
        argv.setdefault(name, []).append(args)

    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    # the stand-in computes nothing: give the compact head valid slots (padded positions, -1 = unused)
    monkeypatch.setattr(ops, "supervised_rows", lambda lab, cap: torch.tensor(
        [39, 58] + [-1] * (cap - 2) + [129] + [-1] * (cap - 1) + [-1] * cap + [200] + [-1] * (cap - 1), dtype=torch.int32))
    pol = LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))
    assert not pol.pack_rows                   # a CPU policy keeps the padded layout unless asked
    pol.pack_rows = True
    pol.enable_lora(r=8, alpha=2.0, dropout=0.05)
    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    T = 60
    labels = _labels(T, [[40, 59], [30, 45], [50], [20, 21]])
    monkeypatch.setattr(pol, "splice", lambda ids, lab, rows, nb, idx, T_hint=None: (
        torch.zeros(4 * T, dims.hidden_size, dtype=torch.bfloat16), labels, torch.zeros(4, T, dtype=torch.int32), T))
    pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    M = 60 + 46 + 51 + 22
    assert pol._stash["pack"].M == M
    pol.backward_logps(torch.zeros(4))
    n = dims.num_layers
    assert calls.count("rlaifv_attention_varlen_fwd") == calls.count("rlaifv_attention_varlen_bwd") == n
    assert calls.count("rlaifv_rope_pos_fwd") == calls.count("rlaifv_rope_pos_bwd") == n
    assert "rlaifv_attention_bwd_split" not in calls and "rlaifv_rope_fwd_gqa" not in calls
    assert calls.count("rlaifv_attention_fwd") == dims.clip_layers_used          # the CLIP tower is not packed
    assert all(a[10] == M for a in argv["rlaifv_attention_varlen_fwd"])      # n_rows
    assert calls.count("rlaifv_dropout_rows_fwd") == 2 * 4 * n and "rlaifv_dropout_fwd" not in calls
    assert calls.count("rlaifv_dropout_rows_bwd_add") == 4 * n
