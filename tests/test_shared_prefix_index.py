"""CPU tests of shared prompt prefixes' host side: pos0 from crafted spliced labels and sources (first difference,
first supervised row, rounding to 128), the shared RowPacking and its padded-row map, the policy's conditions for
sharing, and the launch sequence against a recording stand-in for the C ABI."""
import ctypes

import pytest
import torch

from oracle import llava_dpo_oracle as O

IGN = -100


def _pair_batch(T, firsts, diffs, lasts=None):
    """Spliced labels and sources of a preference batch [2b, T]: sequence s is labelled from firsts[s] + 1 (its first
    supervised row firsts[s]) to lasts[s]; pair i's rejected sources differ from position diffs[i] on (None = never)."""
    n = len(firsts)
    lab = torch.full((n, T), IGN, dtype=torch.int64)
    for s, f in enumerate(firsts):
        if f is not None:
            lab[s, f + 1:(lasts[s] if lasts else T - 1) + 1] = 9
    src = torch.arange(T).repeat(n, 1)
    for i, p in enumerate(diffs):
        if p is not None:
            src[n // 2 + i, p:] += 10 ** 6
    return lab, src


def test_pos0_first_difference_first_supervised_row_and_rounding():
    from rlaifv_b200.model import shared_prefix_lengths
    T = 1135
    # pair 0: bench-like (differ at 623, first supervised row 622) -> 512; pair 1: difference first (300) -> 256;
    # pair 2: prefix shorter than 128 -> 0; pair 3: identical sequences, capped at the first supervised row (700) -> 640;
    # pair 4: one side without a supervised row -> 0
    lab, src = _pair_batch(T, [622, 900, 100, 700, None] + [622, 950, 110, 700, 400], [623, 300, 120, None, 600])
    assert shared_prefix_lengths(lab, src).tolist() == [0] * 5 + [512, 256, 0, 640, 0]


def test_shared_packing_layout_and_padded_row_map():
    from rlaifv_b200.model import pack_rows
    T = 700
    lab, src = _pair_batch(T, [640, 99, 639, 299], [645, 300], lasts=[689, 199, 699, 309])
    pk = pack_rows(lab, src)
    assert pk.shared and pk.pos0_h.tolist() == [0, 0, 512, 0] and pk.partner_h.tolist() == [2, -1, 0, -1]
    assert torch.equal(pk.pos0, pk.pos0_h) and torch.equal(pk.partner, pk.partner_h)
    own = [690, 200, 700 - 512, 310]
    assert pk.cu.tolist() == [0, 690, 890, 1078, 1388] and pk.M == sum(own) and pk.max_len == 690
    assert pk.pos[890:893].tolist() == [512, 513, 514] and pk.rows[890:893].tolist() == [2 * T + 512 + i for i in range(3)]
    assert pk.pos[1077].item() == 699 and pk.rows[1077].item() == 3 * T - 1
    # a rejected position below pos0 -> the chosen sequence's row; at or above -> its own rows; -1 stays -1
    rp = torch.tensor([2 * T + 10, 2 * T + 511, 2 * T + 512, 2 * T + 699, T + 5, 3 * T + 7, -1], dtype=torch.int32)
    assert pk.packed_rows(rp).tolist() == [10, 511, 890, 1077, 695, 1085, -1]


def test_one_row_suffix_and_equal_length_batch_share():
    from rlaifv_b200.model import pack_rows
    T = 258
    # rejected: first supervised row 256 and last label at 257 -> 2 own rows; the batch has no padding to drop
    lab, src = _pair_batch(T, [256, 256], [None])
    pk = pack_rows(lab, src)
    assert pk is not None and pk.pos0_h.tolist() == [0, 256] and pk.M == T + 2
    assert pack_rows(lab) is None                          # without sources: nothing to drop, as before


def test_no_sharing_cases_keep_todays_packing():
    from rlaifv_b200.model import PREFIX_MAX_SEQ, pack_rows
    T = 400
    lab, src = _pair_batch(T, [100, 200], [50], lasts=[300, 350])
    ref = pack_rows(lab)
    for got in (pack_rows(lab, src), pack_rows(lab[:1], src[:1])):   # every pos0 is 0; an odd batch
        assert not got.shared and got.pos0 is None
    got = pack_rows(lab, src)
    assert got.cu.tolist() == ref.cu.tolist() and torch.equal(got.rows, ref.rows) and torch.equal(got.pos, ref.pos)
    n = PREFIX_MAX_SEQ + 2                                 # more sequences than one attention launch takes
    lab, src = _pair_batch(T, [300] * n, [None] * (n // 2), lasts=[350] * n)
    got = pack_rows(lab, src)
    assert not got.shared and got.M == n * 351


class _Recorder:
    def __init__(self, monkeypatch):
        from rlaifv_b200 import lib, ops
        self.calls, self.argv = [], {}

        def fake_call(name, *args):
            assert len(args) == len(lib._SIGNATURES[name]), name
            self.calls.append(name)
            self.argv.setdefault(name, []).append(args)
        monkeypatch.setattr(lib, "call", fake_call)
        monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
        monkeypatch.setattr(lib, "load",
                            lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
        monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)


@pytest.mark.parametrize("share,dropout", [(False, 0.0), (True, 0.0), (True, 0.05)])
def test_launch_sequence_dry_run(monkeypatch, share, dropout):
    """share_prefix on (LoRA dropout 0): the decoder's attention goes through the prefix entry points with the shared
    row count; off, or with dropout, the sequence is today's packed one."""
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    from rlaifv_b200 import ops
    rec = _Recorder(monkeypatch)
    c = O.TINY
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    T = 300
    # first supervised rows 200 / 149 (chosen), 210 / 159 (rejected): both pairs share 128 rows (equal sources)
    lab, _ = _pair_batch(T, [200, 149, 210, 159], [None, None], lasts=[250, 200, 299, 170])
    slots = [200, 149, 210, 159]
    monkeypatch.setattr(ops, "supervised_rows", lambda labels, cap: torch.tensor(
        sum(([s * T + t] + [-1] * (cap - 1) for s, t in enumerate(slots)), []), dtype=torch.int32))
    pol = LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))
    assert not pol.share_prefix                  # off by default
    pol.pack_rows, pol.share_prefix = True, share
    pol.enable_lora(r=8, alpha=2.0, dropout=dropout)
    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    monkeypatch.setattr(pol, "splice", lambda ids, lab_, rows, nb, idx, T_hint=None: (
        torch.zeros(4 * T, dims.hidden_size, dtype=torch.bfloat16), lab, torch.zeros(4, T, dtype=torch.int32), T))
    pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    pk = pol._stash["pack"]
    shared = share and dropout == 0.0
    M = 251 + 201 + 172 + 43 if shared else 251 + 201 + 300 + 171
    assert pk.M == M and pk.shared == shared
    # the compact head reads the rejected sequences' supervised rows from their own packed rows
    cap = batch["concatenated_input_ids"].shape[1]
    assert pol._stash["x_rows"][[0, cap, 2 * cap, 3 * cap]].tolist() == (
        [200, 251 + 149, 452 + 210 - 128, 624 + 159 - 128] if shared else [200, 251 + 149, 452 + 210, 752 + 159])
    pol.backward_logps(torch.zeros(4))
    n = dims.num_layers
    fwd, bwd = ("rlaifv_attention_varlen_prefix_fwd", "rlaifv_attention_varlen_prefix_bwd")
    old = ("rlaifv_attention_varlen_fwd", "rlaifv_attention_varlen_bwd")
    used, unused = ((fwd, bwd), old) if shared else (old, (fwd, bwd))
    assert rec.calls.count(used[0]) == rec.calls.count(used[1]) == n
    assert not any(name in rec.calls for name in unused)
    assert all(a[12 if shared else 10] == M for a in rec.argv[used[0]])      # n_rows
    assert rec.calls.count("rlaifv_rope_pos_fwd") == rec.calls.count("rlaifv_rope_pos_bwd") == n


def test_share_prompt_prefix_flag_defaults_off():
    from rlaifv_b200.train_llava15 import parse_args_into_dataclasses
    assert parse_args_into_dataclasses([])[2].share_prompt_prefix is False
    assert parse_args_into_dataclasses(["--share_prompt_prefix", "True"])[2].share_prompt_prefix is True
