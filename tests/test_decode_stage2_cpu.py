"""Second stage of the decoder without a GPU: the oracle's attempt order against the reference's own ``output_from`` walk, the
host decoder (``clair3_b200.decode``) against the reference's ``output_from`` results and ``batch_output`` text, and the
launcher's ``--decode_rows`` shard.  Vectors: ``tests/golden/decode_stage2.npz`` (``tests/golden/make_decode_stage2_golden.py``)."""
import os

import numpy as np
import pytest

from clair3_b200 import decode, launcher
from oracle import decode_oracle as dec1
from oracle import decode_stage2_oracle as dec2

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_stage2.npz")
CONFIG_NAMES = ("default", "show_ref", "haploid_precise", "haploid_sensitive", "long_indel", "qual_iupac")


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def make_config(out_dim, name):
    kw = dict(is_show_reference=False, is_debug=False, is_haploid_precise_mode_enabled=False,
              is_haploid_sensitive_mode_enabled=False, is_output_for_ensemble=False, quality_score_for_pass=None, tensor_fn="PIPE",
              input_probabilities=True, add_indel_length=(out_dim == 90), gvcf=False, pileup=(out_dim == 24),
              enable_long_indel=False, maximum_variant_length_that_need_infer=50, keep_iupac_bases=False)
    kw.update({"default": {}, "show_ref": {"is_show_reference": True},
               "haploid_precise": {"is_haploid_precise_mode_enabled": True},
               "haploid_sensitive": {"is_haploid_sensitive_mode_enabled": True},
               "long_indel": {"enable_long_indel": True, "is_show_reference": True,
                              "maximum_variant_length_that_need_infer": 100000},
               "qual_iupac": {"quality_score_for_pass": 12.0, "keep_iupac_bases": True}}[name])
    return decode.OutputConfig(**kw)


class OracleModel:
    """Module-protocol stand-in whose decoder stages are the numpy oracles."""

    def __init__(self, out_dim):
        self.out_dim = out_dim
        self.stage2_calls = []

    def decode_stage1(self, y, ref_gt21):
        return dec1.decode_stage1(y, ref_gt21)

    def decode_stage2(self, y, ref_gt21, sites=None, n_sites=None, k=16):
        self.stage2_calls.append(k)
        return dec2.decode_stage2(y, ref_gt21, sites, n_sites, k)


def ref_gt21_of(pos_strings):
    out = []
    for p in pos_strings:
        seq = str(p).split(":")[-1]
        out.append(decode.GT21_OF_BASE[decode.BASE2ACGT[seq[16 if len(seq) > 1 else 0]]])
    return np.array(out, dtype=np.uint8)


@pytest.mark.parametrize("out_dim", [24, 90])
def test_oracle_attempt_order_is_the_reference_walk(z, out_dim):
    y, gt = z["seq_y%d" % out_dim], z["seq_gt%d" % out_dim]
    rows = z["seq_row%d" % out_dim]
    got = dec2.decode_stage2(y, gt, k=1024)
    assert got["complete"].all()
    assert np.array_equal(got["count"], np.bincount(rows, minlength=len(y)))
    valid = np.arange(1024)[None, :] < got["count"][:, None]
    assert np.array_equal(got["cat"][valid], z["seq_cat%d" % out_dim])
    assert np.array_equal(got["idx"][valid], z["seq_idx%d" % out_dim])
    assert np.array_equal(got["prob"][valid].view(np.uint32), z["seq_prob%d" % out_dim].view(np.uint32))
    # the reference exposes the tie flags of its failed (non-reference) attempts
    nonref = z["seq_cat%d" % out_dim] != 0
    assert np.array_equal(got["tie_mask"][valid][nonref], z["seq_mask%d" % out_dim][nonref])
    assert (got["tie_mask"][valid][~nonref] & 1).all()
    # the fixture exercises ties across categories and a homo_Ref ranked late
    assert (np.bitwise_count(z["seq_mask%d" % out_dim][nonref]) > 1).any()
    assert got["count"].max() == (804 if out_dim == 90 else 24)


@pytest.mark.parametrize("k", [1, 16, 1024])
def test_oracle_prefix_is_consistent_across_k(z, k):
    y, gt = z["seq_y90"], z["seq_gt90"]
    full = dec2.decode_stage2(y, gt, k=1024)
    part = dec2.decode_stage2(y, gt, k=k)
    kk = min(k, 1024)
    assert np.array_equal(part["count"], np.minimum(full["count"], kk))
    assert np.array_equal(part["complete"], (full["count"] <= kk).astype(np.uint8))
    for name in ("cat", "idx", "prob", "tie_mask"):
        assert np.array_equal(part[name], full[name][:, :kk])


@pytest.mark.parametrize("out_dim,tag", [(24, ""), (24, "_long"), (90, ""), (90, "_long")])
def test_output_from_ranked_matches_reference(z, out_dim, tag):
    pre = "real%d_" % out_dim
    y, pos, alts = z[pre + "y"], z[pre + "pos"], z[pre + "alt"]
    gt = ref_gt21_of(pos)
    ranked = dec2.decode_stage2(y, gt, k=1024)
    early = dec1.decode_stage1(y, gt)["is_ref"]
    assert 0 < early.sum() < len(y)
    max_len = 100000 if tag else 50
    for i in range(len(y)):
        seq = str(pos[i]).split(":")[-1]
        _, alt = decode.parse_alt_info(str(alts[i]))
        if early[i]:            # output_from's early-out: stage 1 decides it, and its product is the ranked homo_Ref entry
            ref_pos = list(ranked["cat"][i]).index(0)
            base = decode.BASE2ACGT[seq[16]]
            got = decode.REFERENCE_FLAGS, (base, base), ranked["prob"][i][ref_pos]
        else:
            got = decode.output_from_ranked(seq, 16, ranked["cat"][i], ranked["idx"][i], ranked["prob"][i],
                                            ranked["tie_mask"][i], ranked["count"][i], alt, out_dim == 90, max_len)
        flags, (ref, alt_b), p = got
        assert tuple(int(f) for f in flags) == tuple(int(f) for f in z[pre + "of_flags" + tag][i]), i
        assert (ref, alt_b) == (str(z[pre + "of_ref" + tag][i]), str(z[pre + "of_alt" + tag][i])), i
        assert np.float32(p).view(np.uint32) == z[pre + "of_prob" + tag][i].view(np.uint32), i


@pytest.mark.parametrize("name", CONFIG_NAMES)
@pytest.mark.parametrize("out_dim", [24, 90])
@pytest.mark.parametrize("k", [1, 16])
def test_batch_output_text_matches_reference(z, out_dim, name, k):
    pre = "real%d_" % out_dim
    model = OracleModel(out_dim)
    text = decode.batch_output(model, list(z[pre + "pos"]), list(z[pre + "alt"]), z[pre + "y"], make_config(out_dim, name), k=k)
    want = z[pre + "text_" + name].item()
    assert text == want
    assert model.stage2_calls[0] == k and (k > 1 or model.stage2_calls[1:] == [decode.ENTRIES[out_dim]])


def test_batch_output_accepts_memmap_style_rows(z):
    """The replay reader hands batch_output rows of ``S100`` / ``S2000`` arrays (CallVariants.py:1636-1638)."""
    pre = "real24_"
    pos = np.array([[p.encode()] for p in z[pre + "pos"]], dtype="S100")
    alt = np.array([[a.encode()] for a in z[pre + "alt"]], dtype="S2000")
    text = decode.batch_output(OracleModel(24), pos, alt, z[pre + "y"], make_config(24, "default"))
    assert text == z[pre + "text_default"].item()


def test_empty_batch():
    assert decode.batch_output(OracleModel(90), [], [], np.zeros((0, 90), np.float32), make_config(90, "default")) == ""


@pytest.mark.parametrize("field", ["gvcf", "is_debug", "is_output_for_ensemble"])
def test_out_of_scope_configs_raise(z, field):
    cfg = make_config(24, "default")._replace(**{field: True})
    with pytest.raises(NotImplementedError, match=field):
        decode.batch_output(OracleModel(24), list(z["real24_pos"][:3]), list(z["real24_alt"][:3]), z["real24_y"][:3], cfg)


def _shard_inputs(tmp_path, z, out_dim, n_files=3):
    """Tensor files whose stub predictions are the fixture's real rows, split over a few files."""
    pre = "real%d_" % out_dim
    y, pos, alt = z[pre + "y"], list(z[pre + "pos"]), list(z[pre + "alt"])
    cuts = np.array_split(np.arange(len(y)), n_files)
    prefixes = []
    for f, idx in enumerate(cuts):
        prefix = str(tmp_path / ("pileup_chr_%d" % f))
        np.save(prefix, idx.astype(np.int32).reshape(-1, 1))          # the "tensor" carries the row number
        with open(prefix + ".info", "w") as fh:
            for i in idx:
                fh.write("%s\t%s\n" % (pos[i], alt[i]))
        prefixes.append(prefix)
    return prefixes, y, pos, alt


class _RowModel(OracleModel):
    """predict_stream returns the fixture row named by each tensor."""

    def __init__(self, y):
        super().__init__(y.shape[1])
        self.y = y

    def predict_stream(self, batches, streams=8):
        for x in batches:
            yield self.y[np.asarray(x).reshape(-1).astype(np.int64)]


@pytest.mark.parametrize("drop", [False, True])
def test_launcher_decode_rows(tmp_path, z, drop):
    prefixes, y, pos, alt = _shard_inputs(tmp_path, z, 24)
    model = _RowModel(y)
    cfg = decode.replay_config(pileup=True, add_indel_length=False)
    world, rows = 2, []
    for rank in range(world):
        shard = str(tmp_path / ("pred_%d" % rank))
        launcher.run_rank(model, launcher.split_file_list(prefixes, world)[rank], shard, "pileup", drop_ref_calls=drop,
                          decode_rows=cfg)
        rows.append(open(shard + ".vcf_rows").read())
        # the shard the replay would read decodes to the same rows
        pred = np.load(shard + ".prediction")
        spos = np.load(shard + ".position")
        salt = np.load(shard + ".alt_info")
        assert rows[-1] == decode.batch_output(OracleModel(24), spos, salt, pred, cfg)
    want = decode.batch_output(OracleModel(24), pos, alt, y, cfg)
    assert "".join(rows) == want and want.count("\n") > 50
    assert "LowQual" in want or "PASS" in want


def test_launcher_default_writes_no_rows(tmp_path, z):
    prefixes, y, _, _ = _shard_inputs(tmp_path, z, 24, n_files=1)
    launcher.run_rank(_RowModel(y), prefixes, str(tmp_path / "pred_0"), "pileup")
    assert not os.path.exists(str(tmp_path / "pred_0.vcf_rows"))
