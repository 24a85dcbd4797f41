"""seeddot_nll (SEED-Encoder) without a GPU: the config class, the model's parameter surface and checkpoint loading, the
refusals, the registry, and the oracle against the reference's golden embeddings, losses and gradients
(tests/golden/encoder_seed.npz, tests/golden/seed_grads.npz from oracle/make_golden_seed.py)."""
import argparse
import os

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import MSMarcoConfigDict, SEEDEncoderConfig, SEEDEncoderDot_NLL_LN_B200
from ance_b200.synthetic import random_seed_state_dict, write_seed_checkpoint
from oracle.seed_oracle import SEEDDotOracle, grad_sketch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
P = "seed_encoder.encoder.sentence_encoder."


def _small(**over):
    kw = dict(encoder_layers=2, vocab_size=1000)
    kw.update(over)
    return SEEDEncoderConfig(**kw)


def test_config_defaults_and_round_trip(tmp_path):
    c = SEEDEncoderConfig()
    assert c.model_type == "seed_encoder"
    assert (c.pad_token_id, c.vocab_size, c.encoder_layers, c.encoder_embed_dim, c.encoder_ffn_embed_dim,
            c.encoder_attention_heads) == (1, 32769, 12, 768, 3072, 12)
    assert (c.dropout, c.attention_dropout, c.activation_dropout, c.encoder_layerdrop) == (0.1, 0.1, 0.0, 0.0)
    assert (c.max_positions, c.activation_fn, c.quant_noise_pq, c.encoder_layers_to_keep) == (512, "gelu", 0.0, None)
    assert c.max_source_positions == c.max_target_positions == 512 and c.decoder_output_dim == 768
    assert c.num_labels == 2
    c2 = SEEDEncoderConfig(encoder_layers=3, dropout=0.2, vocab_size=500, activation_dropout=0.05)
    c2.save_pretrained(str(tmp_path))
    back = SEEDEncoderConfig.from_pretrained(str(tmp_path))
    a, b = c2.to_dict(), back.to_dict()
    a.pop("transformers_version", None)
    b.pop("transformers_version", None)
    assert a == b
    assert (back.encoder_layers, back.dropout, back.vocab_size, back.activation_dropout) == (3, 0.2, 500, 0.05)
    # the refresher reads the config through the registry's class
    assert MSMarcoConfigDict["seeddot_nll"].config_class is SEEDEncoderConfig
    got = MSMarcoConfigDict["seeddot_nll"].config_class.from_pretrained(str(tmp_path), num_labels=2,
                                                                        finetuning_task="MSMarco")
    assert got.encoder_layers == 3 and got.pad_token_id == 1


def test_parameter_names_and_order_are_the_reference():
    g = np.load(os.path.join(GOLD, "encoder_seed.npz"))
    names = [str(x) for x in g["param_names"]]
    m = SEEDEncoderDot_NLL_LN_B200(SEEDEncoderConfig())
    assert [n for n, _ in m.named_parameters()] == names
    assert list(m.state_dict()) == names          # the zero type row is not persistent
    sd = random_seed_state_dict(seed=0, n_layer=12)
    assert list(sd) == names
    assert all(tuple(sd[n].shape) == tuple(p.shape) for n, p in m.named_parameters())
    assert tuple(m.get_buffer(P + "type_row").shape) == (1, 768)
    assert not bool(m.get_buffer(P + "type_row").any())


def test_kernel_weight_layout():
    """The weights handed to ance_encoder_weights: q/k/v in the kernels' order whatever the registration order."""
    from ance_b200.models import _param_groups
    m = SEEDEncoderDot_NLL_LN_B200(_small())
    se = m.seed_encoder.encoder.sentence_encoder
    embs, layers, hd = _param_groups(se, (m.embeddingHead, m.norm))
    assert embs[0] is se.embed_tokens.weight and embs[1] is se.embed_positions.weight and embs[2] is se.type_row
    assert embs[3] is se.emb_layer_norm.weight and embs[4] is se.emb_layer_norm.bias
    l0 = se.layers[0]
    assert layers[0][0] is l0.self_attn.q_proj.weight and layers[0][2] is l0.self_attn.k_proj.weight
    assert layers[0][4] is l0.self_attn.v_proj.weight and layers[0][6] is l0.self_attn.out_proj.weight
    assert layers[0][8] is l0.self_attn_layer_norm.weight and layers[0][10] is l0.fc1.weight
    assert layers[0][12] is l0.fc2.weight and layers[0][14] is l0.final_layer_norm.weight
    assert len(layers) == 2 and all(len(x) == 16 for x in layers)
    assert hd == [m.embeddingHead.weight, m.embeddingHead.bias, m.norm.weight, m.norm.bias]
    assert se.embed_positions.weight.shape[0] == 512 + 1 + 1   # max_positions + pad + 1 (learned, offset by pad)
    assert se.embed_tokens.padding_idx == 1 and se.embed_positions.padding_idx == 1


def test_from_pretrained_policy(tmp_path):
    write_seed_checkpoint(str(tmp_path / "ck"), seed=3, n_layer=2, vocab=1000)
    m = SEEDEncoderDot_NLL_LN_B200.from_pretrained(str(tmp_path / "ck"))
    assert isinstance(m.config, SEEDEncoderConfig) and m.config.encoder_layers == 2 and not m.training
    sd = random_seed_state_dict(seed=3, n_layer=2, vocab=1000)
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    # a pretraining checkpoint's extra tensors (decoder, lm_head) are ignored
    extra = dict(sd, **{"lm_head.dense.weight": torch.zeros(3, 3), "decoder.layers.0.fc1.weight": torch.zeros(2)})
    torch.save(extra, str(tmp_path / "ck" / "pytorch_model.bin"))
    SEEDEncoderDot_NLL_LN_B200.from_pretrained(str(tmp_path / "ck"))
    # a missing tensor raises
    del extra["classification_heads.out_proj.bias"]
    torch.save(extra, str(tmp_path / "ck" / "pytorch_model.bin"))
    with pytest.raises(KeyError, match="lacks 1 tensors"):
        SEEDEncoderDot_NLL_LN_B200.from_pretrained(str(tmp_path / "ck"))
    # encoder_layers_to_keep sets the depth (modeling_seed_encoder.py:73-74)
    m = SEEDEncoderDot_NLL_LN_B200(_small(encoder_layers=12, encoder_layers_to_keep="0,5,11"))
    assert len(m.seed_encoder.encoder.sentence_encoder.layers) == 3


def test_registry_builds_the_b200_model_without_the_reference(tmp_path):
    import sys
    assert "model.models" not in sys.modules
    cls = MSMarcoConfigDict["seeddot_nll"].model_class
    with pytest.raises(NotImplementedError, match="stock module.*SEEDEncoderConfig"):
        cls()
    m = cls(_small())
    assert type(m) is SEEDEncoderDot_NLL_LN_B200
    assert type(cls(config=_small())) is SEEDEncoderDot_NLL_LN_B200
    write_seed_checkpoint(str(tmp_path / "ck"), seed=0, n_layer=2, vocab=1000)
    m = cls.from_pretrained(str(tmp_path / "ck"), config=None)
    assert type(m) is SEEDEncoderDot_NLL_LN_B200
    with pytest.raises(NotImplementedError, match="stock module"):
        cls.from_pretrained()
    # the refresher's model loading: the registry's config class, then model_class.from_pretrained
    from ance_b200.drivers import run_ann_data_gen as drv
    args = argparse.Namespace(model_type="SEEDDOT_NLL", config_name="", cache_dir="", device=torch.device("cpu"))
    cfg, _, model = drv.load_model(args, str(tmp_path / "ck"))
    assert isinstance(cfg, SEEDEncoderConfig) and type(model) is SEEDEncoderDot_NLL_LN_B200
    be = drv.B200Backend(argparse.Namespace(device=torch.device("cpu")), model)
    assert be.mask_mode == "ids" and be.pad_id == 1


def test_backend_mask_modes():
    from ance_b200.drivers import run_ann_data_gen as drv
    from ance_b200.models import BiEncoder, RobertaDot_NLL_LN
    from ance_b200.synthetic import roberta_base_config
    a = argparse.Namespace(device=torch.device("cpu"))
    rd = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=1, vocab_size=100))
    assert drv.B200Backend(a, rd).mask_mode == "lens"
    assert drv.B200Backend(a, None).mask_mode == "lens"
    dpr = BiEncoder(argparse.Namespace(num_hidden_layers=1, vocab_size=100))
    for mode in (None, "nonzero", "ids"):
        be = drv.B200Backend(a, dpr, mask_mode=mode)
        assert be.mask_mode == "ids" and be.pad_id == 0
    seed = SEEDEncoderDot_NLL_LN_B200(_small(pad_token_id=5))
    assert drv.B200Backend(a, seed).pad_id == 5


def test_refusals():
    with pytest.raises(NotImplementedError, match="activation_fn"):
        SEEDEncoderDot_NLL_LN_B200(_small(activation_fn="gelu_accurate"))
    with pytest.raises(NotImplementedError, match="activation_fn"):
        SEEDEncoderDot_NLL_LN_B200(_small(activation_fn="relu"))
    with pytest.raises(NotImplementedError, match="quant_noise_pq"):
        SEEDEncoderDot_NLL_LN_B200(_small(quant_noise_pq=0.1))
    with pytest.raises(NotImplementedError, match="use_mean"):
        SEEDEncoderDot_NLL_LN_B200(_small(), argparse.Namespace(use_mean=True))
    ids = torch.full((2, 8), 5, dtype=torch.int64)
    for field in ("activation_dropout", "encoder_layerdrop"):
        m = SEEDEncoderDot_NLL_LN_B200(_small(**{field: 0.1})).set_trainable(True)
        m.train()
        with pytest.raises(NotImplementedError, match=field):
            m.query_emb(ids)
        m.eval()   # eval mode: those layers compute the same as without them; the encoder then asks for a GPU
        with pytest.raises(_lib.AnceError, match="GPU"):
            m.query_emb(ids)
        m.set_trainable(False).train()
        with pytest.raises(_lib.AnceError, match="GPU"):
            m.query_emb(ids)
    m = SEEDEncoderDot_NLL_LN_B200(_small(dropout=0.2, attention_dropout=0.05))
    assert m.set_trainable(True, max_len=512, dropout=True, packed=True)._dropout == (0.2, 0.05)
    with pytest.raises(_lib.AnceError, match="has no backward"):   # the packed inference entry is not trainable
        m.query_emb_packed(ids)


def test_oracle_matches_the_reference_embeddings():
    g = np.load(os.path.join(GOLD, "encoder_seed.npz"))
    orc = SEEDDotOracle(random_seed_state_dict(seed=int(g["seed"]), n_layer=12), n_layer=12)
    with torch.no_grad():
        for key in ("p", "q", "f"):
            ids = torch.from_numpy(g[key + "ids"])
            d = (orc.body_emb(ids) - torch.from_numpy(g[key + "emb"])).abs().max().item()
            assert d < 2e-4, (key, d)
        # the attention_mask argument is ignored (the mask comes from the ids)
        q = torch.from_numpy(g["qids"])
        assert torch.equal(orc.query_emb(q, torch.zeros_like(q)), orc.query_emb(q))
        loss = orc.nll_loss(torch.from_numpy(g["qids"][:3]), torch.from_numpy(g["pids"][:3]),
                            torch.from_numpy(g["pids"][3:]))
    assert abs(float(loss) - float(g["loss"])) < 1e-4
    # the fixture covers what it claims: full rows, prefix padding, pad ids inside rows, a foreign padding id
    for key in ("p", "q"):
        ids = g[key + "ids"]
        pad = ids == 1
        assert (~pad).all(axis=1).any()
        holed = [b for b in range(len(ids)) if pad[b].any() and not pad[b, np.argmax(pad[b]):].all()]
        assert holed
    assert (g["fids"] == 0).sum() > 4 and not (g["fids"] == 1).any()


def test_oracle_matches_the_reference_gradients():
    g = np.load(os.path.join(GOLD, "seed_grads.npz"))
    orc = SEEDDotOracle(random_seed_state_dict(seed=int(g["seed"]), n_layer=2, vocab=1000), n_layer=2)
    leaves = orc.leaves()
    loss = orc.nll_loss(*(torch.from_numpy(g[k]) for k in ("q_ids", "a_ids", "b_ids")))
    loss.backward()
    assert abs(float(loss.detach()) - float(g["loss"])) < 1e-4
    names = [str(x) for x in g["names"]]
    assert set(names) == {k for k in leaves}   # every parameter except the unused classification_heads
    sk = dict(zip(names, torch.from_numpy(g["sketch"])))
    for n in names:
        s = grad_sketch(leaves[n].grad, n)
        scale = sk[n.replace("k_proj", "q_proj")][0]   # the key biases' exact gradient is zero: noise on both sides
        assert float((s - sk[n]).abs().max()) <= 1e-3 * float(scale), n
    assert not g["tok_pad_row"].any() and not g["pos_pad_row"].any()
    assert not leaves[P + "embed_tokens.weight"].grad[1].any()
    assert not leaves[P + "embed_positions.weight"].grad[1].any()
