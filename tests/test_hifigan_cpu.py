"""HiFi-GAN without a GPU: the module tree of models.py (keys, shapes, order, counts), its seeded initialisation, the
fp64 oracle against the same tree run through torch.nn, and every host refusal."""
import warnings

import pytest
import torch

from tests import hifigan_oracle as HO
from tests.common import tensor_digest
from tests.hifigan_common import mel_input, synth_state_dict

import tacotron2_b200 as t2
from tacotron2_b200.hifigan import CONFIGS, Generator, ResBlock1, check_config, get_padding


def expected_keys(h):
    """state_dict keys and shapes of models.py's Generator, restated from the architecture."""
    conv = lambda p, co, ci, k: [(p + ".bias", (co,)), (p + ".weight_g", (co, 1, 1)), (p + ".weight_v", (co, ci, k))]
    c0 = h["upsample_initial_channel"]
    out = conv("conv_pre", c0, 80, 7)
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        ci, co = c0 // 2 ** i, c0 // 2 ** (i + 1)
        out += [("ups.%d.bias" % i, (co,)), ("ups.%d.weight_g" % i, (ci, 1, 1)), ("ups.%d.weight_v" % i, (ci, co, k))]
    n = 0
    for i in range(len(h["upsample_rates"])):
        ch = c0 // 2 ** (i + 1)
        for k, ds in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
            names = (["convs1.%d" % m for m in range(3)] + ["convs2.%d" % m for m in range(3)]
                     if h["resblock"] == "1" else ["convs.%d" % m for m in range(2)])
            for c in names:
                out += conv("resblocks.%d.%s" % (n, c), ch, ch, k)
            n += 1
    return out + conv("conv_post", 1, ch, 7)


@pytest.mark.parametrize("name,count", [("v1", 234), ("v2", 234), ("v3", 69)])
def test_state_dict_keys_shapes_order_and_counts(name, count):
    G = Generator(CONFIGS[name])
    sd = G.state_dict()
    assert len(sd) == count
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == expected_keys(CONFIGS[name])
    assert len(G._weight_table()) == count
    c0 = CONFIGS[name]["upsample_initial_channel"]
    assert tuple(sd["ups.0.weight_g"].shape) == (c0, 1, 1)     # dim 0 of a ConvTranspose1d: the input channel


def test_v1_parameter_count_includes_weight_g():
    G = Generator(CONFIGS["v1"])
    assert sum(p.numel() for p in G.parameters()) == 13936130


def test_hifigan_is_exported_and_takes_an_attribute_config():
    assert t2.HiFiGAN is Generator

    class H:
        pass
    h = H()
    for k, v in CONFIGS["v3"].items():
        setattr(h, k, v)
    assert list(Generator(h).state_dict()) == list(Generator(CONFIGS["v3"]).state_dict())


def _replay(h):
    """models.py's construction, step by step, with torch.nn: the draws a seeded Generator must make, in order."""
    def wn(c):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", FutureWarning)
            return torch.nn.utils.weight_norm(c)

    def init(c):
        c.weight.data.normal_(0.0, 0.01)
    c0 = h["upsample_initial_channel"]
    convs = {"conv_pre": wn(torch.nn.Conv1d(80, c0, 7, 1, padding=3))}
    ups = []
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        ups.append(wn(torch.nn.ConvTranspose1d(c0 // 2 ** i, c0 // 2 ** (i + 1), k, u, padding=(k - u) // 2)))
        convs["ups.%d" % i] = ups[-1]
    n = 0
    for i in range(len(ups)):
        ch = c0 // 2 ** (i + 1)
        for k, ds in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
            if h["resblock"] == "1":
                for m, d in enumerate(ds):
                    convs["resblocks.%d.convs1.%d" % (n, m)] = wn(torch.nn.Conv1d(ch, ch, k, 1, dilation=d, padding=get_padding(k, d)))
                for m in range(3):
                    init(convs["resblocks.%d.convs1.%d" % (n, m)])
                for m in range(3):
                    convs["resblocks.%d.convs2.%d" % (n, m)] = wn(torch.nn.Conv1d(ch, ch, k, 1, dilation=1, padding=get_padding(k, 1)))
                for m in range(3):
                    init(convs["resblocks.%d.convs2.%d" % (n, m)])
            else:
                for m, d in enumerate(ds):
                    convs["resblocks.%d.convs.%d" % (n, m)] = wn(torch.nn.Conv1d(ch, ch, k, 1, dilation=d, padding=get_padding(k, d)))
                for m in range(2):
                    init(convs["resblocks.%d.convs.%d" % (n, m)])
            n += 1
    convs["conv_post"] = wn(torch.nn.Conv1d(ch, 1, 7, 1, padding=3))
    for c in ups:
        init(c)
    init(convs["conv_post"])
    return {p + "." + n: t for p, c in convs.items() for n, t in c.state_dict().items()}


@pytest.mark.parametrize("name", ["v1", "v2", "v3"])
def test_seeded_initialisation_matches_the_models_py_construction(name):
    torch.manual_seed(1234)
    sd = Generator(CONFIGS[name]).state_dict()
    torch.manual_seed(1234)
    ref = _replay(CONFIGS[name])
    assert list(sd) == list(ref)
    assert [tensor_digest(v) for v in sd.values()] == [tensor_digest(v) for v in ref.values()]


def _nn_forward(G, x):
    """models.py's Generator.forward on the module tree (fp64), through torch.nn's own conv modules and hooks."""
    lrelu = torch.nn.functional.leaky_relu
    x = G.conv_pre(x)
    for i in range(G.num_upsamples):
        x = G.ups[i](lrelu(x, 0.1))
        xs = None
        for j in range(G.num_kernels):
            rb = G.resblocks[i * G.num_kernels + j]
            y = x
            if isinstance(rb, ResBlock1):
                for c1, c2 in zip(rb.convs1, rb.convs2):
                    y = c2(lrelu(c1(lrelu(y, 0.1)), 0.1)) + y
            else:
                for c in rb.convs:
                    y = c(lrelu(y, 0.1)) + y
            xs = y if xs is None else xs + y
        x = xs / G.num_kernels
    return torch.tanh(G.conv_post(lrelu(x)))


@pytest.mark.parametrize("name", ["v1", "v2", "v3"])
def test_oracle_matches_the_torch_nn_tree_in_fp64_before_and_after_remove_weight_norm(name):
    G = Generator(CONFIGS[name])
    G.load_state_dict(synth_state_dict(G, 5))
    G = G.double()
    x = mel_input(2, 6, 1).double()
    with torch.no_grad():
        ref = _nn_forward(G, x)
        out = HO.forward(G.state_dict(), CONFIGS[name], x)
        assert tuple(ref.shape) == (2, 1, 256 * 6) == tuple(out.shape)
        assert (out - ref).abs().max().item() < 1e-12
        assert ref.std().item() > 0.05                       # the synthetic weights keep the signal alive
        G.remove_weight_norm()
        assert not any(k.endswith("weight_g") for k in G.state_dict())
        ref2 = _nn_forward(G, x)
        out2 = HO.forward(G.state_dict(), CONFIGS[name], x)
        assert (out2 - ref2).abs().max().item() < 1e-12
        assert (ref2 - ref).abs().max().item() < 1e-12


def test_remove_weight_norm_keeps_one_table_entry_per_slot():
    G = Generator(CONFIGS["v3"])
    G.remove_weight_norm()
    t = G._weight_table()
    assert len(t) == 69 and all(t[i] is None for i in range(1, 69, 3))
    assert all(t[i] is not None for i in range(69) if i % 3 != 1)


def _cfg(**kw):
    h = {k: (list(v) if isinstance(v, list) else v) for k, v in CONFIGS["v1"].items()}
    h.update(kw)
    return h


@pytest.mark.parametrize("kw,match", [
    (dict(upsample_rates=[8, 8, 2, 4], upsample_kernel_sizes=[16, 16, 4, 8]), "product of upsample_rates"),
    (dict(upsample_kernel_sizes=[16, 16, 4, 5]), "upsample_kernel_sizes"),
    (dict(upsample_rates=[8, 8, 4, 1], upsample_kernel_sizes=[16, 16, 8, 2]), "upsample_rates must be even"),
    (dict(upsample_initial_channel=1024), "upsample_initial_channel"),
    (dict(upsample_initial_channel=64), "upsample_initial_channel"),
    (dict(upsample_initial_channel=200), "upsample_initial_channel"),
    (dict(resblock_kernel_sizes=[3, 7, 12]), "resblock_kernel_sizes"),
    (dict(resblock_kernel_sizes=[3, 7, 17]), "resblock_kernel_sizes"),
    (dict(resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 13]]), "resblock_dilation_sizes"),
    (dict(resblock_dilation_sizes=[[1, 3], [1, 3], [1, 3]]), "resblock_dilation_sizes"),
    (dict(resblock="3"), "resblock"),
])
def test_host_refuses_unsupported_configurations_naming_the_field(kw, match):
    with pytest.raises(ValueError, match=match):
        check_config(_cfg(**kw))


def test_published_configurations_pass_the_host_checks():
    for h in CONFIGS.values():
        check_config(h)


def test_forward_refuses_before_any_launch():
    G = Generator(CONFIGS["v3"]).eval()
    with torch.no_grad():
        with pytest.raises(ValueError, match="x must be"):
            G(torch.zeros(2, 79, 5))
        with pytest.raises(ValueError, match="x must be"):
            G(torch.zeros(80, 5))
        with pytest.raises(TypeError, match="float32 or float16"):
            G(torch.zeros(1, 80, 5, dtype=torch.float64))
        with pytest.raises(ValueError, match="lengths must lie"):
            G(torch.zeros(2, 80, 5), lengths=[5, 6])
        with pytest.raises(ValueError, match="lengths must lie"):
            G(torch.zeros(2, 80, 5), lengths=[0, 5])
        with pytest.raises(ValueError, match="lengths must have shape"):
            G(torch.zeros(2, 80, 5), lengths=[5])
        with pytest.raises(TypeError):
            G(torch.zeros(2, 80, 5), lengths=[5.0, 4.0])
        with pytest.raises(ValueError, match="too large"):
            G(torch.zeros(64, 80, 70000).expand(64, 80, 70000))
        with pytest.raises(RuntimeError, match="CUDA device"):
            G(torch.zeros(2, 80, 5))
    bad = Generator(_cfg(resblock_kernel_sizes=[3, 7, 12]))
    with torch.no_grad(), pytest.raises(ValueError, match="resblock_kernel_sizes"):
        bad(torch.zeros(1, 80, 5))


def test_forward_under_autograd_raises():
    G = Generator(CONFIGS["v3"])
    with pytest.raises(NotImplementedError, match="no backward"):
        G(torch.zeros(1, 80, 5))
