"""The training convolutions' form choice, host side: RNC_TRAIN_CONV's accepted values, which layers the TF32 tensor-core form
takes, and its weight pack (UmmaWeights(tf32=True)) against the TF32 hi/lo planes it has always been, bit for bit."""
import types

import pytest
import torch

from test_product_shapes import CFG5_CONV_SIGNATURES
from test_wnet_variants import CONFIGS


def ceil4(c):
    return (c + 3) // 4 * 4


def wnet_layers():
    """(cin, cout, k, Cx) of every weights-net configuration's layers: the input is staged at 136 channels (130 used)."""
    out = []
    for num_ch, filter_sz, _, _ in CONFIGS.values():
        ch = [130] + num_ch + [2]
        out += [(ch[i], ch[i + 1], filter_sz[i], 136 if i == 0 else ceil4(ch[i])) for i in range(len(ch) - 1)]
    return sorted(set(out))


def layer_forms():
    """(cin, cout, kh, kw, Cx) of the forward and (cout, cin, kh, kw, ceil4(cout)) of the data-gradient convolution of every
    config-5 training layer and weights-net layer.  Cx is the channel-last pitch the layer sees; the weights net's first layer
    reads the 136-channel staging."""
    fwd = [(cin, cout, kh, kw, 136 if cin == 130 else ceil4(cin)) for cin, cout, kh, kw, *_ in CFG5_CONV_SIGNATURES]
    fwd += [(cin, cout, k, k, cx) for cin, cout, k, cx in wnet_layers()]
    dgrad = [(cout, cin, kh, kw, ceil4(cout)) for cin, cout, kh, kw, _ in fwd]
    return sorted(set(fwd)), sorted(set(dgrad))


FWD, DGRAD = layer_forms()


def tf32_planes_reference(w, cin_pad):
    """The TF32 pack as it has always been: [CoutPad][taps * ceil32(cin_pad)] fp32 planes, tap-major, hi = w rounded at bit 13
    with ties away from zero (through the int32 view), lo = w - hi, zero bias, unscale 1."""
    cout, cin, kh, kw = w.shape
    coutpad = next((c for c in (32, 64, 128, 192, 256) if cout <= c), (cout + 191) // 192 * 192)
    nblk = (cin_pad + 31) // 32
    ktot = kh * kw * nblk * 32
    wp = torch.zeros(coutpad, kh * kw, nblk * 32, dtype=torch.float32)
    wp[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, kh * kw, cin)
    ws = wp.reshape(coutpad, ktot)
    hi = ((ws.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32).contiguous()
    return dict(w_hi=hi, w_lo=(ws - hi).contiguous(), bias=torch.zeros(coutpad), coutpad=coutpad, ktot=ktot, unscale=1.0,
                cout=cout, kh=kh, kw=kw)


@pytest.mark.parametrize("kind", ["fwd", "dgrad"])
def test_tf32_pack_is_bit_identical(kind):
    """At every layer shape, the forward weight and the flipped, transposed data-gradient weight (as rnc.train._packed forms
    them) pack to the same bits; the shapes reach every output padding and input pitches that are not multiples of 32."""
    from rnc.engine_umma import UmmaWeights
    g = torch.Generator().manual_seed(7)
    pads = set()
    for cin, cout, kh, kw, cx in (FWD if kind == "fwd" else DGRAD):
        shape = (cout, cin, kh, kw) if kind == "fwd" else (cin, cout, kh, kw)       # the layer weight
        w = torch.randn(shape, generator=g) * 10.0 ** torch.randint(-6, 3, shape[:2] + (1, 1), generator=g)
        w.view(-1)[:4] = torch.tensor([0.0, -0.0, 1 + 2 ** -11, -(1 + 2 ** -11)])        # zeros and TF32 ties
        if kind == "dgrad":
            w = w.flip(2, 3).transpose(0, 1).contiguous()
        ref = tf32_planes_reference(w, cx)
        got = UmmaWeights(w, None, [cx], tf32=True)
        for name, v in ref.items():
            g_v = getattr(got, name)
            if isinstance(v, torch.Tensor):
                assert g_v.dtype == torch.float32 and g_v.shape == v.shape, (name, cin, cout, kh, kw, cx)
                assert torch.equal(g_v.view(torch.int32), v.view(torch.int32)), (name, cin, cout, kh, kw, cx)
            else:
                assert g_v == v and type(g_v) is type(v), (name, cin, cout, kh, kw, cx)
        pads.add(ref["coutpad"])
    assert pads >= {32, 64, 128, 192, 256}
    assert any(s[4] % 32 for s in (FWD if kind == "fwd" else DGRAD))


def test_conv_mode_accepts_ffma_and_tf32_only(monkeypatch):
    from rnc.train import _conv_mode
    monkeypatch.delenv("RNC_TRAIN_CONV", raising=False)
    assert _conv_mode() == "ffma"
    for mode in ("ffma", "tf32"):
        monkeypatch.setenv("RNC_TRAIN_CONV", mode)
        assert _conv_mode() == mode
    for bad in ("umma", "foo", "TF32", ""):
        monkeypatch.setenv("RNC_TRAIN_CONV", bad)
        with pytest.raises(ValueError, match="RNC_TRAIN_CONV.*expected 'ffma' or 'tf32'"):
            _conv_mode()


def tf32_decision_reference(eng_mode, mode, Cx, cout):
    """The TF32 form's rule as it has always been: the tensor-core engine, RNC_TRAIN_CONV=tf32, an fp32 output row whose
    32-channel chunks fit the channel-last pitch, and an operand pitch of 4 floats."""
    if eng_mode != "umma" or mode == "ffma" or (cout + 31) // 32 * 32 != (cout + 3) // 4 * 4:
        return False
    return Cx % 4 == 0


@pytest.mark.parametrize("mode", ["ffma", "tf32"])
@pytest.mark.parametrize("eng_mode", ["umma", "ffma"])
def test_tf32_form_rule(monkeypatch, eng_mode, mode):
    """The forward and the data gradient take the TF32 form on the same rule; the exact engine never takes it.  Raw channel
    counts (pitch not a multiple of 4) stand in for operands the form must refuse."""
    from rnc.train import _tf32_ok
    monkeypatch.setenv("RNC_TRAIN_CONV", mode)
    eng = types.SimpleNamespace(mode=eng_mode)
    picked = 0
    for cin, cout, _, _, cx in FWD + DGRAD:
        for Cx in (cx, cin):
            want = tf32_decision_reference(eng_mode, mode, Cx, cout)
            assert _tf32_ok(eng, Cx, cout) is want, (eng_mode, mode, Cx, cout)
            picked += want
    assert (picked > 0) == (eng_mode == "umma" and mode == "tf32")
