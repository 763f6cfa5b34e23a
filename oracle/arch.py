"""Architecture walk of the NCSN++ score network (oracle side).

Restates, as a flat list of layer records, the module list the reference builds
in ``NCSNpp.__init__`` (sgmse/backbones/ncsnpp.py:50-253) and
``NCSNpp_48k.__init__`` (ncsnpp_48k.py:52-256).  Only the configurations the
two registered backbones can reach with ``resblock_type='biggan'``,
``fir=True``, ``progressive in {'output_skip','none'}`` and
``progressive_input in {'input_skip','none'}`` are covered (SURVEY.md §8a).

TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

from dataclasses import dataclass, field, asdict
from typing import List, Tuple


@dataclass
class NetConfig:
    backbone: str = "ncsnpp"            # 'ncsnpp' | 'ncsnpp_48k' | 'ncsnpp_v2'
    nf: int = 128
    ch_mult: Tuple[int, ...] = (1, 1, 2, 2, 2, 2, 2)
    num_res_blocks: int = 2
    attn_resolutions: Tuple[int, ...] = (16,)
    image_size: int = 256
    progressive: str = "output_skip"    # 'output_skip' | 'none'
    progressive_input: str = "input_skip"  # 'input_skip' | 'none'
    fourier_scale: float = 16.0
    scale_by_sigma: bool = True
    init_scale: float = 1.0             # SURVEY.md §0: 0. gives a constant-output net

    @staticmethod
    def ncsnpp(**kw) -> "NetConfig":
        return NetConfig(backbone="ncsnpp", **kw)

    @staticmethod
    def ncsnpp_48k(**kw) -> "NetConfig":
        base = dict(backbone="ncsnpp_48k", attn_resolutions=(), progressive="none",
                    progressive_input="none")
        base.update(kw)
        return NetConfig(**base)

    @staticmethod
    def ncsnpp_v2(**kw) -> "NetConfig":
        """ncsnpp_v2.py:36-395: the same module list as 'ncsnpp' (identical state_dict layout), called as
        ``dnn(x, y, t)`` and without the in-network ``/t`` (scaling lives in ScoreModel.forward, model.py:283-304)."""
        base = dict(backbone="ncsnpp_v2", scale_by_sigma=False)
        base.update(kw)
        return NetConfig(**base)

    def to_dict(self):
        d = asdict(self)
        d["ch_mult"] = list(self.ch_mult)
        d["attn_resolutions"] = list(self.attn_resolutions)
        return d


@dataclass
class Layer:
    idx: int            # index into all_modules (-1: output_layer)
    kind: str           # gfp | linear | conv3 | conv1 | resblock | attn | combine | gn
    cin: int = 0
    cout: int = 0
    up: bool = False
    down: bool = False
    params: List[Tuple[str, Tuple[int, ...]]] = field(default_factory=list)


def gn_groups(c: int) -> int:
    # nn.GroupNorm(num_groups=min(C // 4, 32), eps=1e-6)   layerspp.py:219,231,67
    return min(c // 4, 32)


def _resblock(idx, cin, cout, up=False, down=False) -> Layer:
    p = [("GroupNorm_0.weight", (cin,)), ("GroupNorm_0.bias", (cin,)),
         ("Conv_0.weight", (cout, cin, 3, 3)), ("Conv_0.bias", (cout,)),
         ("Dense_0.weight", (cout, None)), ("Dense_0.bias", (cout,)),
         ("GroupNorm_1.weight", (cout,)), ("GroupNorm_1.bias", (cout,)),
         ("Conv_1.weight", (cout, cout, 3, 3)), ("Conv_1.bias", (cout,))]
    if cin != cout or up or down:           # layerspp.py:233-234
        p += [("Conv_2.weight", (cout, cin, 1, 1)), ("Conv_2.bias", (cout,))]
    return Layer(idx, "resblock", cin, cout, up, down, p)


def _attn(idx, c) -> Layer:
    p = [("GroupNorm_0.weight", (c,)), ("GroupNorm_0.bias", (c,))]
    for k in range(4):
        p += [(f"NIN_{k}.W", (c, c)), (f"NIN_{k}.b", (c,))]
    return Layer(idx, "attn", c, c, params=p)


def build_layers(cfg: NetConfig) -> List[Layer]:
    """Module list in ``all_modules`` order + the trailing ``output_layer``."""
    nf, L = cfg.nf, len(cfg.ch_mult)
    res = [cfg.image_size // (2 ** i) for i in range(L)]
    temb_dim = 4 * nf
    out: List[Layer] = []

    def add(layer: Layer):
        out.append(layer)

    def n():
        return len(out)

    add(Layer(n(), "gfp", params=[("W", (nf,))]))
    add(Layer(n(), "linear", 2 * nf, temb_dim, params=[("weight", (temb_dim, 2 * nf)), ("bias", (temb_dim,))]))
    add(Layer(n(), "linear", temb_dim, temb_dim, params=[("weight", (temb_dim, temb_dim)), ("bias", (temb_dim,))]))
    add(Layer(n(), "conv3", 4, nf, params=[("weight", (nf, 4, 3, 3)), ("bias", (nf,))]))

    hs_c = [nf]
    in_ch = nf
    for lvl in range(L):
        for _ in range(cfg.num_res_blocks):
            out_ch = nf * cfg.ch_mult[lvl]
            add(_resblock(n(), in_ch, out_ch))
            in_ch = out_ch
            if res[lvl] in cfg.attn_resolutions:
                add(_attn(n(), in_ch))
            hs_c.append(in_ch)
        if lvl != L - 1:
            add(_resblock(n(), in_ch, in_ch, down=True))
            if cfg.progressive_input == "input_skip":
                add(Layer(n(), "combine", 4, in_ch,
                          params=[("Conv_0.weight", (in_ch, 4, 1, 1)), ("Conv_0.bias", (in_ch,))]))
            hs_c.append(in_ch)

    in_ch = hs_c[-1]
    add(_resblock(n(), in_ch, in_ch))
    add(_attn(n(), in_ch))
    add(_resblock(n(), in_ch, in_ch))

    for lvl in reversed(range(L)):
        for _ in range(cfg.num_res_blocks + 1):
            out_ch = nf * cfg.ch_mult[lvl]
            add(_resblock(n(), in_ch + hs_c.pop(), out_ch))
            in_ch = out_ch
        if res[lvl] in cfg.attn_resolutions:
            add(_attn(n(), in_ch))
        if cfg.progressive == "output_skip":
            add(Layer(n(), "gn", in_ch, in_ch, params=[("weight", (in_ch,)), ("bias", (in_ch,))]))
            add(Layer(n(), "conv3", in_ch, 4, params=[("weight", (4, in_ch, 3, 3)), ("bias", (4,))]))
        if lvl != 0:
            add(_resblock(n(), in_ch, in_ch, up=True))
    assert not hs_c
    if cfg.progressive != "output_skip":
        add(Layer(n(), "gn", in_ch, in_ch, params=[("weight", (in_ch,)), ("bias", (in_ch,))]))
        add(Layer(n(), "conv3", in_ch, 4, params=[("weight", (4, in_ch, 3, 3)), ("bias", (4,))]))
    # fill the Dense_0 fan-in
    for l in out:
        l.params = [(k, tuple(temb_dim if d is None else d for d in s)) for k, s in l.params]
    out.append(Layer(-1, "conv1", 4, 2, params=[("weight", (2, 4, 1, 1)), ("bias", (2,))]))
    return out


def state_dict_manifest(cfg: NetConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) in the order of ``NCSNpp(...).state_dict()``: ``output_layer`` first
    (it is assigned before ``all_modules``, ncsnpp.py:104,253), then ``all_modules.{i}.*``."""
    layers = build_layers(cfg)
    man = [(f"output_layer.{k}", s) for k, s in layers[-1].params]
    for l in layers[:-1]:
        man += [(f"all_modules.{l.idx}.{k}", s) for k, s in l.params]
    return man
