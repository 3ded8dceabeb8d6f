"""Shared test helpers: build OUR modules from a golden `spec` and load the reference state_dict."""
import glob
import hashlib
import os

import numpy as np
import torch

import normflows as nf


def build_layer(L):
    t = L["type"]
    if t == "AutoregressiveRationalQuadraticSpline":
        return nf.flows.AutoregressiveRationalQuadraticSpline(
            L["num_input_channels"], L["num_blocks"], L["num_hidden_channels"],
            num_bins=L.get("num_bins", 8), tail_bound=L.get("tail_bound", 3.0))
    if t == "CoupledRationalQuadraticSpline":
        return nf.flows.CoupledRationalQuadraticSpline(
            L["num_input_channels"], L["num_blocks"], L["num_hidden_channels"],
            num_bins=L.get("num_bins", 8), tail_bound=L.get("tail_bound", 3.0),
            reverse_mask=L.get("reverse_mask", False))
    if t == "LULinearPermute":
        return nf.flows.LULinearPermute(L["num_channels"])
    if t == "MaskedAffineFlow":
        return nf.flows.MaskedAffineFlow(torch.tensor([1.0, 0.0]), nf.nets.MLP([2, 4, 2]), nf.nets.MLP([2, 4, 2]))
    if t == "ActNorm":
        return nf.flows.ActNorm(L.get("shape", 2))
    if t == "AffineCouplingBlock":
        return nf.flows.AffineCouplingBlock(nf.nets.MLP(L["mlp"]), scale_map=L.get("scale_map", "exp"),
                                            split_mode=L.get("split_mode", "channel"))
    if t == "Permute":
        return nf.flows.Permute(L["num_channels"], mode=L.get("mode", "shuffle"))
    raise KeyError(t)


def build_model(spec, sd=None):
    flows = [build_layer(L) for L in spec["flows"]]
    d = spec["q0"]["shape"][0]
    trainable = sd is None or "q0.loc" in sd and False
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(d, trainable=False), flows)
    if sd is not None:
        tsd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
        # the reference registers trainable q0 params; ours may be buffers -- same keys either way
        missing, unexpected = model.load_state_dict(tsd, strict=True)
        assert not missing and not unexpected
    return model


def annotate_spec(spec, sd):
    """Fill in constructor details the golden spec leaves implicit (MLP sizes, channel counts)."""
    for i, L in enumerate(spec["flows"]):
        p = f"flows.{i}."
        if L["type"] == "AffineCouplingBlock":
            ks = sorted({int(k[len(p + "flows.1.param_map.net."):].split(".")[0]) for k in sd
                         if k.startswith(p + "flows.1.param_map.net.")})
            sizes = [sd[f"{p}flows.1.param_map.net.{ks[0]}.weight"].shape[1]]
            sizes += [sd[f"{p}flows.1.param_map.net.{k}.weight"].shape[0] for k in ks]
            L["mlp"] = sizes
        if L["type"] == "Permute":
            L["num_channels"] = spec["q0"]["shape"][0]
        if L["type"] == "ActNorm":
            L["shape"] = spec["q0"]["shape"][0]
    return spec


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.max(np.abs(a - b) / (np.abs(b) + 1e-12))


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def check_digests(sd, digests, what):
    """sd must be bit-identical to the arrays the golden was minted from (digests: key -> sha256)."""
    assert set(sd) == set(digests), f"{what}: state_dict keys differ from the golden's"
    bad = [k for k in sd if sha256(sd[k]) != digests[k]]
    assert not bad, f"{what}: rebuilt entries differ from the reference's: {bad[:5]}"


def nsf_model(kind, d, layers, hidden, blocks, seed, sigma, tail_bound=3.0, bins=8, lu_identity=True):
    """tests/golden/make_golden.py nsf() with this package's classes: constructors under torch.manual_seed(seed) (they
    draw from torch's generator exactly like the reference's), then every parameter moved by sigma * randn (seed + 1)."""
    torch.manual_seed(seed)
    flows = []
    for i in range(layers):
        if kind == "ar":
            flows += [nf.flows.AutoregressiveRationalQuadraticSpline(d, blocks, hidden, num_bins=bins, tail_bound=tail_bound)]
        else:
            flows += [nf.flows.CoupledRationalQuadraticSpline(d, blocks, hidden, num_bins=bins, tail_bound=tail_bound,
                                                             reverse_mask=bool(i % 2))]
        flows += [nf.flows.LULinearPermute(d, identity_init=lu_identity)]
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(d, trainable=False), flows)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(sigma * torch.randn(p.shape, generator=g, dtype=p.dtype))
    return model


def state_dict_from_recipe(recipe, digests):
    """The state_dict of a golden stored as a rebuild recipe (make_golden.py dump(recipe=...)), checked bit for bit."""
    r = dict(recipe)
    assert r.pop("builder") == "nsf", recipe
    sd = {k: v.detach().numpy() for k, v in nsf_model(**r).state_dict().items()}
    check_digests(sd, digests, f"nsf recipe {recipe}")
    return sd


def load_npz_parts(path):
    """<stem>.npz and its continuations <stem>.2.npz, ... (make_golden.py save_parts) as one dict."""
    stem = path[:-4]
    out = {}
    for fn in [path] + sorted(glob.glob(stem + ".[0-9].npz")):
        f = np.load(fn, allow_pickle=False)
        out.update({k: f[k] for k in f.files})
    return out
