"""Host-side boundary logic for real checkpoints and configuration files (no torch kernels, no CUDA).

  * `parse_conf` / `Conf`          the subset of HOCON the reference's confs use, with pyhocon's accessors
                                   (reference reconstruction/exp_runner_generic_blender_val.py:44-91 reads the file with
                                   pyhocon, which is not installed here);
  * `latest_checkpoint`            the lexicographically last `checkpoints/ckpt*.pth` (reference :137-149);
  * `recon_states`                 the per-network state dicts of a `ckpt_*.pth` (reference load_checkpoint :435-512:
                                   keys that the network does not have are dropped, a missing entry is reported);
  * `zero123_sampling_state`       the weights `sample_model_batch` actually samples with: the reference wraps sampling in
                                   `model.ema_scope()` (utils/zero123_utils.py:63, ldm/models/diffusion/ddpm.py:180-193),
                                   which copies the `model_ema.*` shadow (LitEma, ldm/modules/ema.py:14-21: parameter name
                                   with the dots removed) over `model.*` -- so the EMA shadow is what must be loaded.
"""
from __future__ import annotations

import os
import re


# --------------------------------------------------------------------------------------------- HOCON subset
class Conf(dict):
    """Nested dict with pyhocon's access pattern: conf['a.b.c'], conf.get_int('a.b', default=...), `in`."""

    def _walk(self, key):
        cur = self
        for part in key.split("."):
            if not isinstance(cur, dict) or part not in cur:
                raise KeyError(key)
            cur = dict.__getitem__(cur, part)
        return cur

    def __getitem__(self, key):
        return self._walk(key) if isinstance(key, str) and "." in key else dict.__getitem__(self, key)

    def __setitem__(self, key, value):
        if isinstance(key, str) and "." in key:
            head, tail = key.rsplit(".", 1)
            dict.__setitem__(self._walk(head), tail, value)
        else:
            dict.__setitem__(self, key, value)

    def __contains__(self, key):
        try:
            self[key]
            return True
        except KeyError:
            return False

    _missing = object()

    def get(self, key, default=None):
        try:
            return self[key]
        except KeyError:
            return default

    def _typed(self, key, default, cast):
        try:
            v = self[key]
        except KeyError:
            if default is Conf._missing:
                raise
            return default
        return cast(v)

    def get_int(self, key, default=_missing):
        return self._typed(key, default, int)

    def get_float(self, key, default=_missing):
        return self._typed(key, default, float)

    def get_bool(self, key, default=_missing):
        return self._typed(key, default, lambda v: v if isinstance(v, bool) else str(v).lower() in ("true", "yes", "on", "1"))

    def get_string(self, key, default=_missing):
        return self._typed(key, default, str)

    def get_list(self, key, default=_missing):
        return self._typed(key, default, list)


_TOKEN = re.compile(r"""[ \t\r]*(?:(?P<brace>[{}\[\]])|(?P<eq>[=:])|(?P<comma>,)|(?P<nl>\n)|"(?P<q>[^"]*)"|(?P<w>[^\s{}\[\]=:,"]+))""")


def _scalar(tok):
    low = tok.lower()
    if low in ("true", "yes", "on"):
        return True
    if low in ("false", "no", "off"):
        return False
    if low == "null":
        return None
    try:
        return int(tok)
    except ValueError:
        pass
    try:
        return float(tok)
    except ValueError:
        return tok


def parse_conf(text: str) -> Conf:
    """`key = value`, `key { ... }`, `[a, b]` lists (comma- or newline-separated), `#` / `//` comments, optional commas
    after values, unquoted strings (paths).  Enough for every file under reference reconstruction/confs/."""
    text = re.sub(r"(#|//)[^\n]*", "", text)
    toks, pos = [], 0
    while pos < len(text):
        m = _TOKEN.match(text, pos)
        if not m:
            if text[pos:].strip() == "":
                break
            raise ValueError("conf: cannot tokenise at %r" % text[pos:pos + 30])
        pos = m.end()
        if m.group("brace"):
            toks.append(("b", m.group("brace")))
        elif m.group("eq"):
            toks.append(("=", "="))
        elif m.group("comma"):
            toks.append((",", ","))
        elif m.group("nl"):
            toks.append(("n", "\n"))
        elif m.group("q") is not None:
            toks.append(("s", m.group("q")))
        else:
            toks.append(("w", m.group("w")))
    i = 0

    def skip_sep():
        nonlocal i
        while i < len(toks) and toks[i][0] in (",", "n"):
            i += 1

    def value():
        nonlocal i
        kind, tok = toks[i]
        if (kind, tok) == ("b", "{"):
            i += 1
            return obj("}")
        if (kind, tok) == ("b", "["):
            i += 1
            out = []
            while True:
                skip_sep()
                if toks[i] == ("b", "]"):
                    i += 1
                    return out
                out.append(value())
        i += 1
        if kind == "s":
            return tok
        # an unquoted value runs to the end of the line / next separator (paths such as ./data)
        parts = [tok]
        while i < len(toks) and toks[i][0] == "w":
            parts.append(toks[i][1])
            i += 1
        return _scalar(parts[0]) if len(parts) == 1 else " ".join(parts)

    def obj(close):
        nonlocal i
        out = Conf()
        while True:
            skip_sep()
            if i >= len(toks):
                if close is None:
                    return out
                raise ValueError("conf: unterminated object")
            if close is not None and toks[i] == ("b", close):
                i += 1
                return out
            kind, key = toks[i]
            if kind not in ("w", "s"):
                raise ValueError("conf: expected a key, got %r" % (key,))
            i += 1
            if i < len(toks) and toks[i][0] == "=":
                i += 1
                while i < len(toks) and toks[i][0] == "n":
                    i += 1
            v = value()
            cur = out
            parts = key.split(".")
            for part in parts[:-1]:
                cur = cur.setdefault(part, Conf())
            if isinstance(v, dict) and isinstance(dict.get(cur, parts[-1]), dict):
                dict.get(cur, parts[-1]).update(v)      # HOCON merges repeated objects
            else:
                dict.__setitem__(cur, parts[-1], v)

    return obj(None)


def load_conf(path) -> Conf:
    with open(path) as fh:
        return parse_conf(fh.read())


# --------------------------------------------------------------------------------------------- reconstruction checkpoints
def latest_checkpoint(base_exp_dir):
    """reference exp_runner_generic_blender_val.py:137-149: names starting with 'ckpt' and ending in 'pth', sorted as
    strings, the last one.  Returns the full path or None if the folder holds none."""
    folder = os.path.join(base_exp_dir, "checkpoints")
    if not os.path.isdir(folder):
        return None
    names = sorted(n for n in os.listdir(folder) if n.startswith("ckpt") and n[-3:] == "pth")
    return os.path.join(folder, names[-1]) if names else None


RECON_NETWORKS = {"pyramid_feature_network": "pyramid_feature_network", "sdf_network_lod0": "sdf_network_lod0",
                  "rendering_network_lod0": "rendering_network_lod0", "variance_network_lod0": "variance_network_lod0"}
RECON_NETWORKS_LOD1 = {k: k for k in ("pyramid_feature_network_lod1", "sdf_network_lod1", "rendering_network_lod1",
                                      "variance_network_lod1")}


def recon_states(checkpoint: dict, report=None, num_lods=1):
    """{network name -> state dict} for the four lod-0 networks of a `ckpt_*.pth` (the keys save_checkpoint writes,
    reference :480-503).  A network the file does not hold is reported ("<name> load fails", as the reference prints) and
    left out, so that the caller keeps its initialisation -- the reference's behaviour, made visible.  The four lod-1
    networks are passed through when the file holds them; with num_lods = 2 a file that lacks one is refused (KeyError):
    a lod-1 level with initial weights would refine the surface with noise."""
    out = {}
    for name, key in RECON_NETWORKS.items():
        if key in checkpoint and checkpoint[key] is not None:
            out[name] = checkpoint[key]
        elif report is not None:
            report(f"{key} load fails")
    for name, key in RECON_NETWORKS_LOD1.items():
        if checkpoint.get(key) is not None:
            out[name] = checkpoint[key]
        elif num_lods > 1:
            raise KeyError(f"num_lods = 2 but the checkpoint has no {key!r}")
    return out


# --------------------------------------------------------------------------------------------- Zero123 checkpoints
def ema_shadow_name(param_name: str) -> str:
    """LitEma.m_name2s_name (reference ldm/modules/ema.py:16-21): '.' is not allowed in buffer names, so it is removed."""
    return param_name.replace(".", "")


def zero123_sampling_state(sd: dict, model_param_names, use_ema=True, report=None):
    """The state dict Zero123 samples with.  `sd` is a Lightning-style checkpoint state dict (`model.diffusion_model.*`,
    `model_ema.*`, `first_stage_model.*`, `cond_stage_model.*`, `cc_projection.*`, schedule buffers); `model_param_names`
    are the parameter names of the DiffusionWrapper (`diffusion_model.input_blocks.0.0.weight`, ...).  With use_ema and
    an EMA shadow present, every `model.<name>` entry is replaced by `model_ema.<name without dots>`; a shadow that covers
    only part of the parameters is an error (the reference would fail in copy_to too)."""
    out = {k: v for k, v in sd.items() if not k.startswith("model_ema.")}
    has_ema = any(k.startswith("model_ema.") and k not in ("model_ema.decay", "model_ema.num_updates") for k in sd)
    if use_ema and has_ema:
        missing = []
        for name in model_param_names:
            key = "model_ema." + ema_shadow_name(name)
            if key in sd:
                out["model." + name] = sd[key]
            else:
                missing.append(name)
        if missing:
            raise KeyError(f"EMA shadow (model_ema.*) lacks {len(missing)} of {len(list(model_param_names))} parameters, "
                           f"e.g. {missing[0]!r}: refusing to sample with a mix of EMA and raw weights")
        if report is not None:
            report("sampling with the EMA weights (model_ema.*), as the reference's ema_scope() does")
    elif report is not None:
        report("checkpoint has no EMA shadow: sampling with model.* as stored" if use_ema else "EMA weights ignored on request")
    return out
