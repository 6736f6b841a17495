"""Run configurations as plain nested dicts, from the reference's `configs/` tree or from one YAML file (a run's `parsed.yaml`).

Only the composition features the reference's shipped configs use are built (hydra and OmegaConf are not dependencies):

  * a `defaults:` list with entries `/group: option`, `/config`, a relative `name` (same directory), `override /group: option` and
    `_self_` (where the file's own keys are merged; last when it is absent); `override hydra/...` entries are ignored;
  * a file's package: `# @package _global_` puts its keys at the root, otherwise they land under its directory (`dataset/colmap.yaml`
    under `dataset:`);
  * interpolations `${a.b}` (absolute), string concatenation (`${render.pipeline_type}Bwd`) and the resolvers `${div:x,y}` and
    `${int_list:[...]}` (threedgrut/utils/misc.py:26, train.py:24).

`key=value` overrides are parsed as YAML scalars and applied to the composed config before its interpolations are resolved, as hydra
applies them; an unknown key raises KeyError, `+key=value` adds one.  The `hydra:` section is dropped."""
from __future__ import annotations

import copy
import os
import re

import yaml

RESOLVERS = {"div": lambda a, b: a / b, "int_list": lambda lst: [int(x) for x in lst]}


def load(config_dir=None, config_name=None, config_file=None, overrides=()) -> dict:
    """The resolved config: composed from `config_name` (e.g. "apps/colmap_3dgut_mcmc.yaml") under `config_dir`, or read from
    `config_file`; then `overrides` ("key=value" / "+key=value") and the interpolations."""
    if (config_file is None) == (config_name is None):
        raise ValueError("pass config_file, or config_dir and config_name")
    if config_file is not None:
        with open(config_file) as f:
            conf = yaml.safe_load(f) or {}
        conf.pop("defaults", None)
    else:
        if config_dir is None:
            raise ValueError("config_name needs config_dir")
        conf = compose(config_dir, config_name)
    conf.pop("hydra", None)
    apply_overrides(conf, overrides)
    return resolve(conf)


# ---- composition ---------------------------------------------------------------------------------------------------------------------

def _read(root: str, name: str):
    """(contents, header package or None) of the config `name` (path under root, with or without .yaml)."""
    path = os.path.join(root, name if name.endswith(".yaml") else name + ".yaml")
    if not os.path.isfile(path):
        raise FileNotFoundError(f"config {name!r} not found under {root}")
    with open(path) as f:
        text = f.read()
    m = re.search(r"^#\s*@package\s+(\S+)", text, re.M)
    return yaml.safe_load(text) or {}, (m.group(1) if m else None)


def _merge(dst: dict, src: dict) -> dict:
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(dst[k], v)
        else:
            dst[k] = copy.deepcopy(v)
    return dst


def _place(package: str, contents: dict) -> dict:
    out = contents
    for key in reversed([p for p in package.split(".") if p]):
        out = {key: out}
    return out


def compose(root: str, name: str) -> dict:
    """The unresolved config `name` under `root`, its defaults list expanded."""
    return _compose(root, name.removesuffix(".yaml").lstrip("/"), {})


def _compose(root: str, name: str, chosen: dict) -> dict:
    contents, header = _read(root, name)
    directory = os.path.dirname(name)
    package = "" if header == "_global_" else (directory.replace("/", ".") if header in (None, "_group_") else header)
    defaults = contents.pop("defaults", None) or []
    # this file's overrides of group choices apply to the whole subtree; an outer file's override wins over an inner one's
    chosen = dict(chosen)
    for entry in defaults:
        if isinstance(entry, dict):
            (key, option), = entry.items()
            if key.startswith("override "):
                group = key[len("override "):].strip().lstrip("/")
                if not group.startswith("hydra/"):
                    chosen.setdefault(group, option)
    if "_self_" not in defaults:
        defaults = list(defaults) + ["_self_"]
    out = {}
    for entry in defaults:
        if entry == "_self_":
            _merge(out, _place(package, contents))
        elif isinstance(entry, str):
            target = entry.lstrip("/") if entry.startswith("/") else os.path.join(directory, entry)
            _merge(out, _compose(root, target, chosen))
        else:
            (key, option), = entry.items()
            if key.startswith("override "):
                continue
            group = key.lstrip("/") if key.startswith("/") else os.path.join(directory, key)
            if option is None:
                continue
            _merge(out, _compose(root, f"{group}/{chosen.get(group, option)}", chosen))
    return out


# ---- overrides -----------------------------------------------------------------------------------------------------------------------

def parse_scalar(text: str):
    """A command-line value as YAML reads it, with exponent floats without a dot (1e-3) read as floats as hydra reads them."""
    value = yaml.safe_load(text) if text.strip() else ""
    if isinstance(value, str):
        try:
            return float(value) if re.fullmatch(r"[-+]?(\d+\.?\d*|\.\d+)[eE][-+]?\d+", value) else value
        except ValueError:
            return value
    return value


def apply_overrides(conf: dict, overrides) -> dict:
    for item in overrides:
        if "=" not in item:
            raise ValueError(f"override {item!r}: expected key=value")
        key, text = item.split("=", 1)
        add = key.startswith("+")
        key = key.lstrip("+")
        *parents, leaf = key.split(".")
        node = conf
        for i, p in enumerate(parents):
            if not isinstance(node.get(p), dict):
                if not add:
                    raise KeyError(f"override {item!r}: key {'.'.join(parents[:i + 1])!r} is not in the config (use +{key}=... to add it)")
                node[p] = {}
            node = node[p]
        if add and leaf in node:
            raise KeyError(f"override {item!r}: {key!r} is already in the config (drop the '+' to change it)")
        if not add and leaf not in node:
            raise KeyError(f"override {item!r}: key {key!r} is not in the config (use +{key}=... to add it)")
        node[leaf] = parse_scalar(text)
    return conf


# ---- interpolation -------------------------------------------------------------------------------------------------------------------

def _lookup(root: dict, path: str, stack):
    node = root
    for k in path.split("."):
        if not isinstance(node, dict) or k not in node:
            raise KeyError(f"interpolation ${{{path}}}: key not found")
        node = node[k]
    if path in stack:
        raise ValueError(f"interpolation ${{{path}}}: cycle through {' -> '.join(stack)}")
    return _value(root, node, stack + (path,))


def _close(text: str, start: int) -> int:
    """Index of the `}` that closes the `${` at start."""
    depth, i = 0, start
    while i < len(text):
        if text.startswith("${", i):
            depth, i = depth + 1, i + 2
            continue
        if text[i] == "}":
            depth -= 1
            if depth == 0:
                return i
        i += 1
    raise ValueError(f"unterminated interpolation in {text!r}")


def _expr(root: dict, body: str, stack):
    m = re.fullmatch(r"\s*([A-Za-z_][\w]*)\s*:(.*)", body, re.S)
    if m and m.group(1) in RESOLVERS:
        args_text = _string(root, m.group(2), stack)
        args = [parse_scalar(a) if isinstance(a, str) else a for a in yaml.safe_load(f"[{args_text}]")]
        return RESOLVERS[m.group(1)](*args)
    if m:
        raise ValueError(f"resolver {m.group(1)!r} is not built (built: {', '.join(RESOLVERS)})")
    return _lookup(root, body.strip(), stack)


def _string(root: dict, text: str, stack):
    """text with every interpolation replaced: the value itself when text is one interpolation, else the concatenated string."""
    if "${" not in text:
        return text
    start = text.index("${")
    end = _close(text, start)
    if start == 0 and end == len(text) - 1:
        return _expr(root, text[2:end], stack)
    parts, i = [], 0
    while "${" in text[i:]:
        start = text.index("${", i)
        end = _close(text, start)
        parts += [text[i:start], str(_expr(root, text[start + 2:end], stack))]
        i = end + 1
    return "".join(parts + [text[i:]])


def _value(root: dict, node, stack=()):
    if isinstance(node, dict):
        return {k: _value(root, v, stack) for k, v in node.items()}
    if isinstance(node, list):
        return [_value(root, v, stack) for v in node]
    if isinstance(node, str):
        return _string(root, node, stack)
    return node


def resolve(conf: dict) -> dict:
    """A copy of conf with every interpolation resolved."""
    return _value(conf, conf)
