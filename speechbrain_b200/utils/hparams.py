"""A HyperPyYAML-subset loader + ``Pretrained.from_hparams`` for local directories (SURVEY 8f N1).

The reference builds every inference interface from a ``hyperparams.yaml`` with the HyperPyYAML package
(inference/interfaces.py:385-489); that package is not installable offline, so this module implements the part of the
format the ASR inference YAMLs use:

* ``!new:dotted.Class`` (mapping -> kwargs, sequence -> positional args, empty -> no args), ``!name:dotted.callable``
  (``functools.partial``), ``!apply:dotted.callable``;
* ``!ref <key>`` -- the SAME object every time (like a YAML alias), dotted sub-keys ``<a.b>``, string interpolation
  ``!ref <save_folder>/lm.ckpt`` and simple arithmetic ``!ref <a> * 2``; ``!copy <key>``;
* tuples written ``(64, 32)``; ``!include:`` / ``!applyref`` are not built and raise.

Objects are constructed lazily (only what ``modules`` / ``pretrainer`` / the needed hparams reach), so the training-only
entries of a recipe YAML (augmentations, optimisers, schedulers, loggers) never have to exist here.  Dotted names under
``speechbrain.`` resolve to this package's drop-in mirrors; a name with no mirror raises NotImplementedError when reached."""
import ast
import functools
import importlib
import os
import re
import types

import yaml

PACKAGE = __name__.split(".")[0]  # "speechbrain_b200"
_REF = re.compile(r"<([A-Za-z_][\w.]*)>")


class _Tagged:
    def __init__(self, kind, name, node):
        self.kind, self.name, self.node = kind, name, node


def resolve_name(dotted):
    """Import ``a.b.C``; ``speechbrain.`` maps onto this package's mirrors."""
    names = [dotted]
    if dotted == "speechbrain" or dotted.startswith("speechbrain."):
        names = [PACKAGE + dotted[len("speechbrain"):]]
    last_err = None
    for name in names:
        parts = name.split(".")
        for i in range(len(parts) - 1, 0, -1):
            try:
                obj = importlib.import_module(".".join(parts[:i]))
            except ImportError as e:  # noqa: PERF203
                last_err = e
                continue
            try:
                for p in parts[i:]:
                    obj = getattr(obj, p)
                return obj
            except AttributeError as e:
                last_err = e
                break
    if dotted.startswith("speechbrain"):
        raise NotImplementedError(f"{dotted} has no {PACKAGE} mirror (only the ASR inference hot path is built): {last_err}")
    raise ImportError(f"cannot resolve {dotted}: {last_err}")


class HParams:
    """Lazy view of a HyperPyYAML-subset document: ``hp["key"]`` constructs (once) and returns the value."""

    def __init__(self, text, overrides=None):
        self.root = yaml.compose(text, Loader=yaml.SafeLoader)
        if self.root is None or not isinstance(self.root, yaml.MappingNode):
            raise ValueError("hyperparams: the top level must be a mapping")
        self.nodes = {k.value: v for k, v in self.root.value}
        self.overrides = dict(overrides or {})
        self.cache = {}
        self._building = []

    def keys(self):
        return list(self.nodes)

    def __contains__(self, key):
        return key in self.nodes or key in self.overrides

    def __getitem__(self, key):
        head, _, rest = key.partition(".")
        if head not in self.cache:
            if head in self.overrides:
                self.cache[head] = self.overrides[head]
            else:
                if head not in self.nodes:
                    raise KeyError(f"hyperparams: <{key}> is not defined")
                if head in self._building:
                    raise ValueError(f"hyperparams: circular reference through <{head}>")
                self._building.append(head)
                try:
                    self.cache[head] = self._build(self.nodes[head])
                finally:
                    self._building.pop()
        val = self.cache[head]
        for part in rest.split(".") if rest else []:
            val = val[part] if isinstance(val, dict) else getattr(val, part)
        return val

    def get(self, key, default=None):
        return self[key] if key in self else default

    # ------------------------------------------------------------------ construction
    def _scalar(self, node):
        tag, v = node.tag, node.value
        if tag == "tag:yaml.org,2002:str" and node.style is None and re.fullmatch(r"\(.*\)", v.strip()):
            try:
                return ast.literal_eval(v.strip())  # HyperPyYAML's implicit tuple
            except (ValueError, SyntaxError):
                return v
        return yaml.SafeLoader.construct_object(_loader_for(node), node, deep=True)

    def _ref(self, expr):
        expr = expr.strip()
        m = _REF.fullmatch(expr)
        if m:
            return self[m.group(1)]
        vals = {}

        def sub(mm):
            v = self[mm.group(1)]
            vals[mm.group(1)] = v
            return str(v)
        text = _REF.sub(sub, expr)
        if vals and all(isinstance(v, (int, float)) and not isinstance(v, bool) for v in vals.values()) and \
                re.fullmatch(r"[\d\s.+\-*/()%eE]+", text):
            return _safe_arith(text)
        return text

    def _build(self, node):
        tag = node.tag or ""
        if tag.startswith("!ref") or tag.startswith("!copy"):
            val = self._ref(node.value)
            if tag.startswith("!copy"):
                import copy
                val = copy.deepcopy(val)
            return val
        for kind in ("new", "name", "apply"):
            if tag.startswith(f"!{kind}:"):
                target = resolve_name(tag[len(kind) + 2:])
                args, kwargs = [], {}
                if isinstance(node, yaml.MappingNode):
                    kwargs = {k.value: self._build(v) for k, v in node.value}
                elif isinstance(node, yaml.SequenceNode):
                    args = [self._build(v) for v in node.value]
                elif node.value not in ("", None):
                    args = [self._scalar(_retag(node))]
                if kind == "name":
                    return functools.partial(target, *args, **kwargs) if (args or kwargs) else target
                return target(*args, **kwargs)
        if tag.startswith("!include") or tag.startswith("!applyref") or tag.startswith("!module"):
            raise NotImplementedError(f"hyperparams: tag {tag} is not built")
        if tag == "!tuple":
            return tuple(self._build(v) for v in node.value)
        if tag.startswith("!") and not tag.startswith("!!"):
            raise NotImplementedError(f"hyperparams: unknown tag {tag}")
        if isinstance(node, yaml.MappingNode):
            return {self._build(k) if not isinstance(k, yaml.ScalarNode) else k.value: self._build(v) for k, v in node.value}
        if isinstance(node, yaml.SequenceNode):
            return [self._build(v) for v in node.value]
        return self._scalar(node)


def _retag(node):
    """A tagged scalar's payload resolved as a plain YAML scalar (e.g. ``!new:Foo 3``)."""
    tag = yaml.SafeLoader.yaml_implicit_resolvers  # noqa: F841  (resolver table lives on the class)
    resolver = yaml.resolver.Resolver()
    return yaml.ScalarNode(resolver.resolve(yaml.ScalarNode, node.value, (True, False)), node.value)


def _loader_for(node):
    ld = yaml.SafeLoader("")
    return ld


def _safe_arith(text):
    tree = ast.parse(text, mode="eval")
    ok = (ast.Expression, ast.BinOp, ast.UnaryOp, ast.Constant, ast.Add, ast.Sub, ast.Mult, ast.Div, ast.FloorDiv, ast.Mod,
          ast.Pow, ast.USub, ast.UAdd)
    for n in ast.walk(tree):
        if not isinstance(n, ok):
            raise ValueError(f"hyperparams: unsupported arithmetic in !ref: {text}")
    return eval(compile(tree, "<ref>", "eval"), {"__builtins__": {}})  # noqa: S307 (AST whitelisted above)


def load_hyperpyyaml(yaml_stream, overrides=None):
    """Mirror of hyperpyyaml.load_hyperpyyaml for the subset above; returns the lazy ``HParams`` view."""
    text = yaml_stream.read() if hasattr(yaml_stream, "read") else yaml_stream
    if isinstance(overrides, str):
        overrides = yaml.safe_load(overrides) or {}
    return HParams(text, overrides)


def load_pretrained_interface(cls, source, hparams_file="hyperparams.yaml", overrides=None, run_opts=None):
    """inference/interfaces.py:385-489 (``Pretrained.from_hparams``) for a local ``source`` directory: load the YAML, run the
    ``pretrainer`` (collect_files(default_source=source) + load_collected()), build ``cls(modules, hparams, run_opts)``."""
    source = str(source)
    path = os.path.join(source, hparams_file)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found (from_hparams loads local directories only: no network)")
    with open(path) as f:
        hp = load_hyperpyyaml(f, overrides)
    if "modules" not in hp:
        raise ValueError("hyperparams: `modules` is required")
    modules = hp["modules"]
    if "pretrainer" in hp:
        pre = hp["pretrainer"]
        pre.set_collect_in(source)
        pre.collect_files(default_source=source)
        pre.load_collected()
    needed = {k: hp[k] for k in getattr(cls, "HPARAMS_NEEDED", []) if k in hp}
    missing = [k for k in getattr(cls, "HPARAMS_NEEDED", []) if k not in hp]
    if missing:
        raise ValueError(f"Need hparams {missing}")
    for opt in ("transformer_beam_search", "transducer_beam_search", "sample_rate", "test_beam_search", "tokenizer"):
        if opt in hp:
            needed[opt] = hp[opt]
    return cls(modules=modules, hparams=types.SimpleNamespace(**needed), run_opts=run_opts)
