"""Object builder of the experiment configuration
(behaviour of neuralmonkey/config/builder.py:19-249).

A section with `class=dotted.path` becomes the object `path(**other options)`; references
`<section>` are built on demand and shared; a constructor parameter `name: str` defaults to
the section name.  Symbol resolution tries, in order: the literal module path, the `tf.`
compatibility namespace (neuralmonkey_b200.tf), and `neuralmonkey_b200.<path>` - the place
the reference looks for `neuralmonkey.<path>` - so unmodified Neural Monkey INI files
resolve to the H100 implementations.
"""
import importlib
from argparse import Namespace
from collections import OrderedDict
from collections.abc import Iterable
from inspect import Parameter, isclass, isfunction, signature
from typing import Any, Dict, Set, Tuple

from neuralmonkey_b200.config.exceptions import ConfigBuildException, ConfigInvalidValueException
from neuralmonkey_b200.logging import debug, warn

PACKAGE = "neuralmonkey_b200"


class ClassSymbol:
    """A dotted class / function name from the configuration."""

    def __init__(self, string: str) -> None:
        self.clazz = string

    def __repr__(self) -> str:
        return "ClassSymbol({})".format(self.clazz)

    def create(self) -> Any:
        parts = self.clazz.split(".")
        attr, module_path = parts[-1], ".".join(parts[:-1])
        module = None
        if parts[0] == "tf":
            module = importlib.import_module(PACKAGE + ".tf")
            for part in parts[1:-1]:
                module = getattr(module, part)
        else:
            for candidate in (PACKAGE + "." + module_path, module_path):
                try:
                    module = importlib.import_module(candidate)
                    break
                except ImportError as exc:
                    # a module that exists but fails inside must not be masked
                    if exc.name not in (candidate, candidate.split(".")[0]) and \
                            not candidate.startswith(str(exc.name)):
                        raise
            if module is None:
                raise Exception("Cannot import module {}.".format(module_path))
        try:
            return getattr(module, attr)
        except AttributeError as exc:
            raise Exception(("Interpretation '{}' as type name, class '{}' does not exist. "
                             "Did you mean file './{}'? \n{}").format(self.clazz, attr, self.clazz, exc))


class ObjectRef:
    """`<name.attr1.attr2>`: a section object, optionally followed by attribute accesses."""

    def __init__(self, expression: str) -> None:
        self.expression = expression
        self.name, *self.attr_chain = expression.split(".")
        self._obj = None

    def __repr__(self) -> str:
        return "ObjectRef({})".format(self.expression)

    def bind(self, value: Any) -> None:
        self._obj = value

    @property
    def target(self) -> Any:
        value = self._obj
        for attr in self.attr_chain:
            value = getattr(value, attr)
        return value


def build_object(value: Any, all_dicts: Dict[str, Any], existing: Dict[str, Any], depth: int) -> Any:
    """Resolve a parsed value recursively (lists, tuples, references, class symbols)."""
    if depth > 20:
        raise AssertionError("Config recursion should not be deeper that 20.")
    if isinstance(value, tuple):
        return tuple(build_object(v, all_dicts, existing, depth + 1) for v in value)
    if isinstance(value, Iterable) and not isinstance(value, str):
        return [build_object(v, all_dicts, existing, depth + 1) for v in value]
    if isinstance(value, ObjectRef):
        if value.name not in existing:
            existing[value.name] = instantiate_class(value.name, all_dicts, existing, depth)
        value.bind(existing[value.name])
        return value.target
    if isinstance(value, ClassSymbol):
        return value.create()
    return value


def instantiate_class(name: str, all_dicts: Dict[str, Any], existing: Dict[str, Any],
                      depth: int) -> Any:
    if name not in all_dicts:
        raise ConfigInvalidValueException(name, "Undefined object")
    this_dict = all_dicts[name]
    if "class" not in this_dict:
        raise ConfigInvalidValueException(name, "Undefined object type")
    clazz = this_dict["class"].create()
    if not isclass(clazz) and not isfunction(clazz):
        raise ConfigInvalidValueException(name, "Cannot instantiate object with '{}'".format(clazz))
    arguments = {key: build_object(val, all_dicts, existing, depth + 1)
                 for key, val in this_dict.items() if key != "class"}
    sig = signature(clazz)
    if "name" in sig.parameters and "name" not in arguments:
        if sig.parameters["name"].annotation == str:
            arguments["name"] = name
        else:
            debug("'name' parameter of {} is not annotated as str: section name not used"
                  .format(this_dict["class"].clazz), "configBuild")
    try:
        bound = sig.bind(**arguments)
    except TypeError as exc:
        raise ConfigBuildException(clazz, exc)
    debug("Instantiating class {} with arguments {}".format(clazz, arguments), "configBuild")
    return clazz(*bound.args, **bound.kwargs)


def build_config(config_dicts: Dict[str, Any], ignore_names: Set[str],
                 warn_unused: bool = False) -> Tuple[Dict[str, Any], Dict[str, Any]]:
    """Build everything [main] refers to; `tf_manager` is built last (builder.py:231-234)."""
    if "main" not in config_dicts:
        raise Exception("Configuration does not contain the main block.")
    existing = OrderedDict()  # type: Dict[str, Any]
    main_config = config_dicts["main"]
    existing["main"] = Namespace(**main_config)
    configuration = OrderedDict()  # type: Dict[str, Any]
    for key, value in sorted(main_config.items(), key=lambda t: t[0] if t[0] != "tf_manager" else "zzz"):
        if key not in ignore_names:
            try:
                configuration[key] = build_object(value, config_dicts, existing, 0)
            except Exception as exc:
                raise ConfigBuildException(key, exc) from None
    if warn_unused:
        unused = config_dicts.keys() - (set(existing.keys()) | {"main"})
        if unused:
            warn("Configuration contains unused sections: " + str(unused) + ".")
    return configuration, existing
