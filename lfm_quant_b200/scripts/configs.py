"""Flag registry with the reference's API (scripts/configs.py:9-188): DEFINE_{string,integer,boolean,float,
list_*}, a lazily parsed ``ConfigValues`` attribute bag and ``--config FILE`` (whitespace-separated argv tokens).

Behaviour kept: unknown flags are ignored (parse_known_args); booleans accept ``--x``, ``--x=True|t|1`` and
``--nox``; values given on the command line after ``--config`` override the file, values before it are
overridden by the file (argparse left-to-right order, as in the reference).
"""
from __future__ import absolute_import, division, print_function

import argparse

_TRUE = ('true', 't', '1')


class _ConfigFileAction(argparse.Action):
    """--config FILE: re-parse the file's tokens into the same namespace (scripts/configs.py:9-14)."""

    def __call__(self, parser, namespace, values, option_string=None):
        with open(values) as fh:
            tokens = fh.read().split()
        parser.parse_known_args(tokens, namespace)


def _new_parser():
    p = argparse.ArgumentParser()
    p.add_argument('--config', action=_ConfigFileAction, help='File containing configuration')
    return p


_global_parser = _new_parser()
_defined = set()


def reset():
    """Forget every registered flag (tests build several configs in one process)."""
    global _global_parser
    _global_parser = _new_parser()
    _defined.clear()


class ConfigValues(object):
    """Attribute bag over the parsed flags; parses argv on first access (scripts/configs.py:24-56)."""

    def __init__(self, argv=None):
        self.__dict__['__configs'] = {}
        self.__dict__['__parsed'] = False
        self.__dict__['__argv'] = argv

    def _parse_configs(self):
        ns, _ = _global_parser.parse_known_args(self.__dict__.get('__argv'))
        store = self.__dict__.setdefault('__configs', {})
        for k, v in vars(ns).items():
            store[k] = v
        self.__dict__['__parsed'] = True

    def __getattr__(self, name):
        if not self.__dict__.get('__parsed', False):
            self._parse_configs()
        try:
            return self.__dict__['__configs'][name]
        except KeyError:
            raise AttributeError(name)

    def __setattr__(self, name, value):
        if not self.__dict__.get('__parsed', False):
            self._parse_configs()
        self.__dict__['__configs'][name] = value

    def as_dict(self):
        if not self.__dict__.get('__parsed', False):
            self._parse_configs()
        return dict(self.__dict__['__configs'])

    # deep copies are used by the ensemble path of the reference (runtime/model_execution.py:168)
    def __deepcopy__(self, memo):
        import copy
        c = ConfigValues(self.__dict__.get('__argv'))
        c.__dict__['__configs'] = copy.deepcopy(self.as_dict(), memo)
        c.__dict__['__parsed'] = True
        return c

    # pickling (a hyper-parameter search saves its population, scripts/param_search/genetic_algorithm.py) stores the
    # parsed values; without these, unpickling would look __setstate__ up through __getattr__, which parses argv
    def __getstate__(self):
        return self.as_dict()

    def __setstate__(self, state):
        self.__dict__['__configs'] = dict(state)
        self.__dict__['__parsed'] = True
        self.__dict__['__argv'] = None


def _define(name, default, doc, typ):
    if name in _defined:
        return
    _defined.add(name)
    _global_parser.add_argument('--' + name, default=default, help=doc, type=typ)


def DEFINE_string(name, default, doc):
    _define(name, default, doc, str)


def DEFINE_integer(name, default, doc):
    _define(name, default, doc, int)


def DEFINE_float(name, default, doc):
    _define(name, default, doc, float)


def DEFINE_boolean(name, default, doc):
    if name in _defined:
        return
    _defined.add(name)
    _global_parser.add_argument('--' + name, nargs='?', const=True, default=default, help=doc,
                                type=lambda v: v.lower() in _TRUE)
    _global_parser.add_argument('--no' + name, action='store_false', dest=name)


DEFINE_bool = DEFINE_boolean


def _define_list(name, default, doc, typ, wrap):
    if name in _defined:
        return
    _defined.add(name)
    _global_parser.add_argument('--' + name, nargs='*', help=doc, default=wrap(default), type=typ)


def DEFINE_list_integer(name, default, doc):
    _define_list(name, default, doc, int, lambda d: [int(d)] if d is not None else [None])


def DEFINE_list_float(name, default, doc):
    _define_list(name, default, doc, float, lambda d: [float(d)] if d is not None else [None])


def DEFINE_list_string(name, default, doc):
    _define_list(name, default, doc, str, lambda d: [d])


def DEFINE_list_boolean(name, default, doc):
    _define_list(name, default, doc, lambda v: v.lower() in _TRUE, lambda d: [d])
