"""Plugin loading the way Coach does it (rl_coach/utils.py:334-404): components are named by ``'module:Class'`` path
strings carried by their Parameters object and instantiated with the intersection of constructor argument names and
parameter attributes."""
import contextlib
import gc
import importlib
import inspect

import torch


def short_dynamic_import(module_path_and_attribute: str):
    module_path, attr = module_path_and_attribute.split(":")
    if module_path.endswith(".py"):
        module_path = module_path[:-3].replace("/", ".")
    return getattr(importlib.import_module(module_path), attr)


def dynamic_import_and_instantiate_module_from_params(module_parameters, path=None, positional_args=(),
                                                      extra_kwargs=None):
    if path is None:
        path = module_parameters.path
    cls = short_dynamic_import(path)
    ctor_args = set(inspect.getfullargspec(cls).args)
    kwargs = {k: v for k, v in module_parameters.__dict__.items() if k in ctor_args}
    for k, v in (extra_kwargs or {}).items():
        if k in ctor_args:
            kwargs[k] = v
    return cls(*positional_args, **kwargs)


@contextlib.contextmanager
def graph_capture(graph):
    """``torch.cuda.graph(graph)`` with Python's cyclic garbage collector held off.  Agents are often reference cycles
    (a graphed step holds a bound method of its agent), so pinned staging buffers of dead agents are freed only when
    the collector runs; freeing a pinned block that served an asynchronous copy records a CUDA event on that copy's
    stream, which invalidates a capture in progress.  Garbage is collected before the capture instead."""
    gc.collect()
    enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(graph):
            yield
    finally:
        if enabled:
            gc.enable()
