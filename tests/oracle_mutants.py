"""Source mutants of the CPU oracles, shared by the edge-case modules (score_edges.py, fit_edges.py).

A mutant is a table entry name -> (what a kernel would get wrong, the functions patched, [(oracle text, mutant text)]).
Each function is named (module, qualified name), a method as "Class.method".  Inside `mutant(table, name)` each
function's source has every edit that applies to it replaced (at least one must apply, each exactly once), is compiled
in its module's namespace and bound wherever the original is held: module globals (the oracles import each other's
functions by name) or, for a method, its class.  Everything is restored on exit."""
import contextlib
import inspect
import sys
import textwrap


def _replace(fn, new):
    """Bind `new` wherever a loaded module holds `fn`"""
    undo = []
    for m in list(sys.modules.values()):
        d = getattr(m, "__dict__", None)
        if not d:
            continue
        for k, v in list(d.items()):
            if v is fn:
                undo.append((d, k, v))
                d[k] = new
    return undo


@contextlib.contextmanager
def mutant(table, name, **extra):
    """The oracle with mutant `name` of `table` applied; `extra` adds names the mutant texts use to the namespace"""
    _, funcs, edits = table[name]
    undo = []
    try:
        for modname, qual in funcs:
            mod = sys.modules[modname]
            owner, _, fname = qual.rpartition(".")
            cls = getattr(mod, owner) if owner else None
            fn = cls.__dict__[fname] if cls is not None else getattr(mod, fname)
            src = textwrap.dedent(inspect.getsource(fn))
            hit = False
            for old, new in edits:
                if old in src:
                    assert src.count(old) == 1, (name, qual, old)
                    src, hit = src.replace(old, new), True
            assert hit, f"mutant {name}: no edit applies to {modname}.{qual}"
            ns = dict(vars(mod), **extra)
            exec(compile(src, f"<mutant {name} of {modname}.{qual}>", "exec"), ns)
            if cls is not None:
                setattr(cls, fname, ns[fname])
                undo.append((None, (cls, fname), fn))
            else:
                undo += _replace(fn, ns[fname])
        yield
    finally:
        for d, k, v in reversed(undo):
            if d is None:
                setattr(*k, v)
            else:
                d[k] = v
