"""ORACLE SHIM: ujson's load / loads / dump / dumps over the standard json module. The reference's data.py reads its
measurement and label files with ujson.load; every float in the generated route (oracle/synthetic_route.py) is dyadic, so both
parsers give the same doubles."""
import json


def load(fp, **kw):
    return json.load(fp, **kw)


def loads(s, **kw):
    return json.loads(s, **kw)


def dump(obj, fp, **kw):
    return json.dump(obj, fp, **kw)


def dumps(obj, **kw):
    return json.dumps(obj, **kw)
