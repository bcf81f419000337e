"""ORACLE / TEST INFRASTRUCTURE ONLY. Empty stand-in so team_code_transfuser/point_pillar.py:6
imports; PointPillars is off by default (config.py:42) and out of scope."""


def scatter_mean(*a, **k):
    raise NotImplementedError


def scatter_max(*a, **k):
    raise NotImplementedError
