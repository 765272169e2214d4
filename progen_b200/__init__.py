"""progen_b200 — H100-native (sm_90a) ProGen training + sampling engine (drop-in for lucidrains/progen's `ProGen`)."""


def __getattr__(name):
    if name == 'ProGen':
        from .progen import ProGen
        return ProGen
    raise AttributeError(name)
