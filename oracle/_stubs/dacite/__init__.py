"""Stand-in for dacite (absent offline) so that the reference's view_sampler_evaluation.py imports: from_dict
builds the IndexEntry dataclass from a JSON entry, casting lists to tuples (Config(cast=[tuple]))."""
import dataclasses


class Config:
    def __init__(self, cast=()):
        self.cast = list(cast)


def from_dict(data_class, data, config=None):
    cast = config.cast if config is not None else []
    kw = {}
    for f in dataclasses.fields(data_class):
        v = data[f.name]
        kw[f.name] = tuple(v) if tuple in cast and isinstance(v, list) else v
    return data_class(**kw)
