"""Renderer plugin registry with the call surface of the reference's `gaustudio/renderers/__init__.py:1-28`:
`@register(name)` adds a class, `make(config)` instantiates one from a name or from a mapping with a `name`
key (the whole mapping is handed to the constructor); missing / unknown names raise ValueError."""
from collections.abc import Mapping

renderers = {}  # name -> class (public, like the reference's module-level dict)


def register(name):
    def _add(cls):
        renderers[name] = cls
        return cls
    return _add


def _split(config):
    if isinstance(config, str):
        return config, {}
    if isinstance(config, Mapping) or hasattr(config, "get"):
        return config.get("name"), config
    raise ValueError("Renderer name is required")


def make(config):
    name, options = _split(config)
    if not name:
        raise ValueError("Renderer name is required")
    try:
        cls = renderers[name]
    except KeyError:
        raise ValueError(f"Unknown renderer: {name}") from None
    return cls(options)


from . import vanilla_renderer  # noqa: E402,F401  (the only renderer on the hot path; SURVEY.md §2.1)
from . import surfel_renderer  # noqa: E402,F401  (2DGS: configs/2dgs.yaml)
from . import mip_renderer  # noqa: E402,F401  (Mip-Splatting)
from . import scaffold_renderer  # noqa: E402,F401  (Scaffold-GS)
