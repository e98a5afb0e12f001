from .array import ArrayCatalog
from .uniform import UniformCatalog, RandomCatalog
from .lognormal import LogNormalCatalog
from .species import MultipleSpeciesCatalog
from .halos import HaloCatalog, PopulatedHaloCatalog

__all__ = ["ArrayCatalog", "UniformCatalog", "RandomCatalog", "LogNormalCatalog", "MultipleSpeciesCatalog", "HaloCatalog",
           "PopulatedHaloCatalog"]
