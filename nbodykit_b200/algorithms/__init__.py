from .fftpower import FFTPower, FFTBase, ProjectedFFTPower, project_to_basis
from .fftcorr import FFTCorr
from .fftrecon import FFTRecon
from .fof import FOF
from .cgm import CylindricalGroups
from .paircount import SimulationBoxPairCount, SimulationBox2PCF
from .threeptcf import SimulationBox3PCF, SurveyData3PCF
from .surveypaircount import SurveyDataPairCount, SurveyData2PCF
from .convpower import ConvolvedFFTPower, FKPCatalog, FKPWeightFromNbar, FKPCatalogMesh

FKPPower = ConvolvedFFTPower

__all__ = ['FOF', 'CylindricalGroups', 'SimulationBoxPairCount', 'SimulationBox2PCF', 'SimulationBox3PCF', 'SurveyDataPairCount',
           'SurveyData2PCF', 'SurveyData3PCF', 'FFTCorr', 'FFTRecon', 'FFTPower', 'ProjectedFFTPower', 'FFTBase', 'project_to_basis', 'ConvolvedFFTPower', 'FKPPower', 'FKPCatalog',
           'FKPWeightFromNbar', 'FKPCatalogMesh']
