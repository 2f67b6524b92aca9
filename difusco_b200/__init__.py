"""difusco_b200: H100-native (sm_90a) implementation of DIFUSCO's denoising-inference hot path.

Host mirror of the reference interface (same module / class / method names):
    difusco_b200.models.gnn_encoder.GNNEncoder
    difusco_b200.utils.diffusion_schedulers.{CategoricalDiffusion, GaussianDiffusion, InferenceSchedule}
    difusco_b200.pl_meta_model.COMetaModel, pl_tsp_model.TSPModel, pl_mis_model.MISModel
All device work goes through the C-ABI library libdifusco_b200.so (include/difusco_b200.h).
"""
__version__ = "0.1.0"
