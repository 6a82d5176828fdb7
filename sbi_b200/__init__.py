"""sbi_b200: H100-native (sm_90a) density-estimator training and posterior evaluation,
drop-in at sbi's builder / estimator API.  See DESIGN.md and INTEGRATION.md."""
__version__ = "0.1.0"
