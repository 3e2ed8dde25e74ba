"""The reconstruction stage's image datasets (reference: cmr_data/): CUB-200-2011 (`cub.CUBDataset`) and PASCAL3D+
(`p3d.P3dDataset`) with their annotation masks and SfM poses, run_reconstruction.py's `ImageDataset` wrapper, and the device
path that builds a whole batch in one kernel (`base.BaseDataset.to_device`)."""
