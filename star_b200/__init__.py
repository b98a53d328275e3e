"""star_b200 -- Hopper-native (sm_90a, H100) implementation of the STAR
video-super-resolution denoising hot path (NJU-PCALab/STAR,
video_to_video/: VideoToVideo_sr.test -> GaussianDiffusion.sample_sr ->
ControlledV2VUNet.forward).  See DESIGN.md."""
__version__ = "0.1.0"
