"""Global config object (reference: video_to_video/utils/config.py:11).
Only the three fields the hot path reads are kept
(video_to_video_model.py:36,68-69): model_path, negative_prompt,
positive_prompt -- the prompt strings are data, quoted from config.py:160-167."""


class _Cfg(dict):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.__dict__ = self


cfg = _Cfg(__name__="Config: STAR sm_90a")
cfg.model_path = None
cfg.negative_prompt = ("painting, oil painting, illustration, drawing, art, sketch, oil painting, cartoon, "
                       "CG Style, 3D render, unreal engine, blurring, dirty, messy, worst quality, low quality, "
                       "frames, watermark, signature, jpeg artifacts, deformed, lowres, over-smooth")
cfg.positive_prompt = ("Cinematic, High Contrast, highly detailed, taken using a Canon EOS R camera,   "
                       "hyper detailed photo - realistic maximum detail, 32k, Color Grading, ultra HD, "
                       "extreme meticulous detailing,  skin pore detailing, hyper sharpness, perfect without "
                       "deformations.")
