"""LLFF loading is outside the NeRFace render path (SURVEY.md §2 row 9); the name is kept importable because the
reference's scripts import it (train_transformed_rays.py:17-21)."""


def load_llff_data(*args, **kwargs):
    raise NotImplementedError("LLFF datasets are out of scope of the H100 NeRFace render path")
