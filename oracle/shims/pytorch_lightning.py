"""Import shim: the reference's dataset module (dataset.py:9) derives BeatDataModule from
pytorch_lightning.LightningDataModule, whose only use there is save_hyperparameters() in the constructor.
pytorch_lightning is not installed here.  TEST INFRASTRUCTURE ONLY."""


class LightningDataModule:
    def save_hyperparameters(self, *args, **kwargs):
        pass
