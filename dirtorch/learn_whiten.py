"""dirtorch.learn_whiten (extension): fit a PCA whitening on the GPU and store it in a checkpoint."""
from dirb200.pipeline import learn_whiten_main

if __name__ == "__main__":
    learn_whiten_main()
