"""dirtorch.cluster_features (extension): split a descriptor collection into K clusters with exact spherical k-means."""
from dirb200.cluster import cluster_features_main

if __name__ == "__main__":
    cluster_features_main()
