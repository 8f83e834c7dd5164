"""dirtorch.find_duplicates (extension): every pair of descriptors with exact score >= a threshold, their groups, or the
overlap of two sets."""
from dirb200.duplicates import find_duplicates_main

if __name__ == "__main__":
    find_duplicates_main()
