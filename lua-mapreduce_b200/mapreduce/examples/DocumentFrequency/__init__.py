"""Document frequency: for every word, the number of files it occurs in -- the df of TF-IDF (see init.py)."""
