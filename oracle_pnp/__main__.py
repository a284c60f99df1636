from . import build

if __name__ == "__main__":
    print("oracle built:", build(force=True, verbose=True))
