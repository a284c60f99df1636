from . import build

if __name__ == "__main__":
    print(build(force=True, verbose=True))
