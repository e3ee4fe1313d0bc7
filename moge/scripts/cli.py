import os
os.environ['OPENCV_IO_ENABLE_OPENEXR'] = '1'
from pathlib import Path
import sys
if (_package_root := str(Path(__file__).absolute().parents[2])) not in sys.path:
    sys.path.insert(0, _package_root)

import click


@click.group(help='MoGe command line interface.')
def cli():
    pass


def main():
    from moge.scripts import infer, infer_panorama
    cli.add_command(infer.main, name='infer')
    cli.add_command(infer_panorama.main, name='infer_panorama')
    cli()


if __name__ == '__main__':
    main()
